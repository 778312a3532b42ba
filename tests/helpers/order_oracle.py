"""Independent oracle of the memory-ordering check (gsb_order_probe): its words, pairing, the words a CTA checks, and an
exhaustive enumerator of sequentially consistent interleavings of each litmus unit, against which the C classifier's
generalised (thresholded) predicates are proved on small iteration counts."""
import itertools

MP_RELACQ, MP_FENCE, SB_SC, IRIW_SC, CORR, MP_RELAXED = range(6)
UNITS = 6
MP_UNITS = (MP_RELACQ, MP_FENCE, MP_RELAXED)
ALLOWED, OVERLAP, WEAK, FORBIDDEN, CORRUPT, LOST = range(6)
M32 = 0xFFFFFFFF
KEY_SALT = 0x4F524452


def mix32(h):
    h &= M32
    h ^= h >> 16
    h = (h * 0x85EBCA6B) & M32
    h ^= h >> 13
    h = (h * 0xC2B2AE35) & M32
    h ^= h >> 16
    return h


def key(rank, slot):
    return mix32(((rank << 3) | slot) ^ KEY_SALT)


def word(seed, k, i):
    return (i << 32) | mix32(seed ^ k ^ i)


def distances(n, seed):
    return [1, n // 2, 1 + seed % (n - 1)]


def iriw_step(n, d):
    """The first e of d, d + 1, ... (1..n-1, wrapping) with e, 2e, 3e all nonzero mod n."""
    e = d % n or 1
    for _ in range(n):
        if all(k * e % n for k in (1, 2, 3)):
            return e
        e = 1 if e + 1 == n else e + 1
    return 0


def pairing(unit, n, d, r):
    if unit == SB_SC:
        return [(r + d) % n, (r - d) % n]
    if unit == IRIW_SC:
        e = iriw_step(n, d)
        return [(r - 2 * e) % n, (r - e) % n, (r + e) % n]
    return [(r + d) % n]


def iriw_instance(n, d, r):
    """The four CTAs of the IRIW instance CTA r classifies: writer of x, writer of y, reader A (r), reader B."""
    x, y, other = pairing(IRIW_SC, n, d, r)
    return x, y, r, other


OBS_READS = {MP_RELACQ: 5, MP_FENCE: 5, MP_RELAXED: 5, SB_SC: 2, IRIW_SC: 4, CORR: 2}
FINAL_READS = {MP_RELACQ: 5, MP_FENCE: 5, MP_RELAXED: 5, SB_SC: 1, IRIW_SC: 2, CORR: 1}


def words_per_cta(unit, observations):
    """u64 words one CTA reads and checks in one launch: every observation's reads, then the final reads."""
    return OBS_READS[unit] * observations + FINAL_READS[unit]


# ---- the textbook litmus tests, binary: a judged outcome is forbidden iff no SC interleaving produces it

def forbidden_binary(unit, it, i=0):
    """The oracle's predicate on one observation's iterations (as gsb_order_classify takes the words)."""
    if unit in MP_UNITS:
        return min(it[1:5]) < it[0]
    if unit == SB_SC:
        a, b = it[0], it[1]
        return (a < i and b < i) or (a > i and b > i)
    if unit == IRIW_SC:
        a, b, c, d = it[:4]
        return a > d and c > b
    return it[1] < it[0] or it[2] < it[1]  # CORR


def _interleavings(threads):
    """Every interleaving of the threads' op lists (each op a callable on the shared state returning a read or None)."""
    n = len(threads)
    total = sum(len(t) for t in threads)

    def rec(pos, state, reads):
        if sum(pos) == total:
            yield reads
            return
        for t in range(n):
            if pos[t] < len(threads[t]):
                kind, loc, val, tag = threads[t][pos[t]]
                st = dict(state)
                rd = dict(reads)
                if kind == "w":
                    st[loc] = val
                else:
                    rd[tag] = st.get(loc, 0)
                p = list(pos)
                p[t] += 1
                yield from rec(tuple(p), st, rd)

    yield from rec(tuple([0] * n), {}, {})


def sc_outcomes(unit, m):
    """The set of read-value tuples an SC interleaving of the unit's litmus test with m iterations per writer reaches.

    MP: writer stores d0..d3 then f for i = 1..m; reader reads f then d0..d3 once -> (f, d0, d1, d2, d3).
    SB: two threads, each stores its x = i, then reads the other's, for i = 1..m -> (a_1..a_m, b_1..b_m).
    IRIW: writers x = 1..m and y = 1..m; reader A reads x then y, reader B y then x, once -> (a, b, c, d).
    CORR: writer x = 1..m; reader reads x four times (two observations) -> (r1, r2, r3, r4).
    (Fences are no-ops under SC; every fenced unit is judged against these outcomes.)"""
    if unit in MP_UNITS:
        w = [op for i in range(1, m + 1) for op in
             [("w", f"d{j}", i, None) for j in range(4)] + [("w", "f", i, None)]]
        r = [("r", "f", None, 0)] + [("r", f"d{j}", None, 1 + j) for j in range(4)]
        threads, width = [w, r], 5
    elif unit == SB_SC:
        a = [op for i in range(1, m + 1) for op in (("w", "x", i, None), ("r", "y", None, i - 1))]
        b = [op for i in range(1, m + 1) for op in (("w", "y", i, None), ("r", "x", None, m + i - 1))]
        threads, width = [a, b], 2 * m
    elif unit == IRIW_SC:
        threads = [[("w", "x", i, None) for i in range(1, m + 1)], [("w", "y", i, None) for i in range(1, m + 1)],
                   [("r", "x", None, 0), ("r", "y", None, 1)], [("r", "y", None, 2), ("r", "x", None, 3)]]
        width = 4
    else:
        threads = [[("w", "x", i, None) for i in range(1, m + 1)], [("r", "x", None, j) for j in range(4)]]
        width = 4
    return {tuple(r[j] for j in range(width)) for r in _interleavings(threads)}


def judged(unit, outcome, m):
    """The observations gsb_order_classify judges in one SC outcome: (iterations as it takes them, iteration)."""
    if unit in MP_UNITS or unit == IRIW_SC:
        return [(list(outcome), 0)]
    if unit == SB_SC:
        return [([outcome[i - 1], outcome[m + i - 1]], i) for i in range(1, m + 1)]
    r = outcome  # CORR: the first observation follows the initial value
    return [([0, r[0], r[1]], 0), ([r[1], r[2], r[3]], 0)]
