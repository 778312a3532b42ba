"""CPU oracle of gsb_shared_atomic_probe — TEST INFRASTRUCTURE ONLY (the product never imports it).

Restates, with Python integers and numpy, the shared-memory atomic check of gsb_shared_atomic.h: one CTA's area, the
value of every contribution, and the words a clean run leaves. The hash, the float integers and their f16 / bf16
encoders are the L2 atomic oracle's (atomic_oracle.py). Float words are summed as integers, with each word's sum of
magnitudes asserted under the type's exact bound, then encoded. TICKET's and CAS's slots are checked as permutations of
the contributor ids, and exchanged values as the values of ids 0 .. COUNT (COUNT's being the starting word), each once.
"""
from __future__ import annotations

import struct

import numpy as np

from tests.helpers import atomic_oracle as ao

INT32, WIDE, FLOAT, TICKET, CAS = range(5)
UNITS = range(5)
NAMES = ["int32", "wide", "float", "ticket", "cas"]
THREADS, WARPS, REPS = 256, 8, 4
SPREAD_BYTES, HOT_WORDS, HOT_STRIDE = 8192, 32, 128
AREA_BYTES = SPREAD_BYTES + HOT_WORDS * HOT_STRIDE
AREA_WORDS = AREA_BYTES // 4
COUNT = WARPS * REPS  # contributions to a hot word of one CTA
ENTRIES = COUNT + 1
FORMS = 4
NO_ID = 0xFFFFFFFF
TAG, BOUND_TAG, EXCH_TAG, PAIR_TAG = 0x00400000, 0x00200000, 0x00100000, 0x00080000
M32, M64 = (1 << 32) - 1, (1 << 64) - 1
TICKET_EXCH = {1: 16, 2: 32, 3: 48}  # byte offset in the hot slot of form f's exchange word
EXCH_WORDS = {1: 1, 2: 2, 3: 4}
CAS64, CAS128 = 8, 16
SPREAD, HOT = 0, 1
BOUND = {"f32": 1 << 24, "f64": 1 << 53, "f16": 1 << 11, "bf16": 1 << 8}


def ub(unit: int) -> int:
    return 8 if unit in (WIDE, FLOAT) else 4


def n_units(unit: int) -> int:
    return AREA_BYTES // ub(unit)


def has_spread(unit: int) -> bool:
    return unit not in (TICKET, CAS)


def rounds(unit: int) -> int:
    return 2 * (SPREAD_BYTES // ub(unit) // THREADS)


def spread_unit(unit: int, t: int, r: int) -> int:
    n = SPREAD_BYTES // ub(unit)
    k, warp, lane = r // 2, t // 32, t % 32
    if r % 2:
        return (t * 32 + k) % n
    return k * THREADS + warp * 32 + (lane + 4 * k + warp) % 32


def hot_unit(unit: int, lane: int) -> int:
    return (SPREAD_BYTES + lane * HOT_STRIDE) // ub(unit)


def logical(unit: int, u: int) -> int:
    b = u * ub(unit)
    return (b - SPREAD_BYTES) // HOT_STRIDE if b >= SPREAD_BYTES else u


def kind(unit: int, u: int) -> int:
    return logical(unit, u) % {INT32: 10, WIDE: 6, FLOAT: 4}.get(unit, 1)


def h32(seed: int, a: int, b: int) -> int:
    return int(ao._hash(seed, a & M32, b & M32)[0])


def h64(seed: int, a: int, b: int) -> int:
    return int(ao.hash64(seed, np.uint32(a & M32), b & M32)[0])


def key(unit: int, seed: int, phase: int, t: int, r: int) -> int:
    return h64(seed, unit << 28 | phase << 27 | TAG, t * 32 + r)


def init_key(unit: int, seed: int, u: int) -> int:
    return h64(seed, unit << 28 | ao.INIT_TAG | TAG, u)


def bound(unit: int, seed: int, x: int) -> int:
    return 8 + h32(seed, unit << 28 | BOUND_TAG, x) % 24


def exch(seed: int, f: int, lane: int, ident: int, c: int) -> int:
    return h32(seed, TICKET << 28 | EXCH_TAG | f << 8 | lane, ident * 4 + c)


def exch_value(seed: int, f: int, lane: int, ident: int) -> int:
    """form f's exchanged value of id `ident` as one integer (little-endian words)"""
    return sum(exch(seed, f, lane, ident, c) << (32 * c) for c in range(EXCH_WORDS[f]))


def cas64_start(seed: int, lane: int) -> int:
    return h32(seed, CAS << 28 | PAIR_TAG, lane) << 32


def pair(seed: int, lane: int, count: int) -> int:
    return h64(seed, CAS << 28 | PAIR_TAG | 1 << 8 | lane, count & M32)


def _ival(fmt: str, phase: int, h: int) -> int:
    op = {"f32": ao.FADD32, "f64": ao.FADD64, "half": ao.HADD2}[fmt]
    return int(ao.ival(op, phase, np.uint64(h))[()])


def _init_ival(fmt: str, phase: int, h: int) -> int:
    if fmt == "half":
        return _ival(fmt, phase, h)
    return (h & M32) % 255 - 127


def _f32(v: int) -> int:
    return struct.unpack("<I", struct.pack("<f", float(v)))[0]


def _f64(v: int) -> int:
    return struct.unpack("<Q", struct.pack("<d", float(v)))[0]


def _half2(k: int, lo: int, hi: int) -> int:
    enc = ao._bf16 if k else ao._f16
    return int(enc(np.array([lo]))[0]) | int(enc(np.array([hi]))[0]) << 16


def contributions(unit: int):
    """(phase, thread, round or repetition, unit) of every contribution of one CTA, in issue order per thread"""
    out = []
    if has_spread(unit):
        for t in range(THREADS):
            for r in range(rounds(unit)):
                out.append((SPREAD, t, r, spread_unit(unit, t, r)))
        for t in range(THREADS):
            for r in range(REPS):
                out.append((HOT, t, r, hot_unit(unit, t % 32)))
    return out


def init_units(unit: int, seed: int) -> list:
    """the starting value of every unit, in the unit's bits"""
    w = []
    for u in range(n_units(unit)):
        h = init_key(unit, seed, u)
        k, hot = kind(unit, u), u * ub(unit) >= SPREAD_BYTES
        phase = HOT if hot else SPREAD
        hi = h & (M32 << 32)
        if unit == INT32:
            v = {1: M32, 2: 0, 4: 0x7FFFFFFF, 5: 0x80000000, 6: M32, 7: 0}.get(k, h & M32)
            if k in (8, 9):
                v = (h & M32) % 40
        elif unit == WIDE:
            v = {1: M64, 2: 0, 4: (1 << 63) - 1, 5: 0}.get(k, h)
        elif unit == FLOAT:
            if k == 0:
                v = hi | _f32(_init_ival("f32", phase, h))
            elif k == 1:
                v = _f64(_init_ival("f64", phase, h))
            else:
                v = hi | _half2(k - 2, _init_ival("half", phase, h & 0xFFFF), _init_ival("half", phase, (h >> 16) & 0xFFFF))
        else:
            v = h & M32
            if hot:
                off, lane = (u * 4 - SPREAD_BYTES) % HOT_STRIDE, (u * 4 - SPREAD_BYTES) // HOT_STRIDE
                if off == 0:
                    v = 0
                elif unit == TICKET:
                    for f, o in TICKET_EXCH.items():
                        if o <= off < o + 4 * EXCH_WORDS[f]:
                            v = exch(seed, f, lane, COUNT, (off - o) // 4)
                else:
                    if off in (CAS64, CAS64 + 4):
                        v = (cas64_start(seed, lane) >> (8 * (off - CAS64))) & M32
                    elif CAS128 <= off < CAS128 + 8:
                        v = 0
                    elif off in (CAS128 + 8, CAS128 + 12):
                        v = (pair(seed, lane, 0) >> (8 * (off - CAS128 - 8))) & M32
        w.append(v)
    return w


def abs_sums(unit: int, seed: int, skip=False):
    """FLOAT: (sums, sums of magnitudes), two per unit (the halves; f32 and f64 use the first), starting value in"""
    s = [[0, 0] for _ in range(n_units(unit))]
    a = [[0, 0] for _ in range(n_units(unit))]

    def add(u, i, v):
        s[u][i] += v
        a[u][i] += abs(v)
    for u in range(n_units(unit)):
        h, k = init_key(unit, seed, u), kind(unit, u)
        phase = HOT if u * 8 >= SPREAD_BYTES else SPREAD
        if k < 2:
            add(u, 0, _init_ival("f32" if k == 0 else "f64", phase, h))
        else:
            add(u, 0, _init_ival("half", phase, h & 0xFFFF))
            add(u, 1, _init_ival("half", phase, (h >> 16) & 0xFFFF))
    for phase, t, r, u in ([] if skip else contributions(unit)):
        h, k = key(unit, seed, phase, t, r), kind(unit, u)
        if k < 2:
            add(u, 0, _ival("f32" if k == 0 else "f64", phase, h))
        else:
            add(u, 0, _ival("half", phase, h & 0xFFFF))
            add(u, 1, _ival("half", phase, (h >> 16) & 0xFFFF))
    return s, a


def _to_words(unit: int, units: list) -> np.ndarray:
    out = []
    for v in units:
        out += [(v >> (32 * i)) & M32 for i in range(ub(unit) // 4)]
    return np.array(out, dtype=np.uint64)


def expected(unit: int, seed: int, skip=False, lose=None) -> np.ndarray:
    """the AREA_WORDS words of one CTA after a clean run (skip: a CTA that issued nothing; lose: the index into
    contributions(unit) of one contribution the atomic unit dropped)"""
    w = init_units(unit, seed)
    if unit == FLOAT:
        s, a = abs_sums(unit, seed, skip)
        if lose is not None:  # restate without that contribution
            phase, t, r, u = contributions(unit)[lose]
            h, k = key(unit, seed, phase, t, r), kind(unit, u)
            if k < 2:
                s[u][0] -= _ival("f32" if k == 0 else "f64", phase, h)
            else:
                s[u][0] -= _ival("half", phase, h & 0xFFFF)
                s[u][1] -= _ival("half", phase, (h >> 16) & 0xFFFF)
        for u in range(n_units(unit)):
            k, hi = kind(unit, u), w[u] & (M32 << 32)
            if k == 0:
                assert a[u][0] < BOUND["f32"]
                w[u] = hi | _f32(s[u][0])
            elif k == 1:
                assert a[u][0] < BOUND["f64"]
                w[u] = _f64(s[u][0])
            else:
                assert max(a[u]) < BOUND["bf16" if k == 3 else "f16"]
                w[u] = hi | _half2(k - 2, s[u][0], s[u][1])
        return _to_words(unit, w)
    contrib = [] if skip else contributions(unit)
    for i, (phase, t, r, u) in enumerate(contrib):
        if i == lose:
            continue
        h, k = key(unit, seed, phase, t, r), kind(unit, u)
        x = w[u]
        if unit == WIDE:
            one = 1 << ((h & M32) % 64)
            v = {1: ~one & M64, 2: one}.get(k, h)
            s64 = lambda z: z - (1 << 64) if z >> 63 else z  # noqa: E731
            w[u] = [(x + v) & M64, x & v, x | v, x ^ v, v if s64(v) < s64(x) else x, max(v, x)][k]
            continue
        one = 1 << ((h & M32) % 32)
        v = {1: ~one & M32, 2: one, 8: bound(unit, seed, logical(unit, u)), 9: bound(unit, seed, logical(unit, u))}.get(
            k, h & M32)
        s32 = lambda z: z - (1 << 32) if z >> 31 else z  # noqa: E731
        w[u] = [(x + v) & M32, x & v, x | v, x ^ v, v if s32(v) < s32(x) else x, v if s32(v) > s32(x) else x,
                min(v, x), max(v, x), 0 if x >= v else x + 1, v if x == 0 or x > v else x - 1][k]
    words = _to_words(unit, w)
    if unit in (TICKET, CAS) and not skip:
        for lane in range(HOT_WORDS):
            base = (SPREAD_BYTES + lane * HOT_STRIDE) // 4
            words[base] = COUNT
            if unit == CAS:
                c64, p = cas64_start(seed, lane) + COUNT, pair(seed, lane, COUNT)
                words[base + 2], words[base + 3] = c64 & M32, c64 >> 32
                words[base + 4:base + 8] = [COUNT, 0, p & M32, p >> 32]
    return words


def compared(unit: int) -> np.ndarray:
    """mask of the words the kernel compares: all but TICKET's exchange words"""
    m = np.ones(AREA_WORDS, dtype=bool)
    if unit == TICKET:
        for lane in range(HOT_WORDS):
            base = SPREAD_BYTES + lane * HOT_STRIDE
            for f, o in TICKET_EXCH.items():
                m[(base + o) // 4:(base + o) // 4 + EXCH_WORDS[f]] = False
    return m


def mismatch(unit: int, want: np.ndarray, got: np.ndarray):
    """(words, bits) that differ, over the compared words"""
    m = compared(unit)
    x = (np.asarray(want, dtype=np.uint64) ^ np.asarray(got, dtype=np.uint64))[m]
    return int((x != 0).sum()), int(sum(bin(int(v)).count("1") for v in x))


def words_per_cta(unit: int) -> int:
    return int(compared(unit).sum())


def issued_per_cta(unit: int) -> int:
    if has_spread(unit):
        return THREADS * (rounds(unit) + REPS)
    return THREADS * REPS * (4 if unit == TICKET else 3)


def clean_slots(unit: int, seed: int, order=None) -> dict:
    """one CTA's slots after a clean run, as {(form, lane): [entry, ...]}: add / CAS forms hold the id of each ticket,
    exchange forms the value returned to each id and then the final word. `order` permutes the contributors (the order
    the atomic unit served them in)."""
    order = list(range(COUNT)) if order is None else list(order)
    out = {}
    forms = 4 if unit == TICKET else 3
    for lane in range(HOT_WORDS):
        for f in range(forms):
            if unit == CAS or f == 0:
                ent = [0] * COUNT
                for ticket, ident in enumerate(order):
                    ent[ticket] = ident
            else:
                prev, ent = exch_value(seed, f, lane, COUNT), [0] * ENTRIES
                for ident in order:
                    ent[ident], prev = prev, exch_value(seed, f, lane, ident)
                ent[COUNT] = prev
            out[(f, lane)] = ent
    return out


def bad_entries(unit: int, seed: int, slots: dict, torn=()) -> int:
    """entries that do not name every contributor once (exchange forms: the values of ids 0 .. COUNT), plus every b128
    pair in `torn` (a count and an upper half) whose halves do not belong together"""
    bad = 0
    for (f, lane), ent in slots.items():
        if unit == TICKET and f > 0:
            want = {exch_value(seed, f, lane, i): i for i in range(COUNT + 1)}
            ids = [want.get(v) for v in ent]
            limit = COUNT + 1
        else:
            ids, limit = list(ent), COUNT
        seen = set()
        for i in ids:
            if i is None or not 0 <= i < limit or i in seen:
                bad += 1
            else:
                seen.add(i)
    for lane, (count, hi) in torn:
        bad += hi != pair(seed, lane, count)
    return bad


def skipped_slots(unit: int, seed: int) -> dict:
    """the slots of a CTA that issued nothing: every entry empty, the exchange words' final value their start"""
    out = {}
    for lane in range(HOT_WORDS):
        for f in range(4 if unit == TICKET else 3):
            if unit == TICKET and f > 0:
                out[(f, lane)] = [NO_ID] * COUNT + [exch_value(seed, f, lane, COUNT)]
            else:
                out[(f, lane)] = [NO_ID] * COUNT
    return out


# ---- DSMEM and REDAS: every other rank of a cluster sends its atomics into a rank's area

DSMEM, REDAS = 5, 6
CLUSTER_UNITS = (DSMEM, REDAS)
ALL_UNITS = range(7)
ALL_NAMES = NAMES + ["dsmem", "redas"]
DSMEM_U64, DSMEM_F32, DSMEM_CAS = 1024, 2048, 2816
PEER_OPS = {DSMEM: 9, REDAS: 5}
REDAS_BYTES = 24  # one thread to one peer: add.u32 4, add.u64 8, xor 4, max 4, inc 4


def peer_key(unit: int, seed: int, q: int, t: int, j: int) -> int:
    return h64(seed, unit << 28 | TAG | q << 8, t * 32 + j)


def peer_word(unit: int, t: int, j: int) -> int:
    if unit == DSMEM:
        if j < 4:
            return t + 256 * j
        if j < 6:
            return DSMEM_U64 + 2 * (t + 256 * (j - 4))
        if j < 9:
            return DSMEM_F32 + t + 256 * (j - 6)
        return DSMEM_CAS + 8 * (t % 32)
    return [t, 256 + 2 * t, 768 + t, 1024 + t, 1280 + t][j]


def cluster_init(unit: int, seed: int) -> list:
    w = []
    for i in range(AREA_WORDS):
        h = init_key(unit, seed, i) & M32
        if unit == DSMEM:
            v = h
            if DSMEM_F32 <= i < DSMEM_CAS:
                v = _f32(_init_ival("f32", SPREAD, h))
            elif i >= DSMEM_CAS and (i - DSMEM_CAS) % 8 == 0:
                v = 0
        else:
            v = 0x80000000 if 1024 <= i < 1280 else h % 40 if 1280 <= i < 1536 else h
        w.append(v)
    return w


def cluster_expected(unit: int, seed: int, n: int, rank: int, skip_sender=None) -> np.ndarray:
    """rank `rank`'s area in a cluster of n after every other rank (but skip_sender) sent its atomics"""
    w = cluster_init(unit, seed)
    fsum = {i: _init_ival("f32", SPREAD, init_key(unit, seed, i) & M32) for i in range(DSMEM_F32, DSMEM_CAS)}
    fabs = {i: abs(v) for i, v in fsum.items()}
    s32 = lambda z: z - (1 << 32) if z >> 31 else z  # noqa: E731
    for q in range(n):
        if q == rank or q == skip_sender:
            continue
        for t in range(THREADS):
            for j in range(PEER_OPS[unit] + (unit == DSMEM)):
                i = peer_word(unit, t, j)
                if unit == DSMEM and j == 9:  # the cas.b32 increment
                    w[i] += 1
                    continue
                h = peer_key(unit, seed, q, t, j)
                if (unit == DSMEM and j in (4, 5)) or (unit == REDAS and j == 1):
                    x = (w[i] | w[i + 1] << 32) + h & M64
                    w[i], w[i + 1] = x & M32, x >> 32
                elif unit == DSMEM and j >= 6:
                    f = _ival("f32", SPREAD, h)
                    fsum[i] += f
                    fabs[i] += abs(f)
                elif unit == DSMEM or j == 0:
                    w[i] = (w[i] + h) & M32
                elif j == 2:
                    w[i] ^= h & M32
                elif j == 3:
                    w[i] = h & M32 if s32(h & M32) > s32(w[i]) else w[i]
                else:  # inc.u32 with the word's bound
                    b = bound(unit, seed, t)
                    w[i] = 0 if w[i] >= b else w[i] + 1
    if unit == DSMEM:
        for i, v in fsum.items():
            assert fabs[i] < BOUND["f32"]
            w[i] = _f32(v)
    return np.array(w, dtype=np.uint64)


def cluster_issued_per_cta(unit: int, n: int) -> int:
    return THREADS * (n - 1) * (PEER_OPS[unit] + (unit == DSMEM))
