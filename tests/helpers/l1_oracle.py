"""Independent numpy model of the L1 and constant-cache check (gsb_l1_probe): the HBM probe's pattern words, the read
schedule of every unit, L1_STORE's byte ranges and merged words, the TEX unit's clamp and border answers, the words
each CTA compares, the counts a wrong seed_expect must give, and gsb_fault_classify's four classes. Written from the
description in include/gpushare_b200.h and csrc/gsb_pattern.h, not from the C code."""
import numpy as np

L1_LOAD, L1_STORE, NC, TEX, CONST, PARAM = range(6)
UNITS = range(6)
NAMES = ["l1_load", "l1_store", "nc", "tex", "const", "param"]
THREADS, REGION, STEPS, LINE = 1024, 8192, 8, 8
WIDTH, ROWS, READS_2D, X0, XS, EDGE = 64, 128, 16384, 32, 128, 8
CONST_WORDS, PARAM_WORDS = 4096, 2000
ZERO_TEXEL = (1 << 63) - 1
# forms per unit and reads per thread of each form
FORMS = {L1_LOAD: 3, L1_STORE: 2, NC: 1, TEX: 3, CONST: 2, PARAM: 2}
HOOK_WORDS = {L1_LOAD: REGION, L1_STORE: REGION, NC: REGION, TEX: REGION + 2 * READS_2D, CONST: CONST_WORDS,
              PARAM: PARAM_WORDS}
K = np.array([0x9E3779B1, 0x85EBCA77, 0xC2B2AE3D, 0x27D4EB2F], dtype=np.uint64)
C = np.array([0x165667B1, 0xD3A2646C, 0xFD7046C5, 0xB55A4F09], dtype=np.uint64)
M32 = np.uint64(0xFFFFFFFF)
ZERO, STALE, ALIASED, BITS = 1, 2, 3, 4


def mix32(h):
    h = np.asarray(h, dtype=np.uint64) & M32
    h ^= h >> np.uint64(16)
    h = (h * np.uint64(0x85EBCA6B)) & M32
    h ^= h >> np.uint64(13)
    h = (h * np.uint64(0xC2B2AE35)) & M32
    h ^= h >> np.uint64(16)
    return h


def seed_key(seed):
    return int(mix32(np.uint64(seed ^ 0xA5A5A5A5)))


def gen2_seed(seed):
    return ~seed & 0xFFFFFFFF


def pattern(w, key):
    """(n, 4) uint32 pattern words of word indices w under the mixed key."""
    w = np.atleast_1d(np.asarray(w, dtype=np.uint64))
    m = mix32((w & M32) ^ (((w >> np.uint64(32)) * np.uint64(0x9E3779B1)) & M32))
    lanes = ((m[:, None] * K[None, :] + C[None, :]) & M32) ^ np.uint64(key)
    return lanes.astype(np.uint32)


def order(p, q):
    """region word of sequence position q in pass p of L1_LOAD / NC"""
    q = np.asarray(q, dtype=np.int64)
    kind = 0 if p == 0 else (p - 1) % 5
    if kind == 0:
        return q
    if kind == 1:
        return REGION - 1 - q
    s = {2: 32, 3: 128, 4: 512}[kind]
    g = (REGION // LINE) // s
    line = q // LINE
    return ((line % g) * s + line // g) * LINE + q % LINE


def store_span(w):
    """(lo, width) of the bytes L1_STORE overwrites in buffer words w"""
    w = np.asarray(w, dtype=np.uint64)
    h = mix32((w & M32) ^ (((w >> np.uint64(32)) * np.uint64(0x85EBCA77)) & M32) ^ np.uint64(0x4C315354))
    width = np.left_shift(1, (h % np.uint64(5)).astype(np.int64))
    lo = ((h >> np.uint64(8)) % (16 // width).astype(np.uint64)).astype(np.int64) * width
    return lo, width


def writer(i):
    return (np.asarray(i) % THREADS) ^ 512


def merged(w, seed):
    """(n, 4) words L1_STORE reads back: generation 2 bytes over [lo, lo + width), generation 1 elsewhere"""
    w = np.atleast_1d(np.asarray(w, dtype=np.uint64))
    g1 = pattern(w, seed_key(seed)).view(np.uint8).reshape(-1, 16)
    g2 = pattern(w, seed_key(gen2_seed(seed))).view(np.uint8).reshape(-1, 16)
    lo, width = store_span(w)
    b = np.arange(16)[None, :]
    sel = (b >= lo[:, None]) & (b < (lo + width)[:, None])
    return np.where(sel, g2, g1).astype(np.uint8).view(np.uint32).reshape(-1, 4)


def tex_coord(i, c, ctas):
    i = np.asarray(i, dtype=np.int64)
    dy = -EDGE if c == 0 else EDGE if c == ctas - 1 else 0
    return i % XS - X0, c * ROWS + i // XS + dy


def texel(x, y, rows, clamp):
    """buffer word of the texel a 2-D read at (x, y) returns, -1 for a border read outside the array"""
    x, y = np.asarray(x), np.asarray(y)
    inside = (x >= 0) & (x < WIDTH) & (y >= 0) & (y < rows)
    w = np.clip(y, 0, rows - 1) * WIDTH + np.clip(x, 0, WIDTH - 1)
    return w if clamp else np.where(inside, w, -1)


def steps(unit, form):
    if form >= FORMS[unit]:
        return 0
    if unit == TEX and form > 0:
        return READS_2D // THREADS
    if unit == CONST:
        return CONST_WORDS if form == 0 else CONST_WORDS // THREADS
    if unit == PARAM:
        return PARAM_WORDS if form == 0 else 2
    return STEPS


def schedule(unit, form, p, c, ctas, t, s):
    """the word read (t, s) of pass p of form `form` returns (-1: none; ZERO_TEXEL: border)"""
    q = s * THREADS + t
    base = c * REGION
    if unit in (L1_LOAD, NC):
        return base + int(order(p, q))
    if unit == L1_STORE or (unit == TEX and form == 0):
        return base + q
    if unit == TEX:
        x, y = tex_coord(q, c, ctas)
        w = int(texel(x, y, ctas * ROWS, form == 1))
        return ZERO_TEXEL if w < 0 else w
    if form == 0:
        return s
    return q if unit == CONST or q < PARAM_WORDS else -1


def words_per_cta(unit, passes=8):
    """16-byte words one CTA compares in one launch"""
    if unit == L1_LOAD:
        return 3 * passes * REGION
    if unit == NC:
        return passes * REGION
    if unit == L1_STORE:
        return 2 * REGION
    if unit == TEX:
        return REGION + 2 * READS_2D
    if unit == CONST:
        return THREADS * CONST_WORDS + CONST_WORDS
    return THREADS * PARAM_WORDS + PARAM_WORDS


def _popcount(a):
    a = np.asarray(a, dtype=np.uint32)
    return np.unpackbits(a.view(np.uint8)).reshape(a.shape + (32,)).sum(axis=-1)


def wrong_seed_counts(unit, c, ctas, seed, seed_expect, passes=8):
    """(mismatch_words, mismatch_bits) one CTA finds when the data carry `seed` and it expects `seed_expect`"""
    ks, ke = seed_key(seed), seed_key(seed_expect)
    per_word = int(_popcount(np.array([ks ^ ke], dtype=np.uint32))[0]) * 4 if ks != ke else 0
    intact = per_word != 0
    if unit in (L1_LOAD, NC):
        n = words_per_cta(unit, passes) if intact else 0
        return n, n * per_word
    if unit == L1_STORE:
        w = np.arange(c * REGION, (c + 1) * REGION, dtype=np.uint64)
        bits = _popcount(merged(w, seed) ^ merged(w, seed_expect)).sum(axis=1)
        return REGION * intact + int((bits != 0).sum()), REGION * per_word + int(bits.sum())
    if unit == TEX:
        x, y = tex_coord(np.arange(READS_2D), c, ctas)
        inside = int((texel(x, y, ctas * ROWS, False) >= 0).sum())
        n = (REGION + READS_2D + inside) if intact else 0
        return n, n * per_word
    n = words_per_cta(unit) if intact else 0
    return n, n * per_word


def _intact_key(w, obs):
    base = pattern([w], 0)[0]
    k = np.asarray(obs, dtype=np.uint32) ^ base
    return int(k[0]) if (k == k[0]).all() else None


def classify(offset, expected, observed):
    """(cls, alias_bit, seed_key) of one wrong word, by the rules of gsb_fault_classify"""
    w = offset >> 4
    if not any(int(x) for x in observed):
        return ZERO, 0xFFFFFFFF, 0
    ek, ok = _intact_key(w, expected), _intact_key(w, observed)
    if ok is not None and not (ek is not None and ek == ok):
        return STALE, 0xFFFFFFFF, ok
    for k in range(40):
        ak = _intact_key(w ^ (1 << k), observed)
        if ak is not None:
            return ALIASED, k, ak
    return BITS, 0xFFFFFFFF, 0
