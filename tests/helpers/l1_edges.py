"""The L1 and constant-cache check at its edges: the cases gsb_test_l1_table runs on the twins l1_from_table<UNIT>, and
an exact reference for each. Written from the description of gsb_test_l1_table in include/gpushare_b200.h, not from the
C code: the L1_STORE rounds are replayed byte by byte in numpy (no gsb_copy_merge), the texture answers come from this
file's own texel model (clamp to the nearest edge texel, 0 outside under border), and every other word is the HBM
probe's pattern word of its own index (tests/helpers/l1_oracle.py)."""
from dataclasses import dataclass, field

import numpy as np

from tests.helpers import l1_oracle as lo

THREADS, WARPS, LINE = lo.THREADS, lo.THREADS // 32, lo.LINE
L1_BYTES = 256 * 1024  # the H100's combined L1 data cache and shared memory per SM
REGION_MAX, ROUNDS_MAX, WORD_BITS = 131072, 8, 17
RESIDENT, READ_OWN = 1, 2
TEX_1D = 0x80000000
K0 = 0x9E3779B1
CONST_WORDS, PARAM_WORDS = lo.CONST_WORDS, lo.PARAM_WORDS
TEX_XS = (-(1 << 20), -65, -1, 0, lo.WIDTH - 1, lo.WIDTH, lo.WIDTH + 64, 1 << 20)
TEX_YS = (-(1 << 20), -65, -1, 0, lo.WIDTH - 1, lo.WIDTH, lo.ROWS - 1, lo.ROWS, lo.ROWS + 64, 1 << 20)


def gen_seed(seed, g):
    """the seed whose pattern generation g of a store case stores (0: the probe's seed, the fill)"""
    return (seed ^ (g * K0)) & 0xFFFFFFFF


def entry(word, start, width, gen):
    """one L1_STORE table entry: generation gen over bytes [start, start + width) of region word `word`"""
    return int(word) | int(start) << WORD_BITS | int(width).bit_length() << (WORD_BITS + 4) | int(gen) << 24


def unpack(e):
    e = np.asarray(e, dtype=np.int64)
    code = e >> (WORD_BITS + 4) & 7
    return e & ((1 << WORD_BITS) - 1), e >> WORD_BITS & 15, np.where(code > 0, 1 << np.maximum(code - 1, 0), 0), e >> 24


@dataclass
class Case:
    name: str
    unit: int
    region_words: int
    table: np.ndarray                            # uint32, as gsb_test_l1_table takes it
    rounds: list = field(default_factory=list)   # L1_STORE: per round, 1024 entries (0: no store)
    flags: int = 0

    @property
    def passes(self):
        return len(self.table) // self.region_words if self.unit in (lo.L1_LOAD, lo.NC) else 0


# ---- loads ------------------------------------------------------------------------------------------------------

def _load(name, unit, region, passes):
    """passes: (p, steps, THREADS) region word indices"""
    t = np.asarray(passes, dtype=np.int64)
    assert t.shape[1:] == (region // THREADS, THREADS)
    return Case(name, unit, region, t.astype(np.uint32).ravel())


def _warp_reads(steps):
    """(steps, THREADS) arrays of each read's step k, warp w and lane l"""
    k, t = np.meshgrid(np.arange(steps), np.arange(THREADS), indexing="ij")
    return k, t // 32, t % 32


def broadcast(unit):
    """every lane of a warp reads the same word"""
    region = lo.REGION
    k, w, _ = _warp_reads(region // THREADS)
    return _load("broadcast", unit, region, [((k * WARPS + w) * 37 + 5 * p) % region for p in range(2)])


def same_set_gather(unit, stride_kib):
    """every warp's 32 lanes read 32 different lines stride_kib KiB apart: lines with the same set bits"""
    s = stride_kib * 1024 // (LINE * 16)  # lines per stride
    region = 32 * s * LINE
    k, w, lane = _warp_reads(region // THREADS)
    j = k * WARPS + w
    idx = ((j % s) + lane * s) * LINE + (j // s) % LINE
    return _load(f"gather_{stride_kib}k", unit, region, [idx, idx])


def sectors(unit):
    """every warp reads one 32-byte sector of one line, and every sector of every line is read once"""
    region, steps = lo.REGION, lo.REGION // THREADS
    lines = region // LINE
    n_passes = 4 * lines // (steps * WARPS)
    out = []
    for p in range(n_passes):
        k, w, lane = _warp_reads(steps)
        j = (p * steps + k) * WARPS + w
        out.append((j % lines) * LINE + (j // lines) * 2 + (lane & 1))
    return _load("sectors", unit, region, out)


def strided(region, q, stride_lines=512):
    """region word of position q in a pass that visits lines stride_lines apart back to back"""
    groups = region // LINE // stride_lines
    line = q // LINE
    return ((line % groups) * stride_lines + line // groups) * LINE + q % LINE


def capacity(unit, times):
    """a region `times` the L1's size, read twice in address order, then twice at 64 KiB line strides"""
    region = times * L1_BYTES // 16
    q = np.arange(region).reshape(region // THREADS, THREADS)
    return _load(f"capacity_{times}x", unit, region, [q, q, strided(region, q), strided(region, q)])


def load_cases(unit):
    return [broadcast(unit), *[same_set_gather(unit, s) for s in (4, 16, 64)], sectors(unit), capacity(unit, 2),
            capacity(unit, 4)]


# ---- stores ---------------------------------------------------------------------------------------------------

def _store(name, rounds, flags, region=lo.REGION):
    """rounds: per round a dict thread -> (word, start, width, gen)"""
    ents = []
    for r in rounds:
        e = np.zeros(THREADS, dtype=np.uint32)
        for t, s in r.items():
            e[t] = entry(*s)
        ents.append(e)
    table = np.concatenate([np.array([flags], dtype=np.uint32), *ents])
    return Case(name, lo.L1_STORE, region, table, ents, flags)


SPANS = [(start, width) for width in (1, 2, 4, 8, 16) for start in range(0, 16, width)]


def store_cases():
    out = []
    # 16 single-byte writers from 16 different warps into one word (64 words: lanes of warps 0-15, then 16-31)
    out.append(_store("sixteen_warps_one_word", [{w * 32 + l: (l + 32 * (w // 16), w % 16, 1, 1)
                                                  for w in range(WARPS) for l in range(32)}], RESIDENT))
    # all 31 (start, width) spans, each at each of the 8 words of its own line
    out.append(_store("every_span_every_word", [{4 * (j * LINE + m): (j * LINE + m, s, wd, 1)
                                                 for j, (s, wd) in enumerate(SPANS) for m in range(LINE)}], RESIDENT))
    # four 8-byte writers, one per quarter of the CTA (different warps), fill each 32-byte sector
    out.append(_store("four_writers_one_sector", [{t: (2 * (t % 256) + (t // 256) // 2, 8 * (t // 256 % 2), 8,
                                                       1 + t // 256) for t in range(THREADS)}], RESIDENT))
    # three rounds: whole words, then their upper halves from another warp, then a 4-byte lane from a third
    out.append(_store("three_rounds_overwrite", [
        {t: (4 * t, 0, 16, 1) for t in range(THREADS)},
        {t: (4 * (t ^ 32), 8, 8, 2) for t in range(THREADS)},
        {t: (4 * (t ^ 64), 4 * (t % 4), 4, 3) for t in range(THREADS)},
    ], RESIDENT))
    # stores into lines nobody read: every width, one word per line
    out.append(_store("lines_never_read", [{t: (t * LINE + t % LINE, *_span(t), 1 + t % 3) for t in range(THREADS)}],
                      0))
    # each writer reads its own word back right after its store: halves from two warps, then 16 byte-writers per word,
    # then every width
    out.append(_store("read_own_store", [
        {t: (t % 512, 8 * (t // 512), 8, 1 + t // 512) for t in range(THREADS)},
        {t: (512 + t // 16, t % 16, 1, 3) for t in range(THREADS)},
        {t: (1024 + t, *_span(t), 4) for t in range(THREADS)},
    ], RESIDENT | READ_OWN))
    # every word of a line from a different warp
    out.append(_store("line_from_eight_warps", [{w * 32 + l: ((l + 32 * (w // 8)) * LINE + w % 8, 0, 16, 1)
                                                 for w in range(WARPS) for l in range(32)}], RESIDENT))
    return out


def _span(t):
    width = 1 << (t % 5)
    return (t * 7) % (16 // width) * width, width


def replay(case, ctas, seed, skip=None):
    """(ctas, region, 16) uint8: every CTA's region after the last round, replayed byte by byte from the fill;
    skip=(cta, round): that CTA stores nothing in that round"""
    region = case.region_words
    base = np.arange(ctas, dtype=np.uint64) * np.uint64(region)
    w = (base[:, None] + np.arange(region, dtype=np.uint64)[None, :]).ravel()
    mem = lo.pattern(w, lo.seed_key(seed)).view(np.uint8).reshape(ctas, region, 16).copy()
    for r, ents in enumerate(case.rounds):
        ents = ents[ents != 0]
        words, starts, widths, gens = unpack(ents)
        cs = np.array([c for c in range(ctas) if skip != (c, r)])
        for g in np.unique(gens):
            sel = gens == g
            ws = words[sel]
            vals = lo.pattern((base[:, None] + ws.astype(np.uint64)[None, :]).ravel(),
                              lo.seed_key(gen_seed(seed, int(g)))).view(np.uint8).reshape(ctas, len(ws), 16)
            for b in range(16):
                hit = (starts[sel] <= b) & (b < starts[sel] + widths[sel])
                mem[cs[:, None], ws[hit][None, :], b] = vals[cs][:, hit, b]
    return mem


def store_expected(case, ctas, seed, skip=None):
    """the uint32 expected words gsb_test_l1_table takes: [cta][region word][4]"""
    return replay(case, ctas, seed, skip).view(np.uint32).ravel()


# ---- texture --------------------------------------------------------------------------------------------------

def _tex(name, reads):
    """reads: (x, y) pairs, y = TEX_1D for a 1-D fetch of region word x; padded to whole steps by the caller"""
    assert len(reads) % THREADS == 0
    t = np.array([(x & 0xFFFFFFFF, y & 0xFFFFFFFF) for x, y in reads], dtype=np.uint64).astype(np.uint32)
    return Case(name, lo.TEX, lo.REGION, t.ravel())


def tex_cases():
    reads = [(x, y) for x in TEX_XS for y in TEX_YS]
    reads += [(x, y) for x in (-1, 0, lo.WIDTH - 1, lo.WIDTH) for y in range(lo.ROWS)]  # edge columns on every row
    reads += [(lo.REGION - 1 - i, TEX_1D) for i in range(THREADS - len(reads))]
    last = [(lo.REGION - 1, TEX_1D)] * (THREADS // 2) + [(lo.WIDTH - 1, lo.ROWS - 1), (lo.WIDTH, lo.ROWS)] * (THREADS // 4)
    return [_tex("far_and_edge_texels", reads), _tex("last_texels", last)]


def texel(x, y, rows, clamp):
    """buffer word a point read at texel (x, y) of the 64-wide array of `rows` rows returns; -1: reads as 0"""
    if not clamp and not (0 <= x < lo.WIDTH and 0 <= y < rows):
        return -1
    return min(max(y, 0), rows - 1) * lo.WIDTH + min(max(x, 0), lo.WIDTH - 1)


def tex_reads(case):
    t = case.table.astype(np.int64).reshape(-1, 2)
    return [(int(np.int32(x)), int(np.int32(y)) if y != TEX_1D else None) for x, y in t]


def tex_expected(case, ctas):
    """[cta][read][clamp, border] texel indices (a 1-D read: its word in both)"""
    rows = ctas * lo.ROWS
    out = np.empty((ctas, len(case.table) // 2, 2), dtype=np.int64)
    reads = tex_reads(case)
    for c in range(ctas):
        for r, (x, y) in enumerate(reads):
            if y is None:
                out[c, r] = c * lo.REGION + x
            else:
                out[c, r] = texel(x, c * lo.ROWS + y, rows, True), texel(x, c * lo.ROWS + y, rows, False)
    return out.ravel()


# ---- constant bank and parameter ------------------------------------------------------------------------------

def bank_cases(unit):
    words = CONST_WORDS if unit == lo.CONST else PARAM_WORDS
    out = []
    for d in (1, 2, 4, 8, 16, 32):
        k, w, lane = _warp_reads(4)
        idx = ((k * WARPS + w) * 131 + (lane % d) * 67) % words
        out.append(Case(f"distinct_{d}", unit, words, idx.astype(np.uint32).ravel()))
    out.append(Case("last_word_every_lane", unit, words, np.full(THREADS, words - 1, dtype=np.uint32)))
    return out


# ---- all of them ----------------------------------------------------------------------------------------------

def cases():
    return [*load_cases(lo.L1_LOAD), *load_cases(lo.NC), *store_cases(), *tex_cases(), *bank_cases(lo.CONST),
            *bank_cases(lo.PARAM)]


def case_id(c):
    return f"{lo.NAMES[c.unit]}-{c.name}"


def expected(case, ctas, seed, skip=None):
    """what gsb_test_l1_table takes as `expected` for this case, or None"""
    if case.unit == lo.L1_STORE:
        return store_expected(case, ctas, seed, skip)
    if case.unit == lo.TEX:
        return tex_expected(case, ctas)
    return None


def stores_per_round(case):
    return [int((r != 0).sum()) for r in case.rounds]


def words_per_cta(case):
    """16-byte words one CTA compares"""
    n = len(case.table)
    if case.unit == lo.L1_LOAD:
        return 3 * n
    if case.unit == lo.L1_STORE:
        return (case.region_words * (2 if case.flags & RESIDENT else 1)
                + (sum(stores_per_round(case)) if case.flags & READ_OWN else 0))
    if case.unit == lo.TEX:
        return sum(1 if y is None else 2 for _, y in tex_reads(case))
    return n


def stale_words(case, ctas, seed, cta, rnd):
    """words of CTA `cta` whose read-back differs when it skips round `rnd`"""
    full = replay(case, ctas, seed)[cta]
    skipped = replay(case, ctas, seed, skip=(cta, rnd))[cta]
    return int((full != skipped).any(axis=1).sum())
