"""Independent restatement of the sparse tensor-core check's known answers (csrc/gsb_sparse_kat.h, csrc/gsb_sparse.cc)
in numpy: each unit's compressed operands and patterns, the dense A they stand for, the exact D (a dense GEMM of the
decompressed A) and the per-thread metadata registers. The hash and key are the SM check's oracle's; only the numbers
below are shared with the product, no code is."""
import numpy as np

from . import sm_oracle as so

F16_SP, BF16_SP, TF32_SP, E4M3_SP, E5M2_SP, S8_SP, HMMA_SP = range(7)
UNITS = range(7)
NAMES = ["f16", "bf16", "tf32", "e4m3", "e5m2", "s8", "hmma"]
M, N = 64, 128
KEY_BASE = 32
B_ROW, SA_ROW, SB_ROW, PATTERN_ROW = 0x1000, 0x2000, 0x2001, 0x3000
PAIRS = [(0, 1), (0, 2), (0, 3), (1, 2), (1, 3), (2, 3)]
# unit: (logical K, amp_a, amp_b, sa range, sb range, bound on the kept sum |A'||B'|, operand format)
SHAPES = {
    F16_SP: (512, 255, 127, (-10, 5), (-10, 5), 1 << 23, "f16"),
    BF16_SP: (512, 255, 127, (-40, 40), (-40, 40), 1 << 23, "bf16"),
    TF32_SP: (256, 1023, 63, (-40, 40), (-40, 40), 1 << 23, "tf32"),
    E4M3_SP: (128, 15, 3, (-6, 4), (-6, 6), 1 << 12, "e4m3"),
    E5M2_SP: (128, 7, 7, (-12, 12), (-12, 12), 1 << 12, "e5m2"),
    S8_SP: (512, 128, 128, (0, 0), (0, 0), 1 << 31, "s8"),
    HMMA_SP: (512, 255, 127, (-10, 5), (-10, 5), 1 << 23, "f16"),
}
EIGHT_BIT = (E4M3_SP, E5M2_SP, S8_SP)


def key(unit, seed):
    """HMMA_SP takes F16_SP's key: the same GEMM through mma.sp."""
    return so.key(KEY_BASE + (F16_SP if unit == HMMA_SP else unit), seed)


def group(unit):
    """logical K per group: 4 (two kept), TF32 2 (one kept)"""
    return 2 if unit == TF32_SP else 4


def n_patterns(unit):
    return 2 if unit == TF32_SP else 6


def step_k(unit):
    """logical K of one instruction"""
    return 16 if unit == TF32_SP else 64 if unit in EIGHT_BIT else 32


def _int(unit, h, amp):
    h = np.asarray(h, dtype=np.int64)
    if unit == S8_SP:
        return ((h & 0xFF) ^ 0x80) - 0x80
    return h % (2 * amp + 1) - amp


def operands(unit, seed):
    """(A' 64 x K/2 compressed, patterns 64 x groups, B' K x 128, sa[64], sb[128]) as int64"""
    K, amp_a, amp_b, (a0, a1), (b0, b1) = SHAPES[unit][:5]
    k = key(unit, seed)
    i, c = np.meshgrid(np.arange(M), np.arange(K // 2), indexing="ij")
    A = _int(unit, so.hash_(k, i, c), amp_a)
    i, q = np.meshgrid(np.arange(M), np.arange(K // group(unit)), indexing="ij")
    P = so.hash_(k, PATTERN_ROW + i, q).astype(np.int64) % n_patterns(unit)
    kk, j = np.meshgrid(np.arange(K), np.arange(N), indexing="ij")
    B = _int(unit, so.hash_(k, B_ROW + kk, j), amp_b)
    if unit == S8_SP:
        return A, P, B, np.zeros(M, np.int64), np.zeros(N, np.int64)
    sa = a0 + so.hash_(k, SA_ROW, np.arange(M)).astype(np.int64) % (a1 - a0 + 1)
    sb = b0 + so.hash_(k, SB_ROW, np.arange(N)).astype(np.int64) % (b1 - b0 + 1)
    return A, P, B, sa, sb


def decompress(unit, A, P):
    """The dense 64 x K A' the compressed A' and its patterns stand for (zeros where nothing is kept)."""
    A, P = np.asarray(A, dtype=np.int64), np.asarray(P, dtype=np.int64)
    K = SHAPES[unit][0]
    dense = np.zeros((M, K), np.int64)
    rows = np.arange(M)[:, None]
    if unit == TF32_SP:
        q = np.arange(K // 2)[None, :]
        dense[rows, 2 * q + P] = A
        return dense
    lo = np.array([p[0] for p in PAIRS])[P]
    hi = np.array([p[1] for p in PAIRS])[P]
    q = np.arange(K // 4)[None, :]
    dense[rows, 4 * q + lo] = A[:, 0::2]
    dense[rows, 4 * q + hi] = A[:, 1::2]
    return dense


def gemm_from(unit, A, P, B, sa, sb):
    """The 8192 words of D, row-major, as Python ints (FP32 bits, S8_SP's S32 two's complement): a dense GEMM of the
    decompressed A, its kept sum |A'||B'| asserted under the unit's bound, then scaled and asserted exact in FP32."""
    Ad, B = decompress(unit, A, P), np.asarray(B, dtype=np.int64)
    sa, sb = np.asarray(sa, dtype=np.int64), np.asarray(sb, dtype=np.int64)
    mx = int((np.abs(Ad) @ np.abs(B)).max())
    assert mx < SHAPES[unit][5], (unit, mx)
    D = Ad @ B
    if unit == S8_SP:
        return [int(x) & 0xFFFFFFFF for x in D.reshape(-1)]
    scaled = np.ldexp(D.astype(np.float64), sa[:, None] + sb[None, :])
    f = scaled.astype(np.float32)
    assert np.array_equal(f.astype(np.float64), scaled)
    nz = np.abs(scaled[scaled != 0])
    assert nz.size == 0 or nz.min() >= 2.0 ** -126, unit  # every nonzero D a normal FP32
    return [int(x) for x in f.view(np.uint32).reshape(-1)]


def expected(unit, seed):
    return gemm_from(unit, *operands(unit, seed))


def bound(unit, seed):
    A, P, B, _, _ = operands(unit, seed)
    return int((np.abs(decompress(unit, A, P)) @ np.abs(B)).max()), SHAPES[unit][5]


def code(unit, p):
    """the 4-bit metadata of a group: (i0, i1) as i0 | i1 << 2; TF32 keeps element p as the pair (2p, 2p + 1)"""
    i0, i1 = (2 * p, 2 * p + 1) if unit == TF32_SP else PAIRS[p]
    return i0 | i1 << 2


def meta(unit, P, warp, lane, step):
    """The metadata register lane `lane` of warp `warp` passes at K step `step`, read off the PTX ISA's sparse layout:
    rows of the warp are 16 warp + g and + 8, g = lane / 4. 16-bit and TF32 forms take 8 groups per step; the thread
    pair (lane mod 4) / 2 that the selector names supplies them, its first thread groups 0-3 and its second 4-7, each
    row g in the low half and row g + 8 in the high half; the kernel alternates the selector, so a register carries
    the step of its own pair. 8-bit forms take 16 groups per step, selector 0: thread t of the quad holds 8 groups of
    one row, t even row g, t odd row g + 8, t < 2 the first 8 groups."""
    g, t = lane // 4, lane % 4
    r0 = 16 * warp + g
    word = 0
    if unit in EIGHT_BIT:
        row = r0 + 8 * (t & 1)
        for n in range(8):
            word |= code(unit, int(P[row][16 * step + 8 * (t >> 1) + n])) << (4 * n)
        return word
    carried = step - step % 2 + t // 2
    for half in range(2):
        for n in range(4):
            word |= code(unit, int(P[r0 + 8 * half][8 * carried + 4 * (t % 2) + n])) << (4 * (4 * half + n))
    return word
