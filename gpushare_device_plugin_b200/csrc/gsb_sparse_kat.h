/*
 * gsb_sparse_kat.h — the sparse tensor-core check's known answers (gsb_sparse_probe), shared by its sm_90a kernels
 * (sparse_check_sm90a.cu, sparse_operands_sm90a.cu) and the host side that computes what they must produce
 * (gsb_sparse.cc). Restated independently in tests/helpers/sparse_oracle.py.
 *
 * A is 64 x K (K the logical K) with two of every four K kept (TF32: one of every two). What the instruction takes is
 * the compressed A', 64 x K/2, and a 2-bit index per kept value. Group q of row i keeps the index pair
 * pattern(i, q) = hash(key, 0x3000 + i, q) mod 6 of the six increasing pairs (TF32: mod 2, the element kept), and its
 * stored values are A'[i][2q] (the lower index) and A'[i][2q + 1] (TF32: A'[i][q]). A'[i][c] = int(hash(key, i, c)) *
 * 2^sa_i, B[k][j] = int(hash(key, 0x1000 + k, j)) * 2^sb_j, the scales from hash(key, 0x2000, i) and
 * hash(key, 0x2001, j): every row tag clear of the others. Each unit has its own key, except HMMA_SP: it takes
 * F16_SP's, so the same logical sparse GEMM is issued through mma.sp and through wgmma.sp.
 *
 * Each shape keeps the sum over kept terms of |A'| |B'| under its accumulator's bound, at which every partial sum is
 * exact whatever order the hardware adds the terms in: 2^23 for FP32 accumulators, 2^12 for FP8 inputs (the width
 * measured for dense FP8 wgmma; DESIGN.md §3). S8 sums stay far inside int32.
 *
 * Metadata. A group's 4-bit code is i0 | i1 << 2 for its pair (i0 < i1); TF32 keeps element e as 0x4 (e = 0) or 0xE
 * (e = 1). Per warp w (rows 16w..16w+15) and lane l, g = l / 4, t = l % 4, the register of one instruction's K step:
 *   16-bit and TF32 forms (8 groups per step): the thread pair t / 2 = selector supplies the step's metadata; thread t
 *     holds groups 4 (t mod 2) .. + 3 of row g in nibbles 0-3 and of row g + 8 in nibbles 4-7. The shipped kernels
 *     alternate the selector over K steps, so step s is read from pair s mod 2 and each register carries step
 *     (s & ~1) + t / 2: a selector routed to the wrong pair reads the other step's groups.
 *   8-bit forms (16 groups per step, selector 0): thread t holds groups 8 (t / 2) .. + 7 of row g + 8 (t mod 2).
 * mma.sp m16n8k32 (HMMA_SP) takes the same per-warp layout as the 16-bit wgmma.sp.
 */
#ifndef GSB_SPARSE_KAT_H_
#define GSB_SPARSE_KAT_H_

#include <stdint.h>

#include "gsb_sm_kat.h"
#include "gsb_tensor_kat.h"

#define GSB_SPARSE_KEY_BASE 32u  /* gsb_sm_key unit of sparse unit u: 32 + u, clear of the SM (0-7) and tensor (16-23) keys */
#define GSB_SPARSE_B_ROW 0x1000u
#define GSB_SPARSE_SA_ROW 0x2000u
#define GSB_SPARSE_SB_ROW 0x2001u
#define GSB_SPARSE_PATTERN_ROW 0x3000u
#define GSB_SPARSE_PAIRS 6

GSB_HD int gsb_sparse_is_tf32(uint32_t unit) { return unit == GSB_SPARSE_UNIT_TF32_SP; }
GSB_HD int gsb_sparse_is_8bit(uint32_t unit) {
  return unit == GSB_SPARSE_UNIT_E4M3_SP || unit == GSB_SPARSE_UNIT_E5M2_SP || unit == GSB_SPARSE_UNIT_S8_SP;
}

/* K (logical), amplitudes and scale ranges: each unit takes the dense check's values for its type */
GSB_HD gsb_sm_tensor_shape gsb_sparse_shape(uint32_t unit) {
  gsb_sm_tensor_shape s = {0, 0, 0, 0, 0, 0, 0};
  switch (unit) {
    case GSB_SPARSE_UNIT_F16_SP:
    case GSB_SPARSE_UNIT_HMMA_SP: s = gsb_sm_shape(GSB_SM_UNIT_F16); s.k = 512; break;
    case GSB_SPARSE_UNIT_BF16_SP: s = gsb_sm_shape(GSB_SM_UNIT_BF16); s.k = 512; break;
    case GSB_SPARSE_UNIT_TF32_SP: s = gsb_tensor_shape(GSB_TENSOR_UNIT_TF32); s.k = 256; break;
    case GSB_SPARSE_UNIT_E4M3_SP: s = gsb_sm_shape(GSB_SM_UNIT_E4M3); s.k = 128; break;
    case GSB_SPARSE_UNIT_E5M2_SP: s = gsb_tensor_shape(GSB_TENSOR_UNIT_E5M2); s.k = 128; break;
    case GSB_SPARSE_UNIT_S8_SP: s = gsb_sm_shape(GSB_SM_UNIT_S8); s.k = 512; break;
    default: break;
  }
  return s;
}

GSB_HD uint32_t gsb_sparse_key(uint32_t unit, uint32_t seed) {
  return gsb_sm_key(GSB_SPARSE_KEY_BASE + (unit == GSB_SPARSE_UNIT_HMMA_SP ? (uint32_t)GSB_SPARSE_UNIT_F16_SP : unit),
                    seed);
}

/* Logical K per group (4, TF32 2), groups per row, and logical K of one instruction */
GSB_HD uint32_t gsb_sparse_group_k(uint32_t unit) { return gsb_sparse_is_tf32(unit) ? 2u : 4u; }
GSB_HD uint32_t gsb_sparse_groups(uint32_t unit) { return gsb_sparse_shape(unit).k / gsb_sparse_group_k(unit); }
GSB_HD uint32_t gsb_sparse_step_k(uint32_t unit) {
  return gsb_sparse_is_tf32(unit) ? 16u : gsb_sparse_is_8bit(unit) ? 64u : 32u;
}
/* The count of valid patterns: 6 index pairs, TF32 2 kept elements */
GSB_HD uint32_t gsb_sparse_patterns(uint32_t unit) { return gsb_sparse_is_tf32(unit) ? 2u : (uint32_t)GSB_SPARSE_PAIRS; }

GSB_HD int32_t gsb_sparse_int(uint32_t unit, uint32_t h, int32_t amp) {
  if (unit == GSB_SPARSE_UNIT_S8_SP) return gsb_sm_int(GSB_SM_UNIT_S8, h, amp);
  return gsb_tensor_int(h, amp);
}
/* compressed A'[i][c], c < K / 2 */
GSB_HD int32_t gsb_sparse_a(uint32_t unit, uint32_t key, uint32_t i, uint32_t c) {
  return gsb_sparse_int(unit, gsb_sm_hash(key, i, c), gsb_sparse_shape(unit).amp_a);
}
GSB_HD int32_t gsb_sparse_b(uint32_t unit, uint32_t key, uint32_t k, uint32_t j) {
  return gsb_sparse_int(unit, gsb_sm_hash(key, GSB_SPARSE_B_ROW + k, j), gsb_sparse_shape(unit).amp_b);
}
GSB_HD int32_t gsb_sparse_sa(uint32_t unit, uint32_t key, uint32_t i) {
  const gsb_sm_tensor_shape s = gsb_sparse_shape(unit);
  return unit == GSB_SPARSE_UNIT_S8_SP ? 0 : gsb_sm_scale(gsb_sm_hash(key, GSB_SPARSE_SA_ROW, i), s.sa_min, s.sa_max);
}
GSB_HD int32_t gsb_sparse_sb(uint32_t unit, uint32_t key, uint32_t j) {
  const gsb_sm_tensor_shape s = gsb_sparse_shape(unit);
  return unit == GSB_SPARSE_UNIT_S8_SP ? 0 : gsb_sm_scale(gsb_sm_hash(key, GSB_SPARSE_SB_ROW, j), s.sb_min, s.sb_max);
}
/* the pattern of group q of row i: 0-5 an index pair, TF32 0-1 the element kept */
GSB_HD uint32_t gsb_sparse_pattern(uint32_t unit, uint32_t key, uint32_t i, uint32_t q) {
  return gsb_sm_hash(key, GSB_SPARSE_PATTERN_ROW + i, q) % gsb_sparse_patterns(unit);
}

/* The logical K within its group of stored value `slot` (0 or 1; TF32 0 only) of a group with `pattern` */
GSB_HD uint32_t gsb_sparse_index(uint32_t unit, uint32_t pattern, uint32_t slot) {
  if (gsb_sparse_is_tf32(unit)) return pattern;
  /* (0,1) (0,2) (0,3) (1,2) (1,3) (2,3) */
  const uint32_t lo = pattern < 3 ? 0u : pattern < 5 ? 1u : 2u;
  const uint32_t hi = pattern < 3 ? pattern + 1 : pattern < 5 ? pattern - 1 : 3u;
  return slot ? hi : lo;
}
/* The 4-bit metadata code of a group */
GSB_HD uint32_t gsb_sparse_code(uint32_t unit, uint32_t pattern) {
  if (gsb_sparse_is_tf32(unit)) return pattern ? 0xEu : 0x4u;
  return gsb_sparse_index(unit, pattern, 0) | gsb_sparse_index(unit, pattern, 1) << 2;
}

/* Which (row within the warp's 16, group) nibble n of lane l's metadata register holds at K step `step` */
GSB_HD void gsb_sparse_slot(uint32_t unit, uint32_t l, uint32_t step, uint32_t n, uint32_t *row, uint32_t *q) {
  const uint32_t g = l / 4, t = l % 4;
  if (gsb_sparse_is_8bit(unit)) {
    *row = g + 8 * (t % 2);
    *q = 16 * step + 8 * (t / 2) + n;
  } else {
    const uint32_t carried = (step & ~1u) + t / 2;  // the step this register carries (selector = step mod 2)
    *row = g + 8 * (n / 4);
    *q = 8 * carried + 4 * (t % 2) + n % 4;
  }
}

/* The metadata register of lane l of warp w at K step `step`, from the seed's patterns */
GSB_HD uint32_t gsb_sparse_meta(uint32_t unit, uint32_t key, uint32_t w, uint32_t l, uint32_t step) {
  uint32_t m = 0;
  for (uint32_t n = 0; n < 8; n++) {
    uint32_t row, q;
    gsb_sparse_slot(unit, l, step, n, &row, &q);
    m |= gsb_sparse_code(unit, gsb_sparse_pattern(unit, key, 16 * w + row, q)) << (4 * n);
  }
  return m;
}

/* The test-only operand table (gsb_test_sparse_operands) after the 8192 expected words, as int32: A' (64 x K/2), the
 * patterns (64 x groups), B (K x 128), sa (64), sb (128) */
GSB_HD uint32_t gsb_sparse_table_a(uint32_t unit, uint32_t i, uint32_t c) { return i * (gsb_sparse_shape(unit).k / 2) + c; }
GSB_HD uint32_t gsb_sparse_table_p(uint32_t unit, uint32_t i, uint32_t q) {
  return GSB_SM_M * (gsb_sparse_shape(unit).k / 2) + i * gsb_sparse_groups(unit) + q;
}
GSB_HD uint32_t gsb_sparse_table_b(uint32_t unit, uint32_t k, uint32_t j) {
  return GSB_SM_M * (gsb_sparse_shape(unit).k / 2 + gsb_sparse_groups(unit)) + k * GSB_SM_N + j;
}
GSB_HD uint32_t gsb_sparse_table_sa(uint32_t unit, uint32_t i) { return gsb_sparse_table_b(unit, gsb_sparse_shape(unit).k, 0) + i; }
GSB_HD uint32_t gsb_sparse_table_sb(uint32_t unit, uint32_t j) {
  return gsb_sparse_table_b(unit, gsb_sparse_shape(unit).k, 0) + GSB_SM_M + j;
}
GSB_HD uint32_t gsb_sparse_table_words(uint32_t unit) { return gsb_sparse_table_sb(unit, GSB_SM_N); }

#endif /* GSB_SPARSE_KAT_H_ */
