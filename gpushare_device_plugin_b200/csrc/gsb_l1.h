/*
 * gsb_l1.h — the L1 and constant-cache check's schedule (gsb_l1_probe), shared by its sm_90a kernels
 * (l1_check_sm90a.cu) and the host (gsb_l1.cc, gsb_l1_schedule): which word each read of each thread returns, and the
 * bytes each L1_STORE thread writes. Every word is an HBM-probe pattern word of its own index (gsb_pattern.h), so
 * neither side keeps a table of expected words.
 */
#ifndef GSB_L1_H_
#define GSB_L1_H_

#include <stddef.h>
#include <stdint.h>

#include "../../include/gpushare_b200.h"
#include "gsb_pattern.h"

#define GSB_L1_LINE_WORDS 8u          /* a 128-byte line */
#define GSB_L1_REGION_LINES 1024u     /* GSB_L1_REGION_WORDS / GSB_L1_LINE_WORDS */
#define GSB_L1_TEX_X0 32              /* 2-D reads run x from -GSB_L1_TEX_X0 */
#define GSB_L1_TEX_XS 128             /* over this many columns */
#define GSB_L1_TEX_EDGE 8             /* rows the first (last) CTA's 2-D reads run before (past) the array */
#define GSB_L1_STORE_SALT 0x4C315354u

/* Generation 2 of L1_STORE: the pattern under the complement of the probe's seed. */
GSB_HD uint32_t gsb_l1_gen2_seed(uint32_t seed) { return ~seed; }

/* The region word that sequence position q (0..8191) of pass `pass` reads in L1_LOAD and NC. Pass 0 (cold) and every
 * fifth pass after it run in address order; then reversed; then line permutations of stride s = 32, 128 and 512 lines
 * (4, 16 and 64 KiB), which visit lines l0, l0 + s, l0 + 2 s, ... back to back: lines that share their low set-index
 * bits. */
GSB_HD uint32_t gsb_l1_order(uint32_t pass, uint32_t q) {
  const uint32_t kind = pass == 0 ? 0u : (pass - 1u) % 5u;
  if (kind == 0) return q;
  if (kind == 1) return GSB_L1_REGION_WORDS - 1u - q;
  const uint32_t s = kind == 2 ? 32u : kind == 3 ? 128u : 512u, groups = GSB_L1_REGION_LINES / s;
  const uint32_t p = q / GSB_L1_LINE_WORDS;
  return ((p % groups) * s + p / groups) * GSB_L1_LINE_WORDS + q % GSB_L1_LINE_WORDS;
}

/* The bytes [*lo, *lo + *width) of buffer word w that L1_STORE overwrites: width 1, 2, 4, 8 or 16, aligned. */
GSB_HD void gsb_l1_store_span(uint64_t w, uint32_t *lo, uint32_t *width) {
  const uint32_t h = gsb_mix32((uint32_t)w ^ (uint32_t)(w >> 32) * GSB_PAT_K1 ^ GSB_L1_STORE_SALT);
  *width = 1u << (h % 5u);
  *lo = ((h >> 8) % (16u / *width)) * *width;
}

/* The thread whose L1_STORE writes region word i: the one 512 threads away, so always another warp. */
GSB_HD uint32_t gsb_l1_store_writer(uint32_t i) { return (i % GSB_L1_THREADS) ^ 512u; }

/* What L1_STORE's read-back of buffer word w must return under `seed`: generation 2 over its stored bytes, generation 1
 * elsewhere. */
GSB_HD void gsb_l1_store_expected(uint64_t w, uint32_t seed, uint32_t out[4]) {
  uint32_t lo, width, g1[4], g2[4];
  gsb_l1_store_span(w, &lo, &width);
  gsb_pattern_word(w, gsb_seed_key(seed), g1);
  gsb_pattern_word(w, gsb_seed_key(gsb_l1_gen2_seed(seed)), g2);
  gsb_copy_merge(g2, g1, lo, lo + width, out);
}

/* TEX 2-D read i (0..GSB_L1_TEX_2D_READS) of CTA c of `ctas`: its unnormalized texel coordinates. */
GSB_HD void gsb_l1_tex_coord(uint32_t i, uint32_t c, uint32_t ctas, int32_t *x, int32_t *y) {
  const int32_t dy = c == 0 ? -GSB_L1_TEX_EDGE : c + 1 == ctas ? GSB_L1_TEX_EDGE : 0;
  *x = (int32_t)(i % GSB_L1_TEX_XS) - GSB_L1_TEX_X0;
  *y = (int32_t)(c * GSB_L1_TEX_ROWS + i / GSB_L1_TEX_XS) + dy;
}

/* The buffer word whose value a 2-D read at (x, y) returns on an array of `rows` rows: the nearest edge texel with
 * clamp addressing; with border addressing, -1 outside (the read returns 0). */
GSB_HD int64_t gsb_l1_texel(int32_t x, int32_t y, uint32_t rows, bool clamp) {
  const bool inside = x >= 0 && x < GSB_L1_TEX_WIDTH && y >= 0 && y < (int32_t)rows;
  if (!inside && !clamp) return -1;
  const int32_t xc = x < 0 ? 0 : x >= GSB_L1_TEX_WIDTH ? GSB_L1_TEX_WIDTH - 1 : x;
  const int32_t yc = y < 0 ? 0 : y >= (int32_t)rows ? (int32_t)rows - 1 : y;
  return (int64_t)yc * GSB_L1_TEX_WIDTH + xc;
}

/* Reads per thread of one pass of (unit, form): 0 when the unit has no such form. CONST and PARAM form 0 (uniform)
 * read every word per thread. */
GSB_HD uint32_t gsb_l1_steps(uint32_t unit, uint32_t form) {
  switch (unit) {
    case GSB_L1_UNIT_L1_LOAD: return form < 3 ? GSB_L1_STEPS : 0u;
    case GSB_L1_UNIT_L1_STORE: return form < 2 ? GSB_L1_STEPS : 0u;
    case GSB_L1_UNIT_NC: return form == 0 ? GSB_L1_STEPS : 0u;
    case GSB_L1_UNIT_TEX: return form == 0 ? GSB_L1_STEPS : form < 3 ? GSB_L1_TEX_2D_READS / GSB_L1_THREADS : 0u;
    case GSB_L1_UNIT_CONST:
      return form == 0 ? GSB_L1_CONST_WORDS : form == 1 ? GSB_L1_CONST_WORDS / GSB_L1_THREADS : 0u;
    case GSB_L1_UNIT_PARAM:
      return form == 0 ? GSB_L1_PARAM_WORDS : form == 1 ? (GSB_L1_PARAM_WORDS + GSB_L1_THREADS - 1) / GSB_L1_THREADS : 0u;
    default: return 0u;
  }
}

/* ---- gsb_test_l1_table: the twins' tables (see include/gpushare_b200.h) ---- */

/* The seed whose pattern generation g of an L1_STORE table stores; generation 0 is the probe's seed, the fill. */
GSB_HD uint32_t gsb_l1_table_seed(uint32_t seed, uint32_t g) { return seed ^ g * GSB_PAT_K0; }

/* The fields of one L1_STORE table entry (GSB_L1_STORE_ENTRY); width 0: no store. */
GSB_HD uint32_t gsb_l1_entry_word(uint32_t e) { return e & ((1u << GSB_L1_STORE_WORD_BITS) - 1u); }
GSB_HD uint32_t gsb_l1_entry_lo(uint32_t e) { return e >> GSB_L1_STORE_WORD_BITS & 15u; }
GSB_HD uint32_t gsb_l1_entry_width(uint32_t e) {
  const uint32_t c = e >> (GSB_L1_STORE_WORD_BITS + 4) & 7u;
  return c ? 1u << (c - 1u) : 0u;
}
GSB_HD uint32_t gsb_l1_entry_gen(uint32_t e) { return e >> 24; }

/* Words of each CTA's region a table of `unit` reads: set by the case for the buffer units, fixed otherwise. */
GSB_HD uint32_t gsb_l1_table_fixed_words(uint32_t unit) {
  return unit == GSB_L1_UNIT_TEX ? GSB_L1_REGION_WORDS
         : unit == GSB_L1_UNIT_CONST ? GSB_L1_CONST_WORDS
         : unit == GSB_L1_UNIT_PARAM ? GSB_L1_PARAM_WORDS
                                     : 0u;
}

/* uint32 expected entries per CTA a table of `unit` takes: L1_STORE 4 per region word, TEX 2 per read, none else. */
GSB_HD uint64_t gsb_l1_table_expected_per_cta(uint32_t unit, uint64_t n, uint32_t region_words) {
  return unit == GSB_L1_UNIT_L1_STORE ? 4ull * region_words : unit == GSB_L1_UNIT_TEX ? n : 0ull;
}

/* Host: whether gsb_test_l1_table takes this table (every refusal that needs no device; gsb_l1.cc). */
bool gsb_l1_table_valid(uint32_t unit, const uint32_t *table, size_t n, const uint32_t *expected, size_t n_expected,
                        uint32_t region_words);

/* Indices the corrupt hook accepts for `unit` (see gsb_test_l1_corrupt). */
GSB_HD uint32_t gsb_l1_hook_words(uint32_t unit) {
  switch (unit) {
    case GSB_L1_UNIT_TEX: return GSB_L1_REGION_WORDS + 2u * GSB_L1_TEX_2D_READS;
    case GSB_L1_UNIT_CONST: return GSB_L1_CONST_WORDS;
    case GSB_L1_UNIT_PARAM: return GSB_L1_PARAM_WORDS;
    default: return unit < GSB_L1_UNITS ? GSB_L1_REGION_WORDS : 0u;
  }
}

#endif /* GSB_L1_H_ */
