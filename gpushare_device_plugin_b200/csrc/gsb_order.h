/*
 * gsb_order.h — the memory-ordering check's words, pairing and outcome classes (gsb_order_probe), shared by its sm_90a
 * kernel (order_check_sm90a.cu) and the host (gsb_order.cc, which exports them for the tests). Every shared location
 * is one u64: the iteration in the high half, gsb_mix32(seed ^ key ^ iteration) in the low half.
 */
#ifndef GSB_ORDER_H_
#define GSB_ORDER_H_

#include <stdint.h>

#include "../../include/gpushare_b200.h"
#include "gsb_pattern.h"

#define GSB_ORDER_SLOTS 5                /* locations per CTA: MP's flag (slot 0, also x of the other units), 4 data */
#define GSB_ORDER_LOC_WORDS 2048u        /* u64 words of a CTA's location block (16 KiB) */
#define GSB_ORDER_SCRATCH_WORDS 4096u    /* 16-byte words of a CTA's stress region (64 KiB) */
#define GSB_ORDER_OBS_WORDS 4u           /* u64 words a CTA publishes per SB and IRIW observation */
#define GSB_ORDER_KEY_SALT 0x4F524452u
#if defined(__CUDA_ARCH__)
#define GSB_ORDER_UNROLL _Pragma("unroll")
#else
#define GSB_ORDER_UNROLL
#endif

/* The second grid barrier's bound for `observations` per CTA: GSB_ORDER_WAIT_NS, plus GSB_ORDER_WAIT_NS_PER_OBS per
 * observation for how far the slowest CTA's litmus loop may trail the fastest's. */
GSB_HD uint64_t gsb_order_wait_ns(uint32_t observations) {
  return GSB_ORDER_WAIT_NS + (uint64_t)observations * GSB_ORDER_WAIT_NS_PER_OBS;
}

/* The u64 index of slot s in a CTA's location block: 2 KiB + 128 B apart, so every slot has a line of its own at a
 * different offset within 4 KiB. */
GSB_HD uint32_t gsb_order_slot_word(uint32_t s) { return s * 272u; }

/* The key of slot s of CTA rank r. */
GSB_HD uint32_t gsb_order_key(uint32_t r, uint32_t s) { return gsb_mix32((r << 3 | s) ^ GSB_ORDER_KEY_SALT); }

/* The word iteration i stores at a location of `key` under `seed`. */
GSB_HD uint64_t gsb_order_word(uint32_t seed, uint32_t key, uint32_t i) {
  return (uint64_t)i << 32 | gsb_mix32(seed ^ key ^ i);
}

/* Bits of w's low half that differ from the hash of its high half (0: a word some iteration stored). */
GSB_HD uint32_t gsb_order_bad_bits(uint32_t seed, uint32_t key, uint64_t w) {
  uint32_t x = (uint32_t)w ^ gsb_mix32(seed ^ key ^ (uint32_t)(w >> 32)), c = 0;
  for (; x; x &= x - 1u) c++;
  return c;
}

/* Words of one observation as gsb_order_classify takes them. */
GSB_HD uint32_t gsb_order_obs_words(uint32_t unit) {
  switch (unit) {
    case GSB_ORDER_UNIT_MP_RELACQ:
    case GSB_ORDER_UNIT_MP_FENCE:
    case GSB_ORDER_UNIT_MP_RELAXED: return 5u;
    case GSB_ORDER_UNIT_SB_SC: return 2u;
    case GSB_ORDER_UNIT_IRIW_SC: return 4u;
    case GSB_ORDER_UNIT_CORR: return 3u;
    default: return 0u;
  }
}

/* Words a CTA reads per observation, and once more after the final barrier (both checked). */
GSB_HD uint32_t gsb_order_reads(uint32_t unit) {
  return unit == GSB_ORDER_UNIT_SB_SC ? 2u : unit == GSB_ORDER_UNIT_CORR ? 2u : gsb_order_obs_words(unit);
}
GSB_HD uint32_t gsb_order_final_reads(uint32_t unit) {
  return unit == GSB_ORDER_UNIT_IRIW_SC ? 2u : unit <= GSB_ORDER_UNIT_MP_FENCE || unit == GSB_ORDER_UNIT_MP_RELAXED ? 5u
                                                                                                                 : 1u;
}

GSB_HD uint32_t gsb_order_distance_of(uint32_t k, uint32_t n, uint32_t seed) {
  if (n < 2) return 0u;
  switch (k) {
    case 0: return 1u;
    case 1: return n / 2u;
    case 2: return 1u + seed % (n - 1u);
    default: return 0u;
  }
}

GSB_HD uint32_t gsb_order_iriw_step(uint32_t n, uint32_t d) {
  if (n < 4) return 0u;
  uint32_t e = d % n ? d % n : 1u;
  for (uint32_t t = 0; t < n; t++) {
    if (e % n && 2u * e % n && 3u * e % n) return e;
    e = e + 1u == n ? 1u : e + 1u;
  }
  return 0u;
}

GSB_HD int gsb_order_pairing_of(uint32_t unit, uint32_t n, uint32_t d, uint32_t r, uint32_t ranks[3]) {
  if (unit >= GSB_ORDER_UNITS || n < 2 || d == 0 || d >= n || r >= n) return 0;
  if (unit == GSB_ORDER_UNIT_SB_SC) {
    ranks[0] = (r + d) % n;
    ranks[1] = (r + n - d) % n;
    return 2;
  }
  if (unit == GSB_ORDER_UNIT_IRIW_SC) {
    const uint32_t e = gsb_order_iriw_step(n, d);
    if (!e) return 0;
    ranks[0] = (r + 3u * n - 2u * e) % n;  // x: the instance's first writer
    ranks[1] = (r + 3u * n - e) % n;       // y: its second writer
    ranks[2] = (r + e) % n;                // its other reader
    return 3;
  }
  ranks[0] = (r + d) % n;
  return 1;
}

GSB_HD uint32_t gsb_order_classify_words(uint32_t unit, uint32_t seed, const uint32_t *keys, const uint64_t *words,
                                         uint32_t iteration) {
  const uint32_t nw = gsb_order_obs_words(unit);
  if (!nw) return GSB_ORDER_CLS_CORRUPT;
  uint32_t it[GSB_ORDER_WORDS] = {0, 0, 0, 0, 0};
GSB_ORDER_UNROLL
  for (uint32_t j = 0; j < GSB_ORDER_WORDS; j++) {
    if (j < nw && gsb_order_bad_bits(seed, keys[j], words[j])) return GSB_ORDER_CLS_CORRUPT;
    it[j] = j < nw ? (uint32_t)(words[j] >> 32) : 0u;
  }
  switch (unit) {
    case GSB_ORDER_UNIT_SB_SC: {
      const uint32_t a = it[0], b = it[1], i = iteration;
      if ((a < i && b < i) || (a > i && b > i)) return GSB_ORDER_CLS_FORBIDDEN;
      return a == i || b == i ? GSB_ORDER_CLS_OVERLAP : GSB_ORDER_CLS_ALLOWED;
    }
    case GSB_ORDER_UNIT_IRIW_SC:
      if (it[0] > it[3] && it[2] > it[1]) return GSB_ORDER_CLS_FORBIDDEN;
      return it[0] != it[3] || it[1] != it[2] ? GSB_ORDER_CLS_OVERLAP : GSB_ORDER_CLS_ALLOWED;
    case GSB_ORDER_UNIT_CORR:
      if (it[1] < it[0] || it[2] < it[1]) return GSB_ORDER_CLS_FORBIDDEN;
      return it[2] > it[1] ? GSB_ORDER_CLS_OVERLAP : GSB_ORDER_CLS_ALLOWED;
    default: {  // MP: the flag, then 4 data
      uint32_t lo = it[1], hi = it[1];
GSB_ORDER_UNROLL
      for (uint32_t j = 2; j < 5; j++) {
        lo = it[j] < lo ? it[j] : lo;
        hi = it[j] > hi ? it[j] : hi;
      }
      if (lo < it[0]) return unit == GSB_ORDER_UNIT_MP_RELAXED ? GSB_ORDER_CLS_WEAK : GSB_ORDER_CLS_FORBIDDEN;
      return hi > it[0] ? GSB_ORDER_CLS_OVERLAP : GSB_ORDER_CLS_ALLOWED;
    }
  }
}

/* A final read after the grid barrier of a location whose writer stored iterations 1..m. */
GSB_HD uint32_t gsb_order_final(uint32_t seed, uint32_t key, uint64_t w, uint32_t m) {
  if (gsb_order_bad_bits(seed, key, w) || (uint32_t)(w >> 32) > m) return GSB_ORDER_CLS_CORRUPT;
  return (uint32_t)(w >> 32) < m ? GSB_ORDER_CLS_LOST : GSB_ORDER_CLS_ALLOWED;
}

/* The inject hook's observation: words with valid hashes that `unit` forbids in `iteration` (1..). */
GSB_HD void gsb_order_forbidden_words(uint32_t unit, uint32_t seed, const uint32_t *keys, uint32_t iteration,
                                      uint64_t *words) {
  switch (unit) {
    case GSB_ORDER_UNIT_SB_SC:
      words[0] = gsb_order_word(seed, keys[0], iteration - 1u);
      words[1] = gsb_order_word(seed, keys[1], iteration - 1u);
      break;
    case GSB_ORDER_UNIT_IRIW_SC:  // a > d, c > b
      words[0] = gsb_order_word(seed, keys[0], 1u);
      words[1] = gsb_order_word(seed, keys[1], 0u);
      words[2] = gsb_order_word(seed, keys[2], 1u);
      words[3] = gsb_order_word(seed, keys[3], 0u);
      break;
    case GSB_ORDER_UNIT_CORR:  // a read older than the one before it
      words[0] = gsb_order_word(seed, keys[0], 1u);
      words[1] = gsb_order_word(seed, keys[1], 0u);
      words[2] = gsb_order_word(seed, keys[2], 0u);
      break;
    default:  // MP: flag 1, data 0 below it
      words[0] = gsb_order_word(seed, keys[0], 1u);
GSB_ORDER_UNROLL
      for (uint32_t j = 1; j < 5; j++) words[j] = gsb_order_word(seed, keys[j], j == 1 ? 0u : 1u);
      break;
  }
}

#endif /* GSB_ORDER_H_ */
