/*
 * gsb_shared_atomic.h — the shared-memory atomic check's geometry and the value of every contribution, shared by its
 * sm_90a kernels (shared_atomic_check_sm90a.cu), the host half of the probe (gsb_device.cu, gsb_shared_atomic.cc) and,
 * compiled as C, the tests' host build.
 *
 * A CTA's area is GSB_SHARED_ATOMIC_AREA_BYTES of its shared memory: the spread region, then GSB_SHARED_ATOMIC_HOT_WORDS
 * hot slots GSB_SHARED_ATOMIC_HOT_STRIDE bytes apart, all in one bank. It is built in "units" of the unit's word size
 * (gsb_shared_atomic_unit_bytes); a word's form (its "kind") follows its logical index: the unit in the spread region,
 * the slot's number in the hot area. The hash, the float integers and their encoders are the L2 atomic check's
 * (gsb_atomic.h).
 *
 * Every value is a function of (unit, seed, phase, thread, round or repetition), never of %smid or blockIdx, so every
 * CTA's area ends the same and one expected area serves them all.
 */
#ifndef GSB_SHARED_ATOMIC_H_
#define GSB_SHARED_ATOMIC_H_

#include <stdint.h>

#include "gsb_atomic.h"

#define GSB_SHARED_ATOMIC_WARPS (GSB_SHARED_ATOMIC_THREADS / 32)
#define GSB_SHARED_ATOMIC_TAG 0x00400000u   /* keys of this check differ from every key of the L2 check */
#define GSB_SHARED_ATOMIC_BOUND_TAG 0x00200000u /* inc / dec: a word's bound */
#define GSB_SHARED_ATOMIC_EXCH_TAG 0x00100000u  /* TICKET: an exchanged value */
#define GSB_SHARED_ATOMIC_PAIR_TAG 0x00080000u  /* CAS: the upper half of a b128 pair */
/* contributions to each hot word of one CTA: its ids are 0 .. count - 1 */
#define GSB_SHARED_ATOMIC_COUNT (GSB_SHARED_ATOMIC_WARPS * GSB_SHARED_ATOMIC_HOT_REPS)
/* TICKET and CAS slots: per CTA, form and hot slot, COUNT entries and one for the final exchange word; 4 words each */
#define GSB_SHARED_ATOMIC_FORMS 4u
#define GSB_SHARED_ATOMIC_ENTRIES (GSB_SHARED_ATOMIC_COUNT + 1u)
#define GSB_SHARED_ATOMIC_SLOT_WORDS (GSB_SHARED_ATOMIC_FORMS * GSB_SHARED_ATOMIC_HOT_WORDS * GSB_SHARED_ATOMIC_ENTRIES * 4u)

/* TICKET's hot slot: the add.u32 counter, then the b32, b64 and b128 exchange words; CAS's: the b32, b64 and b128
 * counters. Byte offsets within the slot. */
#define GSB_SHARED_ATOMIC_TICKET_EXCH32 16u
#define GSB_SHARED_ATOMIC_TICKET_EXCH64 32u
#define GSB_SHARED_ATOMIC_TICKET_EXCH128 48u
#define GSB_SHARED_ATOMIC_CAS64 8u
#define GSB_SHARED_ATOMIC_CAS128 16u

GSB_HD uint32_t gsb_shared_atomic_unit_bytes(uint32_t unit) {
  return unit == GSB_SHARED_ATOMIC_UNIT_WIDE || unit == GSB_SHARED_ATOMIC_UNIT_FLOAT ? 8u : 4u;
}

GSB_HD uint32_t gsb_shared_atomic_units(uint32_t unit) {
  return GSB_SHARED_ATOMIC_AREA_BYTES / gsb_shared_atomic_unit_bytes(unit);
}

/* TICKET and CAS only run the hot phase */
GSB_HD int gsb_shared_atomic_has_spread(uint32_t unit) {
  return unit != GSB_SHARED_ATOMIC_UNIT_TICKET && unit != GSB_SHARED_ATOMIC_UNIT_CAS;
}

/* spread rounds: even ones reach every word once (256 units each), odd ones as many */
GSB_HD uint32_t gsb_shared_atomic_rounds(uint32_t unit) {
  return 2u * (GSB_SHARED_ATOMIC_SPREAD_BYTES / gsb_shared_atomic_unit_bytes(unit) / GSB_SHARED_ATOMIC_THREADS);
}

/* The unit thread t hits in spread round r. Even round 2k: unit k x 256 + warp x 32 + (lane + 4k + warp) mod 32, so
 * the 32 lanes of a warp hit 32 consecutive words and each lane's bank turns with k and warp. Odd round 2k + 1: unit
 * (t x 32 + k) mod n, so the lanes of a warp hit 32 words of one bank at different addresses. */
GSB_HD uint32_t gsb_shared_atomic_spread_unit(uint32_t unit, uint32_t t, uint32_t r) {
  const uint32_t n = GSB_SHARED_ATOMIC_SPREAD_BYTES / gsb_shared_atomic_unit_bytes(unit), k = r >> 1;
  const uint32_t warp = t >> 5, lane = t & 31u;
  if (r & 1u) return (t * 32u + k) % n;
  return k * GSB_SHARED_ATOMIC_THREADS + warp * 32u + (lane + 4u * k + warp) % 32u;
}

/* the unit of hot slot l's first word */
GSB_HD uint32_t gsb_shared_atomic_hot_unit(uint32_t unit, uint32_t l) {
  return (GSB_SHARED_ATOMIC_SPREAD_BYTES + l * GSB_SHARED_ATOMIC_HOT_STRIDE) / gsb_shared_atomic_unit_bytes(unit);
}

GSB_HD int gsb_shared_atomic_is_hot(uint32_t unit, uint32_t u) {
  return u * gsb_shared_atomic_unit_bytes(unit) >= GSB_SHARED_ATOMIC_SPREAD_BYTES;
}

/* INT32: 0 add.u32, 1 and.b32, 2 or.b32, 3 xor.b32, 4 min.s32, 5 max.s32, 6 min.u32, 7 max.u32, 8 inc.u32, 9 dec.u32;
 * WIDE: 0 add.u64, 1 and.b64, 2 or.b64, 3 xor.b64, 4 min.s64, 5 max.u64; FLOAT: 0 f32, 1 f64, 2 f16x2, 3 bf16x2; else
 * 0. By logical index: the unit, or the hot slot it lies in. */
GSB_HD uint32_t gsb_shared_atomic_kind(uint32_t unit, uint32_t u) {
  const uint32_t ub = gsb_shared_atomic_unit_bytes(unit);
  const uint32_t x = gsb_shared_atomic_is_hot(unit, u)
                         ? (u * ub - GSB_SHARED_ATOMIC_SPREAD_BYTES) / GSB_SHARED_ATOMIC_HOT_STRIDE
                         : u;
  return unit == GSB_SHARED_ATOMIC_UNIT_INT32 ? x % 10u
         : unit == GSB_SHARED_ATOMIC_UNIT_WIDE ? x % 6u
         : unit == GSB_SHARED_ATOMIC_UNIT_FLOAT ? x % 4u
                                                : 0u;
}

/* the hash of a contribution: thread t in `phase` (GSB_ATOMIC_PHASE_SPREAD / _HOT), round or repetition r */
GSB_HD uint64_t gsb_shared_atomic_key(uint32_t unit, uint32_t seed, uint32_t phase, uint32_t t, uint32_t r) {
  return gsb_atomic_hash64(seed, unit << 28 | phase << 27 | GSB_SHARED_ATOMIC_TAG, t * 32u + r);
}

/* a starting unit's hash */
GSB_HD uint64_t gsb_shared_atomic_init_key(uint32_t unit, uint32_t seed, uint32_t u) {
  return gsb_atomic_hash64(seed, unit << 28 | GSB_ATOMIC_INIT_TAG | GSB_SHARED_ATOMIC_TAG, u);
}

/* inc / dec: the one bound every contribution to word x (its logical index) takes, 8 .. 31 */
GSB_HD uint32_t gsb_shared_atomic_bound(uint32_t unit, uint32_t seed, uint32_t x) {
  return 8u + gsb_atomic_hash(seed, unit << 28 | GSB_SHARED_ATOMIC_BOUND_TAG, x) % 24u;
}

/* the logical index of unit u: itself in the spread region, its slot in the hot area */
GSB_HD uint32_t gsb_shared_atomic_logical(uint32_t unit, uint32_t u) {
  const uint32_t ub = gsb_shared_atomic_unit_bytes(unit);
  return gsb_shared_atomic_is_hot(unit, u) ? (u * ub - GSB_SHARED_ATOMIC_SPREAD_BYTES) / GSB_SHARED_ATOMIC_HOT_STRIDE
                                           : u;
}

/* The operand of an integer contribution with hash h to unit u of `kind` (INT32, WIDE). */
GSB_HD uint64_t gsb_shared_atomic_operand(uint32_t unit, uint32_t seed, uint32_t kind, uint32_t u, uint64_t h) {
  const uint32_t bits = unit == GSB_SHARED_ATOMIC_UNIT_WIDE ? 64u : 32u;
  const uint64_t mask = bits == 32u ? 0xFFFFFFFFull : ~0ull;
  const uint64_t one = 1ull << ((uint32_t)h % bits);
  switch (kind) {
    case 1: return ~one & mask;  /* and clears a bit */
    case 2: return one;          /* or sets one */
    case 8:
    case 9: return gsb_shared_atomic_bound(unit, seed, gsb_shared_atomic_logical(unit, u));
    default: return h & mask;
  }
}

/* TICKET: the exchanged value of contributor id (id == GSB_SHARED_ATOMIC_COUNT: the starting word) of form f (1 b32,
 * 2 b64, 3 b128) on hot slot l, component c (32-bit words, c < 1, 2 or 4) */
GSB_HD uint32_t gsb_shared_atomic_exch(uint32_t seed, uint32_t f, uint32_t l, uint32_t id, uint32_t c) {
  return gsb_atomic_hash(seed, GSB_SHARED_ATOMIC_UNIT_TICKET << 28 | GSB_SHARED_ATOMIC_EXCH_TAG | f << 8 | l,
                         id * 4u + c);
}

/* CAS: the b64 counter's starting value on hot slot l (a count in the low half, the upper half fixed) and the upper
 * half of the b128 pair {count, pair(count)} */
GSB_HD uint64_t gsb_shared_atomic_cas64_start(uint32_t seed, uint32_t l) {
  return (uint64_t)gsb_atomic_hash(seed, GSB_SHARED_ATOMIC_UNIT_CAS << 28 | GSB_SHARED_ATOMIC_PAIR_TAG, l) << 32;
}
GSB_HD uint64_t gsb_shared_atomic_pair(uint32_t seed, uint32_t l, uint64_t count) {
  return gsb_atomic_hash64(seed, GSB_SHARED_ATOMIC_UNIT_CAS << 28 | GSB_SHARED_ATOMIC_PAIR_TAG | 1u << 8 | l,
                           (uint32_t)count);
}

/* The starting value of unit u, in the unit's bits. */
GSB_HD uint64_t gsb_shared_atomic_init(uint32_t unit, uint32_t seed, uint32_t u) {
  const uint64_t h = gsb_shared_atomic_init_key(unit, seed, u);
  const uint32_t kind = gsb_shared_atomic_kind(unit, u);
  const uint32_t phase = gsb_shared_atomic_is_hot(unit, u) ? GSB_ATOMIC_PHASE_HOT : GSB_ATOMIC_PHASE_SPREAD;
  const uint64_t hi = h & 0xFFFFFFFF00000000ull;  /* the upper half a 32-bit float form leaves alone */
  switch (unit) {
    case GSB_SHARED_ATOMIC_UNIT_INT32:
      switch (kind) {
        case 1: return 0xFFFFFFFFu;
        case 2: return 0u;
        case 4: return 0x7FFFFFFFu;  /* min starts at the largest value, max at the smallest */
        case 5: return 0x80000000u;
        case 6: return 0xFFFFFFFFu;
        case 7: return 0u;
        case 8:
        case 9: return (uint32_t)h % 40u;  /* below, at or above the word's bound */
        default: return (uint32_t)h;
      }
    case GSB_SHARED_ATOMIC_UNIT_WIDE:
      switch (kind) {
        case 1: return ~0ull;
        case 2: return 0u;
        case 4: return 0x7FFFFFFFFFFFFFFFull;
        case 5: return 0u;
        default: return h;
      }
    case GSB_SHARED_ATOMIC_UNIT_FLOAT:
      switch (kind) {
        case 0: return hi | gsb_atomic_f32_bits(gsb_atomic_init_ival(GSB_ATOMIC_OP_FADD32, phase, h));
        case 1: return gsb_atomic_f64_bits(gsb_atomic_init_ival(GSB_ATOMIC_OP_FADD64, phase, h));
        default:
          return hi | gsb_atomic_half2(kind - 2u, gsb_atomic_init_ival(GSB_ATOMIC_OP_HADD2, phase, h & 0xFFFFu),
                                       gsb_atomic_init_ival(GSB_ATOMIC_OP_HADD2, phase, (h >> 16) & 0xFFFFu));
      }
    default: {  /* TICKET, CAS: 4-byte units; the counters start at 0, the exchange words at their starting value */
      if (!gsb_shared_atomic_is_hot(unit, u)) return (uint32_t)h;
      const uint32_t off = (u * 4u - GSB_SHARED_ATOMIC_SPREAD_BYTES) % GSB_SHARED_ATOMIC_HOT_STRIDE;
      const uint32_t l = (u * 4u - GSB_SHARED_ATOMIC_SPREAD_BYTES) / GSB_SHARED_ATOMIC_HOT_STRIDE;
      if (off == 0u) return 0u;
      if (unit == GSB_SHARED_ATOMIC_UNIT_TICKET) {
        if (off >= GSB_SHARED_ATOMIC_TICKET_EXCH32 && off < GSB_SHARED_ATOMIC_TICKET_EXCH32 + 4u)
          return gsb_shared_atomic_exch(seed, 1u, l, GSB_SHARED_ATOMIC_COUNT, 0u);
        if (off >= GSB_SHARED_ATOMIC_TICKET_EXCH64 && off < GSB_SHARED_ATOMIC_TICKET_EXCH64 + 8u)
          return gsb_shared_atomic_exch(seed, 2u, l, GSB_SHARED_ATOMIC_COUNT, (off - GSB_SHARED_ATOMIC_TICKET_EXCH64) / 4u);
        if (off >= GSB_SHARED_ATOMIC_TICKET_EXCH128 && off < GSB_SHARED_ATOMIC_TICKET_EXCH128 + 16u)
          return gsb_shared_atomic_exch(seed, 3u, l, GSB_SHARED_ATOMIC_COUNT, (off - GSB_SHARED_ATOMIC_TICKET_EXCH128) / 4u);
        return (uint32_t)h;
      }
      if (off == GSB_SHARED_ATOMIC_CAS64) return (uint32_t)gsb_shared_atomic_cas64_start(seed, l);
      if (off == GSB_SHARED_ATOMIC_CAS64 + 4u) return (uint32_t)(gsb_shared_atomic_cas64_start(seed, l) >> 32);
      if (off >= GSB_SHARED_ATOMIC_CAS128 && off < GSB_SHARED_ATOMIC_CAS128 + 8u) return 0u;  /* the count */
      if (off == GSB_SHARED_ATOMIC_CAS128 + 8u) return (uint32_t)gsb_shared_atomic_pair(seed, l, 0u);
      if (off == GSB_SHARED_ATOMIC_CAS128 + 12u) return (uint32_t)(gsb_shared_atomic_pair(seed, l, 0u) >> 32);
      return (uint32_t)h;
    }
  }
}

/* 4-byte word w of the starting area */
GSB_HD uint32_t gsb_shared_atomic_init_word(uint32_t unit, uint32_t seed, uint32_t w) {
  const uint32_t ub = gsb_shared_atomic_unit_bytes(unit);
  return (uint32_t)(gsb_shared_atomic_init(unit, seed, w * 4u / ub) >> (8u * (w * 4u % ub)));
}

/* whether the kernel compares 4-byte word w: all but TICKET's exchange words, whose final value depends on the order
 * (they go to the slots and are checked there) */
GSB_HD int gsb_shared_atomic_compared(uint32_t unit, uint32_t w) {
  if (unit != GSB_SHARED_ATOMIC_UNIT_TICKET || w * 4u < GSB_SHARED_ATOMIC_SPREAD_BYTES) return 1;
  const uint32_t off = (w * 4u - GSB_SHARED_ATOMIC_SPREAD_BYTES) % GSB_SHARED_ATOMIC_HOT_STRIDE;
  const int exch32 = off >= GSB_SHARED_ATOMIC_TICKET_EXCH32 && off < GSB_SHARED_ATOMIC_TICKET_EXCH32 + 4u;
  const int exch64 = off >= GSB_SHARED_ATOMIC_TICKET_EXCH64 && off < GSB_SHARED_ATOMIC_TICKET_EXCH64 + 8u;
  const int exch128 = off >= GSB_SHARED_ATOMIC_TICKET_EXCH128 && off < GSB_SHARED_ATOMIC_TICKET_EXCH128 + 16u;
  return !(exch32 || exch64 || exch128);
}

/* the first word of slot entry i of form f (TICKET: 0 add tickets, 1-3 exchanges; CAS: 0-2 b32, b64, b128) on hot slot
 * l of CTA b: 4 words each; an add or CAS ticket t holds the id at entry t, an exchange returned to contributor id its
 * value at entry id and the final exchange word at entry GSB_SHARED_ATOMIC_COUNT */
GSB_HD uint64_t gsb_shared_atomic_slot(uint32_t b, uint32_t f, uint32_t l, uint32_t i) {
  return ((((uint64_t)b * GSB_SHARED_ATOMIC_FORMS + f) * GSB_SHARED_ATOMIC_HOT_WORDS + l) * GSB_SHARED_ATOMIC_ENTRIES + i) *
         4u;
}

/* ---- DSMEM and REDAS: atomics into every other rank's area of a cluster. 4-byte words; 8-byte ones at even words.
 *
 * DSMEM: words [0, 1024) add.u32 (op j = 0..3 of thread t hits word t + 256 j), [1024, 2048) 512 add.u64 words (j = 4,
 * 5: u64 word t + 256 (j - 4)), [2048, 2816) add.f32 (j = 6..8: word 2048 + t + 256 (j - 6)), then 32 cas.b32 counters
 * 8 words apart from word 2816 (lane l of every warp increments counter l once per peer).
 * REDAS: add.u32 word t (j = 0), add.u64 u64 word 128 + t (j = 1), xor.b32 word 768 + t (j = 2), max.s32 word 1024 + t
 * (j = 3), inc.u32 word 1280 + t (j = 4); 24 bytes per thread and peer. The other words keep their starting value. */
#define GSB_SHARED_ATOMIC_DSMEM_U64 1024u
#define GSB_SHARED_ATOMIC_DSMEM_F32 2048u
#define GSB_SHARED_ATOMIC_DSMEM_CAS 2816u
#define GSB_SHARED_ATOMIC_DSMEM_OPS 9u
#define GSB_SHARED_ATOMIC_REDAS_OPS 5u
#define GSB_SHARED_ATOMIC_REDAS_BYTES 24u /* bytes one thread sends one peer */

GSB_HD int gsb_shared_atomic_is_cluster(uint32_t unit) {
  return unit == GSB_SHARED_ATOMIC_UNIT_DSMEM || unit == GSB_SHARED_ATOMIC_UNIT_REDAS;
}

/* the hash of op j of thread t of the CTA of cluster rank q: the same for every peer it is sent to */
GSB_HD uint64_t gsb_shared_atomic_peer_key(uint32_t unit, uint32_t seed, uint32_t q, uint32_t t, uint32_t j) {
  return gsb_atomic_hash64(seed, unit << 28 | GSB_SHARED_ATOMIC_TAG | q << 8, t * 32u + j);
}

/* the first 4-byte word op j of thread t lands on */
GSB_HD uint32_t gsb_shared_atomic_peer_word(uint32_t unit, uint32_t t, uint32_t j) {
  if (unit == GSB_SHARED_ATOMIC_UNIT_DSMEM) {
    if (j < 4u) return t + 256u * j;
    if (j < 6u) return GSB_SHARED_ATOMIC_DSMEM_U64 + 2u * (t + 256u * (j - 4u));
    if (j < 9u) return GSB_SHARED_ATOMIC_DSMEM_F32 + t + 256u * (j - 6u);
    return GSB_SHARED_ATOMIC_DSMEM_CAS + 8u * (t & 31u);
  }
  return j == 0u ? t : j == 1u ? 256u + 2u * t : 768u + 256u * (j - 2u) + t;
}

/* the operand of op j of sender q's thread t (the low 32 bits for the 32-bit ops; REDAS's inc: the word's bound) */
GSB_HD uint64_t gsb_shared_atomic_peer_operand(uint32_t unit, uint32_t seed, uint32_t q, uint32_t t, uint32_t j) {
  const uint64_t h = gsb_shared_atomic_peer_key(unit, seed, q, t, j);
  if (unit == GSB_SHARED_ATOMIC_UNIT_DSMEM && j >= 6u && j < 9u)
    return gsb_atomic_f32_bits(gsb_atomic_ival(GSB_ATOMIC_OP_FADD32, GSB_ATOMIC_PHASE_SPREAD, h));
  if (unit == GSB_SHARED_ATOMIC_UNIT_REDAS && j == 4u) return gsb_shared_atomic_bound(unit, seed, t);
  return h;
}

/* 4-byte word w of a cluster unit's starting area: the same on every rank */
GSB_HD uint32_t gsb_shared_atomic_cluster_init_word(uint32_t unit, uint32_t seed, uint32_t w) {
  const uint32_t h = (uint32_t)gsb_shared_atomic_init_key(unit, seed, w);
  if (unit == GSB_SHARED_ATOMIC_UNIT_DSMEM) {
    if (w >= GSB_SHARED_ATOMIC_DSMEM_F32 && w < GSB_SHARED_ATOMIC_DSMEM_CAS)
      return gsb_atomic_f32_bits(gsb_atomic_init_ival(GSB_ATOMIC_OP_FADD32, GSB_ATOMIC_PHASE_SPREAD, h));
    if (w >= GSB_SHARED_ATOMIC_DSMEM_CAS && (w - GSB_SHARED_ATOMIC_DSMEM_CAS) % 8u == 0u) return 0u;  /* counters */
    return h;
  }
  if (w >= 1024u && w < 1280u) return 0x80000000u;  /* max.s32 starts at the smallest value */
  if (w >= 1280u && w < 1536u) return h % 40u;      /* inc: below, at or above the word's bound */
  return h;
}

#endif /* GSB_SHARED_ATOMIC_H_ */
