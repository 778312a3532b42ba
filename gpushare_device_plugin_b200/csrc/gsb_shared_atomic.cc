/*
 * gsb_shared_atomic.cc — pure host half of shared-memory atomic health: the area a clean run leaves in every CTA, which
 * conditions a gsb_shared_atomic_result raises, and the one log line both daemons print. No CUDA, no state.
 */
#include <stdio.h>
#include <string.h>

#include <string>
#include <vector>

#include "gsb_fenv.h"
#include "gsb_shared_atomic.h"

namespace {

const char *const kUnitName[GSB_SHARED_ATOMIC_UNITS] = {"int32", "wide", "float", "ticket", "cas", "dsmem", "redas"};

int64_t mag(int64_t v) { return v < 0 ? -v : v; }

// The area after a clean run. Float words are summed as integers, with the sum of magnitudes held to the type's exact
// bound, so the result does not depend on the order the atomic unit applied them in.
struct Expect {
  uint32_t unit, seed;
  std::vector<uint64_t> w;
  std::vector<int64_t> sum, abs_sum;  // FLOAT: two per unit (f16x2 and bf16x2 halves; f32 and f64 use the first)

  Expect(uint32_t unit_, uint32_t seed_) : unit(unit_), seed(seed_), w(gsb_shared_atomic_units(unit_)) {
    const bool flt = unit == GSB_SHARED_ATOMIC_UNIT_FLOAT;
    if (flt) sum.assign(2 * w.size(), 0), abs_sum.assign(2 * w.size(), 0);
    for (uint32_t u = 0; u < w.size(); u++) {
      w[u] = gsb_shared_atomic_init(unit, seed, u);
      if (!flt) continue;
      const uint64_t h = gsb_shared_atomic_init_key(unit, seed, u);
      const uint32_t ph = gsb_shared_atomic_is_hot(unit, u) ? GSB_ATOMIC_PHASE_HOT : GSB_ATOMIC_PHASE_SPREAD;
      switch (gsb_shared_atomic_kind(unit, u)) {
        case 0: add(2u * u, gsb_atomic_init_ival(GSB_ATOMIC_OP_FADD32, ph, h)); break;
        case 1: add(2u * u, gsb_atomic_init_ival(GSB_ATOMIC_OP_FADD64, ph, h)); break;
        default:
          add(2u * u, gsb_atomic_init_ival(GSB_ATOMIC_OP_HADD2, ph, h & 0xFFFFu));
          add(2u * u + 1u, gsb_atomic_init_ival(GSB_ATOMIC_OP_HADD2, ph, (h >> 16) & 0xFFFFu));
      }
    }
  }
  void add(size_t i, int64_t v) {
    sum[i] += v;
    abs_sum[i] += mag(v);
  }
  void apply(uint32_t phase, uint32_t t, uint32_t r, uint32_t u) {
    const uint64_t h = gsb_shared_atomic_key(unit, seed, phase, t, r);
    const uint32_t kind = gsb_shared_atomic_kind(unit, u);
    uint64_t &x = w[u];
    if (unit == GSB_SHARED_ATOMIC_UNIT_FLOAT) {
      if (kind == 0u) add(2u * u, gsb_atomic_ival(GSB_ATOMIC_OP_FADD32, phase, h));
      else if (kind == 1u) add(2u * u, gsb_atomic_ival(GSB_ATOMIC_OP_FADD64, phase, h));
      else {
        add(2u * u, gsb_atomic_ival(GSB_ATOMIC_OP_HADD2, phase, h & 0xFFFFu));
        add(2u * u + 1u, gsb_atomic_ival(GSB_ATOMIC_OP_HADD2, phase, (h >> 16) & 0xFFFFu));
      }
      return;
    }
    const uint64_t v = gsb_shared_atomic_operand(unit, seed, kind, u, h);
    if (unit == GSB_SHARED_ATOMIC_UNIT_WIDE) {
      switch (kind) {
        case 0: x += v; break;
        case 1: x &= v; break;
        case 2: x |= v; break;
        case 3: x ^= v; break;
        case 4: x = (int64_t)v < (int64_t)x ? v : x; break;
        default: x = v > x ? v : x; break;
      }
      return;
    }
    const uint32_t a = (uint32_t)x, b = (uint32_t)v;
    uint32_t y = a;
    switch (kind) {
      case 0: y = a + b; break;
      case 1: y = a & b; break;
      case 2: y = a | b; break;
      case 3: y = a ^ b; break;
      case 4: y = (int32_t)b < (int32_t)a ? b : a; break;
      case 5: y = (int32_t)b > (int32_t)a ? b : a; break;
      case 6: y = b < a ? b : a; break;
      case 7: y = b > a ? b : a; break;
      case 8: y = a >= b ? 0u : a + 1u; break;                 // inc.u32
      default: y = a == 0u || a > b ? b : a - 1u; break;       // dec.u32
    }
    x = y;
  }
  // false when a float word's sum of magnitudes reaches its exact-integer bound
  bool finish() {
    if (unit != GSB_SHARED_ATOMIC_UNIT_FLOAT) return true;
    for (uint32_t u = 0; u < w.size(); u++) {
      const uint64_t hi = w[u] & 0xFFFFFFFF00000000ull;
      const int64_t *s = &sum[2u * u], *m = &abs_sum[2u * u];
      switch (gsb_shared_atomic_kind(unit, u)) {
        case 0:
          if (m[0] >= (1ll << 24)) return false;
          w[u] = hi | gsb_atomic_f32_bits(s[0]);
          break;
        case 1:
          if (m[0] >= (1ll << 53)) return false;
          w[u] = gsb_atomic_f64_bits(s[0]);
          break;
        default: {
          const uint32_t kind = gsb_shared_atomic_kind(unit, u) - 2u;
          const int64_t bound = kind ? 1ll << 8 : 1ll << 11;
          if (m[0] >= bound || m[1] >= bound) return false;
          w[u] = hi | gsb_atomic_half2(kind, s[0], s[1]);
        }
      }
    }
    return true;
  }
};

// DSMEM and REDAS: rank `rank`'s area after every other rank of a cluster of n sent it its atomics. Float words are
// summed as integers under the f32 bound, as above.
bool cluster_area(uint32_t unit, uint32_t seed, uint32_t n, uint32_t rank, uint32_t *out) {
  for (uint32_t w = 0; w < GSB_SHARED_ATOMIC_AREA_WORDS; w++) out[w] = gsb_shared_atomic_cluster_init_word(unit, seed, w);
  const bool dsmem = unit == GSB_SHARED_ATOMIC_UNIT_DSMEM;
  const uint32_t ops = dsmem ? GSB_SHARED_ATOMIC_DSMEM_OPS : GSB_SHARED_ATOMIC_REDAS_OPS;
  std::vector<int64_t> sum, abs_sum;
  if (dsmem) {
    sum.assign(GSB_SHARED_ATOMIC_AREA_WORDS, 0), abs_sum.assign(GSB_SHARED_ATOMIC_AREA_WORDS, 0);
    for (uint32_t w = GSB_SHARED_ATOMIC_DSMEM_F32; w < GSB_SHARED_ATOMIC_DSMEM_CAS; w++) {
      const int64_t v = gsb_atomic_init_ival(GSB_ATOMIC_OP_FADD32, GSB_ATOMIC_PHASE_SPREAD,
                                             (uint32_t)gsb_shared_atomic_init_key(unit, seed, w));
      sum[w] = v, abs_sum[w] = mag(v);
    }
  }
  for (uint32_t q = 0; q < n; q++) {
    if (q == rank) continue;
    for (uint32_t t = 0; t < GSB_SHARED_ATOMIC_THREADS; t++)
      for (uint32_t j = 0; j < (dsmem ? ops + 1u : ops); j++) {  // DSMEM's last op is the CAS increment
        const uint32_t w = gsb_shared_atomic_peer_word(unit, t, j);
        if (dsmem && j == GSB_SHARED_ATOMIC_DSMEM_OPS) {
          out[w]++;
          continue;
        }
        const uint64_t v = gsb_shared_atomic_peer_operand(unit, seed, q, t, j);
        const uint32_t v32 = (uint32_t)v;
        const bool wide = dsmem ? (j == 4u || j == 5u) : j == 1u;
        if (wide) {
          const uint64_t x = ((uint64_t)out[w + 1u] << 32 | out[w]) + v;
          out[w] = (uint32_t)x, out[w + 1u] = (uint32_t)(x >> 32);
        } else if (dsmem && j >= 6u) {
          const int64_t f = gsb_atomic_ival(GSB_ATOMIC_OP_FADD32, GSB_ATOMIC_PHASE_SPREAD,
                                            gsb_shared_atomic_peer_key(unit, seed, q, t, j));
          sum[w] += f, abs_sum[w] += mag(f);
        } else if (dsmem || j == 0u) {
          out[w] += v32;
        } else if (j == 2u) {
          out[w] ^= v32;
        } else if (j == 3u) {
          out[w] = (int32_t)v32 > (int32_t)out[w] ? v32 : out[w];
        } else {
          out[w] = out[w] >= v32 ? 0u : out[w] + 1u;  // inc.u32
        }
      }
  }
  if (dsmem)
    for (uint32_t w = GSB_SHARED_ATOMIC_DSMEM_F32; w < GSB_SHARED_ATOMIC_DSMEM_CAS; w++) {
      if (abs_sum[w] >= (1ll << 24)) return false;
      out[w] = gsb_atomic_f32_bits(sum[w]);
    }
  return true;
}

}  // namespace

extern "C" {

int64_t gsb_shared_atomic_expected(uint32_t unit, uint32_t seed, uint32_t cluster, uint32_t rank, uint32_t *out,
                                   size_t cap) {
  if (unit >= GSB_SHARED_ATOMIC_UNITS) return GSB_ERR_INVALID_ARGUMENT;
  if (gsb_shared_atomic_is_cluster(unit) ? cluster < 2u || cluster > 16u || (cluster & (cluster - 1u)) || rank >= cluster
                                         : cluster != 1u || rank != 0u)
    return GSB_ERR_INVALID_ARGUMENT;
  if (!out) return GSB_SHARED_ATOMIC_AREA_WORDS;
  if (cap < GSB_SHARED_ATOMIC_AREA_WORDS) return GSB_ERR_BUFFER_TOO_SMALL;
  const GsbDefaultFpEnv env;
  if (gsb_shared_atomic_is_cluster(unit))
    return cluster_area(unit, seed, cluster, rank, out) ? GSB_SHARED_ATOMIC_AREA_WORDS : GSB_ERR_INVALID_ARGUMENT;
  Expect e(unit, seed);
  if (gsb_shared_atomic_has_spread(unit)) {
    for (uint32_t t = 0; t < GSB_SHARED_ATOMIC_THREADS; t++)
      for (uint32_t r = 0; r < gsb_shared_atomic_rounds(unit); r++)
        e.apply(GSB_ATOMIC_PHASE_SPREAD, t, r, gsb_shared_atomic_spread_unit(unit, t, r));
    for (uint32_t t = 0; t < GSB_SHARED_ATOMIC_THREADS; t++)
      for (uint32_t r = 0; r < GSB_SHARED_ATOMIC_HOT_REPS; r++)
        e.apply(GSB_ATOMIC_PHASE_HOT, t, r, gsb_shared_atomic_hot_unit(unit, t & 31u));
  }
  if (!e.finish()) return GSB_ERR_INVALID_ARGUMENT;
  const uint32_t ub = gsb_shared_atomic_unit_bytes(unit);
  for (uint32_t w = 0; w < GSB_SHARED_ATOMIC_AREA_WORDS; w++)
    out[w] = (uint32_t)(e.w[w * 4u / ub] >> (8u * (w * 4u % ub)));
  if (unit == GSB_SHARED_ATOMIC_UNIT_TICKET || unit == GSB_SHARED_ATOMIC_UNIT_CAS) {
    // every counter ends at the count: TICKET's add counter, CAS's b32, b64 and b128 counters (the pair's upper half
    // the hash of the count)
    for (uint32_t l = 0; l < GSB_SHARED_ATOMIC_HOT_WORDS; l++) {
      uint32_t *slot = out + (GSB_SHARED_ATOMIC_SPREAD_BYTES + l * GSB_SHARED_ATOMIC_HOT_STRIDE) / 4u;
      slot[0] = GSB_SHARED_ATOMIC_COUNT;
      if (unit != GSB_SHARED_ATOMIC_UNIT_CAS) continue;
      const uint64_t c64 = gsb_shared_atomic_cas64_start(seed, l) + GSB_SHARED_ATOMIC_COUNT;
      const uint64_t pair = gsb_shared_atomic_pair(seed, l, GSB_SHARED_ATOMIC_COUNT);
      slot[GSB_SHARED_ATOMIC_CAS64 / 4u] = (uint32_t)c64;
      slot[GSB_SHARED_ATOMIC_CAS64 / 4u + 1u] = (uint32_t)(c64 >> 32);
      slot[GSB_SHARED_ATOMIC_CAS128 / 4u] = GSB_SHARED_ATOMIC_COUNT;
      slot[GSB_SHARED_ATOMIC_CAS128 / 4u + 1u] = 0u;
      slot[GSB_SHARED_ATOMIC_CAS128 / 4u + 2u] = (uint32_t)pair;
      slot[GSB_SHARED_ATOMIC_CAS128 / 4u + 3u] = (uint32_t)(pair >> 32);
    }
  }
  return GSB_SHARED_ATOMIC_AREA_WORDS;
}

// Only units that launched count. A probe that launched nothing (its buffer could not be taken, the device was not
// usable) has a non-OK status and no condition.
uint32_t gsb_shared_atomic_conditions(const gsb_shared_atomic_result *r) {
  if (!r) return 0;
  uint32_t c = 0;
  for (int u = 0; u < GSB_SHARED_ATOMIC_UNITS; u++) {
    const gsb_shared_atomic_run &run = r->run[u];
    if (run.launches == 0) continue;
    if (run.status != GSB_OK || run.timeouts) c |= GSB_SHARED_ATOMIC_FAILED;
    if (run.mismatch_words || run.ticket_faults) c |= GSB_SHARED_ATOMIC_CORRUPT;
  }
  return c;
}

int64_t gsb_shared_atomic_text(const gsb_shared_atomic_result *r, const char *uuid, char *buf, size_t cap) {
  if (!r) return GSB_ERR_INVALID_ARGUMENT;
  std::string s = "shared-memory atomics of ";
  s += uuid && uuid[0] ? uuid : "?";
  uint32_t launches = 0;
  uint64_t faults = 0, timeouts = 0, cas_ns = 0;
  bool ran = false;
  std::string words;
  for (int u = 0; u < GSB_SHARED_ATOMIC_UNITS; u++) {
    const gsb_shared_atomic_run &run = r->run[u];
    words += std::string(" ") + kUnitName[u] + " ";
    if (!run.launches) {
      words += "-";
      continue;
    }
    ran = true;
    launches += run.launches;
    faults += run.ticket_faults;
    timeouts += run.timeouts;
    cas_ns = run.cas_max_ns > cas_ns ? run.cas_max_ns : cas_ns;
    words += run.status != GSB_OK ? std::string("failed") : std::to_string((unsigned long long)run.mismatch_words);
  }
  char tmp[160];
  snprintf(tmp, sizeof tmp, ": seed 0x%08x; launches %u covered %u of %u; mismatching words", r->seed, launches,
           r->sms_covered, r->sm_count);
  s += tmp;
  s += words;
  snprintf(tmp, sizeof tmp, "; ticket faults %llu; timeouts %llu; worst CAS loop %.1f us; faulty SMs",
           (unsigned long long)faults, (unsigned long long)timeouts, (double)cas_ns / 1e3);
  s += tmp;
  bool anyf = false;
  for (uint32_t sm = 0; sm < GSB_SM_MAX; sm++) {
    if (!(r->faulty[sm >> 5] >> (sm & 31u) & 1u)) continue;
    s += " " + std::to_string(sm);
    anyf = true;
  }
  if (!anyf) s += " none";
  const uint32_t c = gsb_shared_atomic_conditions(r);
  s += "; ";
  if (!c) s += ran && r->status == GSB_OK ? "clean" : "not run";
  if (c & GSB_SHARED_ATOMIC_FAILED) s += "FAILED ";
  if (c & GSB_SHARED_ATOMIC_CORRUPT) s += "CORRUPT ";
  if (c) s.pop_back();
  if (!buf) return (int64_t)s.size() + 1;
  if (cap < s.size() + 1) return GSB_ERR_BUFFER_TOO_SMALL;
  memcpy(buf, s.c_str(), s.size() + 1);
  return (int64_t)s.size();
}

}  // extern "C"
