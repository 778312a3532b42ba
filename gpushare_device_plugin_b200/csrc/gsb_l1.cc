/*
 * gsb_l1.cc — pure host half of the L1 and constant-cache check (gsb_l1_probe): the schedule its kernels follow, its
 * conditions and the one log line both daemons print. No CUDA, no state.
 */
#include <stdio.h>
#include <algorithm>
#include <string.h>

#include <string>
#include <vector>

#include "../../include/gpushare_b200.h"
#include "gsb_l1.h"

namespace {

const char *const kUnitName[GSB_L1_UNITS] = {"l1_load", "l1_store", "nc", "tex", "const", "param"};
const char *const kFormName[GSB_L1_FORMS] = {"ca", "plain", "evict_last", "nc"};

}  // namespace

bool gsb_l1_table_valid(uint32_t unit, const uint32_t *table, size_t n, const uint32_t *expected, size_t n_expected,
                        uint32_t region_words) {
  if (unit >= GSB_L1_UNITS || !table || n == 0 || n > GSB_L1_TABLE_MAX || n_expected > GSB_L1_TABLE_EXPECTED_MAX)
    return false;
  const uint32_t fixed = gsb_l1_table_fixed_words(unit);
  if (fixed ? region_words != fixed
            : region_words == 0 || region_words % GSB_L1_THREADS || region_words > GSB_L1_TABLE_REGION_MAX)
    return false;
  const uint64_t per_cta = gsb_l1_table_expected_per_cta(unit, n, region_words);
  if (per_cta == 0 ? n_expected != 0 : !expected || n_expected == 0 || n_expected % per_cta) return false;
  switch (unit) {
    case GSB_L1_UNIT_L1_LOAD:
    case GSB_L1_UNIT_NC:
      if (n % region_words) return false;
      break;
    case GSB_L1_UNIT_L1_STORE: {
      const size_t rounds = (n - 1) / GSB_L1_THREADS;
      if (region_words > 1u << GSB_L1_STORE_WORD_BITS || (n - 1) % GSB_L1_THREADS || rounds == 0 ||
          rounds > GSB_L1_TABLE_ROUNDS_MAX || table[0] & ~(GSB_L1_TABLE_RESIDENT | GSB_L1_TABLE_READ_OWN))
        return false;
      std::vector<uint16_t> stored(region_words);  // the bytes of each word stored so far in the round
      for (size_t r = 0; r < rounds; r++) {
        std::fill(stored.begin(), stored.end(), 0);
        for (uint32_t t = 0; t < GSB_L1_THREADS; t++) {
          const uint32_t e = table[1 + r * GSB_L1_THREADS + t];
          if (e == 0) continue;
          const uint32_t code = e >> (GSB_L1_STORE_WORD_BITS + 4) & 7u, w = gsb_l1_entry_word(e);
          const uint32_t lo = gsb_l1_entry_lo(e), width = gsb_l1_entry_width(e);
          if (code == 0 || code > 5 || gsb_l1_entry_gen(e) == 0 || w >= region_words || lo % width || lo + width > 16)
            return false;
          const uint32_t mask = ((1u << width) - 1u) << lo;
          if (stored[w] & mask) return false;  // a data race: no reference can say which byte wins
          stored[w] = (uint16_t)(stored[w] | mask);
        }
      }
      return true;
    }
    case GSB_L1_UNIT_TEX:
      if (n % (2 * GSB_L1_THREADS)) return false;
      for (size_t r = 0; r < n / 2; r++) {
        const int32_t x = (int32_t)table[2 * r], y = (int32_t)table[2 * r + 1];
        const int32_t lim = 1 << 21;  // (float)(band + y) + 0.5f stays exact
        if (table[2 * r + 1] == GSB_L1_TEX_1D ? x < 0 || x >= (int32_t)GSB_L1_REGION_WORDS
                                               : x <= -lim || x >= lim || y <= -lim || y >= lim)
          return false;
      }
      for (size_t i = 0; i < n_expected; i++)
        if ((int32_t)expected[i] < -1) return false;
      return true;
    default:  // CONST, PARAM
      if (n % GSB_L1_THREADS) return false;
      break;
  }
  for (size_t i = 0; i < n; i++)  // word indices inside the region, the bank or the parameter
    if (table[i] >= region_words) return false;
  return true;
}

extern "C" {

int64_t gsb_l1_schedule(uint32_t unit, uint32_t form, uint32_t pass, uint32_t cta, uint32_t ctas, uint32_t thread,
                        uint32_t step) {
  const uint32_t steps = gsb_l1_steps(unit, form);
  if (steps == 0 || step >= steps || thread >= GSB_L1_THREADS || cta >= ctas || pass >= GSB_L1_PASSES_MAX)
    return GSB_ERR_INVALID_ARGUMENT;
  const bool passes = unit == GSB_L1_UNIT_L1_LOAD || unit == GSB_L1_UNIT_NC;
  if (pass != 0 && !passes) return GSB_ERR_INVALID_ARGUMENT;
  const int64_t base = (int64_t)cta * GSB_L1_REGION_WORDS;
  const uint32_t q = step * GSB_L1_THREADS + thread;
  switch (unit) {
    case GSB_L1_UNIT_L1_LOAD:
    case GSB_L1_UNIT_NC: return base + gsb_l1_order(pass, q);
    case GSB_L1_UNIT_L1_STORE: return base + q;
    case GSB_L1_UNIT_TEX: {
      if (form == 0) return base + q;
      int32_t x, y;
      gsb_l1_tex_coord(q, cta, ctas, &x, &y);
      const int64_t w = gsb_l1_texel(x, y, ctas * GSB_L1_TEX_ROWS, form == 1);
      return w < 0 ? GSB_L1_ZERO_TEXEL : w;
    }
    case GSB_L1_UNIT_CONST: return form == 0 ? step : q;
    default:  // PARAM
      if (form == 0) return step;
      return q < GSB_L1_PARAM_WORDS ? (int64_t)q : (int64_t)GSB_ERR_INVALID_ARGUMENT;
  }
}

uint32_t gsb_l1_conditions(const gsb_l1_result *r) {
  if (!r) return 0;
  uint32_t c = 0;
  for (int u = 0; u < GSB_L1_UNITS; u++) {
    const gsb_l1_unit_result &ur = r->unit[u];
    if (ur.launches == 0) continue;
    if (ur.status != GSB_OK) c |= GSB_L1_FAILED;
    if (ur.mismatch_words) c |= GSB_L1_CORRUPT;
  }
  return c;
}

int64_t gsb_l1_text(const gsb_l1_result *r, const char *uuid, char *buf, size_t cap) {
  if (!r) return GSB_ERR_INVALID_ARGUMENT;
  std::string s = "L1 and constant caches of ";
  s += uuid && uuid[0] ? uuid : "?";
  char head[96];
  snprintf(head, sizeof head, ": seed 0x%08x; SMs covered %u of %u; launches", r->seed, r->sms_covered, r->sm_count);
  s += head;
  for (int u = 0; u < GSB_L1_UNITS; u++) s += std::string(" ") + kUnitName[u] + " " + std::to_string(r->unit[u].launches);
  s += "; mismatching words";
  for (int u = 0; u < GSB_L1_UNITS; u++) {
    const gsb_l1_unit_result &ur = r->unit[u];
    s += std::string(" ") + kUnitName[u] + " " +
         (ur.launches == 0 ? std::string("-")
          : ur.status != GSB_OK ? std::string("failed")
                                : std::to_string((unsigned long long)ur.mismatch_words));
  }
  s += "; faulty SMs";
  bool any = false;
  for (uint32_t sm = 0; sm < GSB_SM_MAX; sm++) {
    if (!(r->faulty[sm >> 5] >> (sm & 31u) & 1u)) continue;
    s += " " + std::to_string(sm);
    any = true;
  }
  if (!any) s += " none";
  const bool load = r->unit[GSB_L1_UNIT_L1_LOAD].launches != 0, nc = r->unit[GSB_L1_UNIT_NC].launches != 0;
  if (load || nc) {
    s += "; warm/cold";
    for (int f = 0; f < GSB_L1_FORMS; f++) {
      char e[48];
      if ((f == GSB_L1_FORM_NC ? nc : load) && r->warm_cold[f] > 0) snprintf(e, sizeof e, " %s %.3g", kFormName[f], r->warm_cold[f]);
      else snprintf(e, sizeof e, " %s -", kFormName[f]);
      s += e;
    }
  }
  if (r->n_records) {
    uint32_t per[5] = {0, 0, 0, 0, 0};
    const uint32_t n = r->n_records < GSB_L1_RECORDS ? r->n_records : GSB_L1_RECORDS;
    for (uint32_t i = 0; i < n; i++) per[r->records[i].cls <= GSB_FAULT_BITS ? r->records[i].cls : 0]++;
    char e[128];
    snprintf(e, sizeof e, "; records %u (zero %u, stale %u, aliased %u, bits %u)", n, per[GSB_FAULT_ZERO],
             per[GSB_FAULT_STALE], per[GSB_FAULT_ALIASED], per[GSB_FAULT_BITS]);
    s += e;
  }
  const uint32_t c = gsb_l1_conditions(r);
  s += "; ";
  bool ran = false;
  for (int u = 0; u < GSB_L1_UNITS; u++) ran = ran || r->unit[u].launches != 0;
  if (!c) s += ran && r->status == GSB_OK ? "clean" : "not run";
  if (c & GSB_L1_FAILED) s += "FAILED ";
  if (c & GSB_L1_CORRUPT) s += "CORRUPT ";
  if (c) s.pop_back();
  if (!buf) return (int64_t)s.size() + 1;
  if (cap < s.size() + 1) return GSB_ERR_BUFFER_TOO_SMALL;
  memcpy(buf, s.c_str(), s.size() + 1);
  return (int64_t)s.size();
}

}  // extern "C"
