/*
 * gsb_order.cc — pure host half of the memory-ordering check (gsb_order_probe): the pairing schedule and outcome
 * classes of gsb_order.h exported for the tests, its conditions and the one log line both daemons print. No CUDA, no
 * state.
 */
#include <stdio.h>
#include <string.h>

#include <string>

#include "../../include/gpushare_b200.h"
#include "gsb_order.h"

namespace {

const char *const kUnitName[GSB_ORDER_UNITS] = {"mp_relacq", "mp_fence", "sb_sc", "iriw_sc", "corr", "mp_relaxed"};

}  // namespace

extern "C" {

uint32_t gsb_order_distance(uint32_t k, uint32_t n, uint32_t seed) { return gsb_order_distance_of(k, n, seed); }

uint32_t gsb_order_iriw_distance(uint32_t n, uint32_t d) { return gsb_order_iriw_step(n, d); }

int gsb_order_pairing(uint32_t unit, uint32_t n, uint32_t d, uint32_t rank, uint32_t ranks[3]) {
  if (!ranks) return 0;
  return gsb_order_pairing_of(unit, n, d, rank, ranks);
}

uint32_t gsb_order_classify(uint32_t unit, uint32_t seed, const uint32_t keys[GSB_ORDER_WORDS],
                            const uint64_t words[GSB_ORDER_WORDS], uint32_t iteration) {
  if (!keys || !words) return GSB_ORDER_CLS_CORRUPT;
  return gsb_order_classify_words(unit, seed, keys, words, iteration);
}

uint32_t gsb_order_conditions(const gsb_order_result *r) {
  if (!r) return 0;
  uint32_t c = 0;
  for (int u = 0; u < GSB_ORDER_UNITS; u++) {
    const gsb_order_unit_result &ur = r->unit[u];
    if (ur.status != GSB_OK) c |= GSB_ORDER_FAILED;
    if (ur.launches == 0) continue;
    if (ur.corrupt) c |= GSB_ORDER_CORRUPT;
    if (ur.forbidden) c |= GSB_ORDER_FORBIDDEN;
    if (ur.lost) c |= GSB_ORDER_LOST;
    if (ur.timeout) c |= GSB_ORDER_TIMEOUT;
  }
  return c;
}

int64_t gsb_order_text(const gsb_order_result *r, const char *uuid, char *buf, size_t cap) {
  if (!r) return GSB_ERR_INVALID_ARGUMENT;
  std::string s = "memory ordering of ";
  s += uuid && uuid[0] ? uuid : "?";
  char head[128];
  snprintf(head, sizeof head, ": seed 0x%08x; %u observations at distances %u %u %u; SMs covered %u of %u; launches",
           r->seed, r->observations, r->distance[0], r->distance[1], r->distance[2], r->sms_covered, r->sm_count);
  s += head;
  for (int u = 0; u < GSB_ORDER_UNITS; u++) {
    s += std::string(" ") + kUnitName[u] + " " + std::to_string(r->unit[u].launches);
    if (r->unit[u].refused) s += " (" + std::to_string(r->unit[u].refused) + " refused)";
  }
  s += "; forbidden";
  for (int u = 0; u < GSB_ORDER_UNITS - 1; u++) {
    const gsb_order_unit_result &ur = r->unit[u];
    s += std::string(" ") + kUnitName[u] + " " +
         (ur.launches == 0 ? std::string("-")
          : ur.status != GSB_OK ? std::string("failed")
                                : std::to_string((unsigned long long)ur.forbidden));
  }
  uint64_t corrupt = 0, lost = 0, timeout = 0;
  for (const gsb_order_unit_result &ur : r->unit) {
    corrupt += ur.corrupt;
    lost += ur.lost;
    timeout += ur.timeout;
  }
  char e[160];
  snprintf(e, sizeof e, "; corrupt %llu, lost %llu, timeouts %llu; overlap", (unsigned long long)corrupt,
           (unsigned long long)lost, (unsigned long long)timeout);
  s += e;
  for (int u = 0; u < GSB_ORDER_UNITS; u++)
    s += std::string(" ") + kUnitName[u] + " " +
         (r->unit[u].launches ? std::to_string((unsigned long long)r->unit[u].overlap) : std::string("-"));
  const gsb_order_unit_result &rx = r->unit[GSB_ORDER_UNIT_MP_RELAXED];
  s += "; relaxed weak " + (rx.launches ? std::to_string((unsigned long long)rx.weak) : std::string("-"));
  s += "; faulty SMs";
  bool any = false;
  for (uint32_t sm = 0; sm < GSB_SM_MAX; sm++) {
    if (!(r->faulty[sm >> 5] >> (sm & 31u) & 1u)) continue;
    s += " " + std::to_string(sm);
    any = true;
  }
  if (!any) s += " none";
  const uint32_t c = gsb_order_conditions(r);
  s += "; ";
  bool ran = false;
  for (int u = 0; u < GSB_ORDER_UNITS; u++) ran = ran || r->unit[u].launches != 0;
  if (!c) s += ran && r->status == GSB_OK ? "clean" : "not run";
  if (c & GSB_ORDER_FAILED) s += "FAILED ";
  if (c & GSB_ORDER_TIMEOUT) s += "TIMEOUT ";
  if (c & GSB_ORDER_CORRUPT) s += "CORRUPT ";
  if (c & GSB_ORDER_FORBIDDEN) s += "FORBIDDEN ";
  if (c & GSB_ORDER_LOST) s += "LOST ";
  if (c) s.pop_back();
  if (!buf) return (int64_t)s.size() + 1;
  if (cap < s.size() + 1) return GSB_ERR_BUFFER_TOO_SMALL;
  memcpy(buf, s.c_str(), s.size() + 1);
  return (int64_t)s.size();
}

}  // extern "C"
