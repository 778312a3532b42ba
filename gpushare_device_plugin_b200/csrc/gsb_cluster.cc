/*
 * gsb_cluster.cc — pure host half of SM-to-SM health: which conditions a gsb_cluster_result raises, what a wrong word
 * holds, and the one log line both daemons print. No CUDA, no state.
 */
#include <stdio.h>
#include <string.h>

#include <string>

#include "gsb_cluster.h"

namespace {

const char *const kPathName[GSB_CLUSTER_PATHS] = {"dsmem_st", "dsmem_ld", "st_async", "bulk_s2s", "multicast"};

// the inverse of an odd multiplier mod 2^32 (Newton: each step doubles the correct low bits; a * a = 1 mod 8)
uint32_t inverse(uint32_t a) {
  uint32_t x = a;
  for (int i = 0; i < 5; i++) x *= 2u - a * x;
  return x;
}

// gsb_mix32 undone, step by step
uint32_t unmix32(uint32_t h) {
  h ^= h >> 16;
  h *= inverse(0xC2B2AE35u);
  h ^= h >> 13;
  h ^= h >> 26;
  h *= inverse(0x85EBCA6Bu);
  h ^= h >> 16;
  return h;
}

bool same(const uint32_t a[4], const uint32_t b[4]) { return !memcmp(a, b, 16); }

}  // namespace

// Every mbarrier a script arms is owed exactly one sender's region: each slot of each area is filled at most once.
bool gsb_cluster_script_valid(uint32_t p, uint32_t n, uint32_t region_words, const uint8_t *route) {
  if (p >= GSB_CLUSTER_PATHS || n < 2 || n > GSB_CLUSTER_MAX_N || (n & (n - 1))) return false;
  if (!route) return true;
  if (!region_words || region_words > gsb_cluster_region_words(p, n, GSB_CLUSTER_SCRIPT_SMEM)) return false;
  const uint32_t slots = gsb_cluster_slots(p, n);
  uint32_t taken[GSB_CLUSTER_MAX_N] = {0};  // per area owner: the slots some pair lands in
  for (uint32_t s = 0; s < n; s++) {
    uint32_t row = GSB_CLUSTER_UNROUTED;
    for (uint32_t d = 0; d < n; d++) {
      const uint32_t t = route[s * n + d];
      if (t == GSB_CLUSTER_UNROUTED) continue;
      if (t >= slots || (s == d && p != GSB_CLUSTER_PATH_MULTICAST)) return false;
      if (p == GSB_CLUSTER_PATH_MULTICAST && row != GSB_CLUSTER_UNROUTED && row != t) return false;
      row = t;
      const uint32_t owner = p == GSB_CLUSTER_PATH_DSMEM_LD ? s : d;
      if (taken[owner] >> t & 1u) return false;
      taken[owner] |= 1u << t;
    }
  }
  return true;
}

extern "C" {

// Only runs that launched count. A probe that launched nothing (its buffer could not be taken, the device was not
// usable) has a non-OK status and no condition, as an SM probe that could not allocate raises none.
uint32_t gsb_cluster_conditions(const gsb_cluster_result *r) {
  if (!r) return 0;
  uint32_t c = 0;
  for (int p = 0; p < GSB_CLUSTER_PATHS; p++)
    for (int k = 0; k < GSB_CLUSTER_SIZES; k++) {
      const gsb_cluster_run &run = r->run[p][k];
      if (run.launches == 0) continue;
      if (run.status != GSB_OK || run.timeouts) c |= GSB_CLUSTER_FAILED;
      if (run.mismatch_words) c |= GSB_CLUSTER_CORRUPT;
    }
  return c;
}

int gsb_cluster_classify(uint32_t seed, uint32_t smem_bytes, const gsb_cluster_record *rec, gsb_cluster_class *out) {
  if (!rec || !out || rec->path >= GSB_CLUSTER_PATHS || rec->n < 2 || rec->n > GSB_CLUSTER_MAX_N ||
      (rec->n & (rec->n - 1)) || rec->src_rank >= rec->n || rec->dst_rank >= rec->n)
    return GSB_ERR_INVALID_ARGUMENT;
  const uint32_t p = rec->path, n = rec->n, s = rec->src_rank, d = rec->dst_rank;
  const uint32_t rw = gsb_cluster_region_words(p, n, smem_bytes);
  if (rec->index >= rw) return GSB_ERR_INVALID_ARGUMENT;
  memset(out, 0, sizeof *out);
  const uint32_t *o = rec->observed;
  for (int l = 0; l < 4; l++) out->flipped_bits += (uint32_t)__builtin_popcount(rec->expected[l] ^ o[l]);
  if (!(o[0] | o[1] | o[2] | o[3])) {
    out->cls = GSB_CLUSTER_CLASS_ZERO;
    return GSB_OK;
  }
  // the background of the area the word was read from: the receiver's (DSMEM_LD: the sender's, which it reads)
  const bool ld = p == GSB_CLUSTER_PATH_DSMEM_LD;
  const uint32_t owner = ld ? s : d, peer = ld ? d : s;
  uint32_t w[4];
  gsb_pattern_word(gsb_cluster_bg_addr(p, n, owner, gsb_cluster_slot(p, n, owner, peer) * rw + rec->index),
                   gsb_cluster_bg_key(seed), w);
  if (same(w, o)) {
    out->cls = GSB_CLUSTER_CLASS_STALE;
    return GSB_OK;
  }
  // an intact data word of the launch: lane 0 gives gsb_word_key(addr), which undoes to lo32 ^ hi32 * K0; each
  // candidate (s', d') fixes hi32, so it names one index i'
  const uint32_t key = gsb_seed_key(seed);
  const uint32_t x = unmix32(((o[0] ^ key) - GSB_PAT_C0) * inverse(GSB_PAT_K0));
  const uint32_t n_dst = p == GSB_CLUSTER_PATH_MULTICAST ? 1u : n;  // MULTICAST: one candidate per source
  for (uint32_t s2 = 0; s2 < n; s2++) {
    for (uint32_t d2 = 0; d2 < n_dst; d2++) {
      const uint32_t dd = p == GSB_CLUSTER_PATH_MULTICAST ? GSB_CLUSTER_EVERY_RANK : d2;
      if (p != GSB_CLUSTER_PATH_MULTICAST && s2 == d2) continue;
      const uint32_t hi = (uint32_t)(gsb_cluster_word_addr(p, n, s2, dd, 0) >> 32);
      const uint32_t i2 = x ^ hi * GSB_PAT_K0;
      if (i2 >= rw) continue;
      gsb_pattern_word(gsb_cluster_word_addr(p, n, s2, dd, i2), key, w);
      if (same(w, o)) {
        out->cls = GSB_CLUSTER_CLASS_MISROUTED;
        out->src_rank = s2;
        out->dst_rank = dd;
        out->index = i2;
        return GSB_OK;
      }
    }
  }
  out->cls = GSB_CLUSTER_CLASS_BITS;
  return GSB_OK;
}

int64_t gsb_cluster_text(const gsb_cluster_result *r, const char *uuid, char *buf, size_t cap) {
  if (!r) return GSB_ERR_INVALID_ARGUMENT;
  std::string s = "SM-to-SM of ";
  s += uuid && uuid[0] ? uuid : "?";
  char tmp[128];
  snprintf(tmp, sizeof tmp, ": seed 0x%08x; active clusters", r->seed);
  s += tmp;
  for (int k = 0; k < GSB_CLUSTER_SIZES; k++) s += " n" + std::to_string(2 << k) + " " + std::to_string(r->max_clusters[k]);
  bool ran = false;
  for (int k = 0; k < GSB_CLUSTER_SIZES; k++) {
    uint32_t launches = 0, covered = 0;
    bool any = false;
    for (int p = 0; p < GSB_CLUSTER_PATHS; p++) {
      const gsb_cluster_run &run = r->run[p][k];
      if (!run.launches) continue;
      covered = any && covered < run.sms_covered ? covered : run.sms_covered;  // the least any path reached
      launches += run.launches;
      any = true;
    }
    if (!any) continue;
    snprintf(tmp, sizeof tmp, "; n%d launches %u covered %u of %u", 2 << k, launches, covered, r->expect_covered[k]);
    s += tmp;
    ran = true;
  }
  s += "; mismatching words";
  uint64_t timeouts = 0;
  for (int p = 0; p < GSB_CLUSTER_PATHS; p++) {
    bool any = false, failed = false;
    uint64_t words = 0;
    for (int k = 0; k < GSB_CLUSTER_SIZES; k++) {
      const gsb_cluster_run &run = r->run[p][k];
      if (!run.launches) continue;
      any = true;
      failed = failed || run.status != GSB_OK;
      words += run.mismatch_words;
      timeouts += run.timeouts;
    }
    s += std::string(" ") + kPathName[p] + " " +
         (!any ? std::string("-") : failed ? std::string("failed") : std::to_string((unsigned long long)words));
  }
  s += "; timeouts " + std::to_string((unsigned long long)timeouts) + "; faulty SMs";
  bool anyf = false;
  for (uint32_t sm = 0; sm < GSB_CLUSTER_SM_MAX; sm++) {
    if (!(r->faulty[sm >> 5] >> (sm & 31u) & 1u)) continue;
    s += " " + std::to_string(sm);
    anyf = true;
  }
  if (!anyf) s += " none";
  const uint32_t c = gsb_cluster_conditions(r);
  s += "; ";
  if (!c) s += ran && r->status == GSB_OK ? "clean" : "not run";
  if (c & GSB_CLUSTER_FAILED) s += "FAILED ";
  if (c & GSB_CLUSTER_CORRUPT) s += "CORRUPT ";
  if (c) s.pop_back();
  if (!buf) return (int64_t)s.size() + 1;
  if (cap < s.size() + 1) return GSB_ERR_BUFFER_TOO_SMALL;
  memcpy(buf, s.c_str(), s.size() + 1);
  return (int64_t)s.size();
}

}  // extern "C"
