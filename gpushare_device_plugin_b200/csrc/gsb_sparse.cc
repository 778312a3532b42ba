/*
 * gsb_sparse.cc — pure host half of sparse tensor-core health: the exact D every SM's sparse-check kernels must produce
 * (from the same gsb_sparse_kat.h the kernels use), which conditions a gsb_sparse_result raises, and the one log line
 * both daemons print. No CUDA, no state.
 */
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <string>
#include <vector>

#include "gsb_fenv.h"
#include "gsb_sparse_kat.h"

namespace {

const char *const kUnitName[GSB_SPARSE_UNITS] = {"f16", "bf16", "tf32", "e4m3", "e5m2", "s8", "hmma"};

// D = A B exactly in integers over the kept terms, then scaled by 2^(sa_i + sb_j): exact in FP32 because every |D'|
// stays under the unit's bound (gsb_sparse_kat.h). S8_SP's D is the int32 sum.
void gemm(uint32_t unit, uint32_t seed, uint32_t *out) {
  const uint32_t key = gsb_sparse_key(unit, seed);
  const uint32_t K = gsb_sparse_shape(unit).k, G = gsb_sparse_groups(unit), gk = gsb_sparse_group_k(unit);
  const uint32_t per = K / 2 / G;  // stored values per group: 2, TF32 1
  std::vector<int64_t> B((size_t)K * GSB_SM_N);
  for (uint32_t k = 0; k < K; k++)
    for (uint32_t j = 0; j < GSB_SM_N; j++) B[k * GSB_SM_N + j] = gsb_sparse_b(unit, key, k, j);
  int32_t sb[GSB_SM_N];
  for (uint32_t j = 0; j < GSB_SM_N; j++) sb[j] = gsb_sparse_sb(unit, key, j);
  for (uint32_t i = 0; i < GSB_SM_M; i++) {
    const int32_t sa = gsb_sparse_sa(unit, key, i);
    int64_t acc[GSB_SM_N] = {0};
    for (uint32_t q = 0; q < G; q++) {
      const uint32_t p = gsb_sparse_pattern(unit, key, i, q);
      for (uint32_t v = 0; v < per; v++) {
        const int64_t a = gsb_sparse_a(unit, key, i, per * q + v);
        const int64_t *b = &B[(size_t)(gk * q + gsb_sparse_index(unit, p, v)) * GSB_SM_N];
        for (uint32_t j = 0; j < GSB_SM_N; j++) acc[j] += a * b[j];
      }
    }
    for (uint32_t j = 0; j < GSB_SM_N; j++) {
      uint32_t &o = out[i * GSB_SM_N + j];
      if (unit == GSB_SPARSE_UNIT_S8_SP) {
        o = (uint32_t)(int32_t)acc[j];
      } else {
        const float x = ldexpf((float)acc[j], sa + sb[j]);
        memcpy(&o, &x, sizeof o);
      }
    }
  }
}

}  // namespace

extern "C" {

int64_t gsb_sparse_expected(uint32_t unit, uint32_t seed, uint32_t *out, size_t cap) {
  if (unit >= GSB_SPARSE_UNITS) return GSB_ERR_INVALID_ARGUMENT;
  if (!out) return GSB_SPARSE_WORDS;
  if (cap < GSB_SPARSE_WORDS) return GSB_ERR_BUFFER_TOO_SMALL;
  const GsbDefaultFpEnv env;
  gemm(unit, seed, out);
  return GSB_SPARSE_WORDS;
}

// Only units that ran count, as in gsb_tensor_conditions.
uint32_t gsb_sparse_conditions(const gsb_sparse_result *r) {
  if (!r) return 0;
  uint32_t c = 0;
  for (int u = 0; u < GSB_SPARSE_UNITS; u++) {
    const gsb_tensor_unit_result &ur = r->unit[u];
    if (ur.launches == 0) continue;
    if (ur.status != GSB_OK) c |= GSB_SPARSE_FAILED;
    if (ur.mismatch_words) c |= GSB_SPARSE_CORRUPT;
  }
  return c;
}

int64_t gsb_sparse_text(const gsb_sparse_result *r, const char *uuid, char *buf, size_t cap) {
  if (!r) return GSB_ERR_INVALID_ARGUMENT;
  std::string s = "sparse tensor cores of ";
  s += uuid && uuid[0] ? uuid : "?";
  char head[96];
  snprintf(head, sizeof head, ": seed 0x%08x; SMs covered %u of %u; launches", r->seed, r->sms_covered, r->sm_count);
  s += head;
  for (int u = 0; u < GSB_SPARSE_UNITS; u++)
    s += std::string(" ") + kUnitName[u] + " " + std::to_string(r->unit[u].launches);
  s += "; mismatching words";
  for (int u = 0; u < GSB_SPARSE_UNITS; u++) {
    const gsb_tensor_unit_result &ur = r->unit[u];
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
  const uint32_t c = gsb_sparse_conditions(r);
  s += "; ";
  bool ran = false;
  for (int u = 0; u < GSB_SPARSE_UNITS; u++) ran = ran || r->unit[u].launches != 0;
  if (!c) s += ran && r->status == GSB_OK ? "clean" : "not run";
  if (c & GSB_SPARSE_FAILED) s += "FAILED ";
  if (c & GSB_SPARSE_CORRUPT) s += "CORRUPT ";
  if (c) s.pop_back();
  if (!buf) return (int64_t)s.size() + 1;
  if (cap < s.size() + 1) return GSB_ERR_BUFFER_TOO_SMALL;
  memcpy(buf, s.c_str(), s.size() + 1);
  return (int64_t)s.size();
}

}  // extern "C"
