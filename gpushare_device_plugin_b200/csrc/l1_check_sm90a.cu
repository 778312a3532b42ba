/*
 * l1_check_sm90a.cu — the L1 and constant-cache check's kernels (gsb_l1_probe): per unit, sm_count CTAs of
 * GSB_L1_THREADS read pattern words through one path of the SM's memory pipeline (L1 hits and stores, the read-only
 * path, the texture unit, the constant bank, the kernel parameters) and compare each with the word computed in
 * registers (gsb_pattern.h). Host code lives in gsb_device.cu (the probe) and gsb_l1.cc (schedule, verdict, text).
 *
 * The instruction bodies live in gsb_l1_isa.inc, which the test-only twins l1_from_table<UNIT> (l1_table_sm90a.cu)
 * compile from too. Nothing here assumes one CTA per SM, a honoured carveout or a load that hits: a CTA reads only
 * its own region and its own stores, so the answers stay exact whatever shares the SM; only coverage and the hit
 * ratio fall. Thread 0 of each CTA sets bit %smid of the launch's coverage bitmap.
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "gsb_internal.h"
#include "gsb_l1.h"

namespace {

// the whole user constant bank: no other kernel of the library declares __constant__
__constant__ uint4 gsb_l1_bank[GSB_L1_CONST_WORDS];

// the PARAM unit's kernel parameter: 32000 bytes of pattern words, read in place from constant bank 0
struct gsb_l1_param {
  uint4 w[GSB_L1_PARAM_WORDS];
};
static_assert(sizeof(gsb_l1_param) == 32000, "the PARAM unit's parameter is 32000 bytes");

#include "gsb_l1_isa.inc"

// ---- L1_LOAD and NC: every pass over the region with one load form, timed per pass ----------------------------------
template <uint32_t UNIT, uint32_t FORM>
__device__ __forceinline__ uint32_t passes(const gsb_l1_args &a, uint32_t sm, uint32_t key) {
  const uint32_t t = threadIdx.x, form = UNIT == GSB_L1_UNIT_NC ? 0u : FORM;
  const uint64_t base = (uint64_t)blockIdx.x * GSB_L1_REGION_WORDS;
  uint32_t n = 0;
  unsigned long long cold = 0, warm = 0;
#pragma unroll 1
  for (uint32_t pass = 0; pass < a.passes; pass++) {
    __syncthreads();
    const long long t0 = clock64();
#pragma unroll 1
    for (uint32_t k = 0; k < GSB_L1_STEPS; k++) {
      const uint32_t i = gsb_l1_order(pass, k * GSB_L1_THREADS + t);
      const uint4 o = load<FORM>(a.buf + base + i);
      const bool hook = form == 0 && pass == 0 && sm == a.hook_smid && i == a.hook_index;
      n += check(a, sm, UNIT, form, base + i, pattern(base + i, key), o, hook);
    }
    __syncthreads();
    const unsigned long long span = (unsigned long long)(clock64() - t0);
    if (pass == 0) cold = span;
    else warm += span;
  }
  if (t == 0) {
    a.spans[((size_t)blockIdx.x * GSB_L1_FORMS + FORM) * 2] = cold;
    a.spans[((size_t)blockIdx.x * GSB_L1_FORMS + FORM) * 2 + 1] = warm;
  }
  return n;
}

__global__ void __launch_bounds__(GSB_L1_THREADS, 1) l1_load(const gsb_l1_args a) {
  const uint32_t sm = smid(), key = gsb_seed_key(a.seed_expect);
  begin(a, sm);
  uint32_t n = passes<GSB_L1_UNIT_L1_LOAD, GSB_L1_FORM_CA>(a, sm, key);
  n += passes<GSB_L1_UNIT_L1_LOAD, GSB_L1_FORM_PLAIN>(a, sm, key);
  n += passes<GSB_L1_UNIT_L1_LOAD, GSB_L1_FORM_EVICT_LAST>(a, sm, key);
  add_words(a.log, n);
}

__global__ void __launch_bounds__(GSB_L1_THREADS, 1) l1_nc(const gsb_l1_args a) {
  const uint32_t sm = smid();
  begin(a, sm);
  add_words(a.log, passes<GSB_L1_UNIT_NC, GSB_L1_FORM_NC>(a, sm, gsb_seed_key(a.seed_expect)));
}

// ---- L1_STORE: lines made resident, partial stores from another warp, read back through L1 -------------------------
__device__ __forceinline__ void store(uint4 *word, uint64_t w, uint32_t key2) {
  uint32_t lo, width;
  gsb_l1_store_span(w, &lo, &width);
  store_bytes(word, lo, width, pattern(w, key2));
}

__global__ void __launch_bounds__(GSB_L1_THREADS, 1) l1_store(const gsb_l1_args a) {
  const uint32_t t = threadIdx.x, sm = smid(), key = gsb_seed_key(a.seed_expect);
  begin(a, sm);
  const uint64_t base = (uint64_t)blockIdx.x * GSB_L1_REGION_WORDS;
  uint32_t n = 0;
#pragma unroll 1
  for (uint32_t k = 0; k < GSB_L1_STEPS; k++) {  // generation 1, through L1
    const uint32_t i = k * GSB_L1_THREADS + t;
    n += check(a, sm, GSB_L1_UNIT_L1_STORE, 0, base + i, pattern(base + i, key), ld_ca(a.buf + base + i), false);
  }
  __syncthreads();
  if (sm != a.skip_smid) {
    const uint32_t key2 = gsb_seed_key(gsb_l1_gen2_seed(a.seed));
#pragma unroll 1
    for (uint32_t k = 0; k < GSB_L1_STEPS; k++) {
      const uint64_t w = base + k * GSB_L1_THREADS + gsb_l1_store_writer(t);
      store(a.buf + w, w, key2);
    }
  }
  __syncthreads();
#pragma unroll 1
  for (uint32_t k = 0; k < GSB_L1_STEPS; k++) {  // the byte merge, through L1
    const uint32_t i = k * GSB_L1_THREADS + t;
    uint32_t e[4];
    gsb_l1_store_expected(base + i, a.seed_expect, e);
    const bool hook = sm == a.hook_smid && i == a.hook_index;
    n += check(a, sm, GSB_L1_UNIT_L1_STORE, 1, base + i, make_uint4(e[0], e[1], e[2], e[3]), ld_ca(a.buf + base + i),
               hook);
  }
  add_words(a.log, n);
}

// ---- TEX: 1-D fetches of the region, 2-D point reads with clamp and border addressing --------------------------------
__global__ void __launch_bounds__(GSB_L1_THREADS, 1) l1_tex(const gsb_l1_args a) {
  const uint32_t t = threadIdx.x, sm = smid(), key = gsb_seed_key(a.seed_expect);
  begin(a, sm);
  const uint64_t base = (uint64_t)blockIdx.x * GSB_L1_REGION_WORDS;
  uint32_t n = 0;
#pragma unroll 1
  for (uint32_t k = 0; k < GSB_L1_STEPS; k++) {
    const uint32_t i = k * GSB_L1_THREADS + t;
    const uint4 o = tex1Dfetch<uint4>(a.tex_linear, (int)(base + i));
    n += check(a, sm, GSB_L1_UNIT_TEX, 0, base + i, pattern(base + i, key), o, sm == a.hook_smid && i == a.hook_index);
  }
#pragma unroll 1
  for (uint32_t k = 0; k < GSB_L1_TEX_2D_READS / GSB_L1_THREADS; k++) {
    const uint32_t i = k * GSB_L1_THREADS + t;
    int32_t x, y;
    gsb_l1_tex_coord(i, blockIdx.x, gridDim.x, &x, &y);
    const float fx = (float)x + 0.5f, fy = (float)y + 0.5f;
    const int64_t wc = gsb_l1_texel(x, y, a.rows, true), wb = gsb_l1_texel(x, y, a.rows, false);
    const uint4 oc = tex2D<uint4>(a.tex_clamp, fx, fy), ob = tex2D<uint4>(a.tex_border, fx, fy);
    const uint32_t ic = GSB_L1_REGION_WORDS + i, ib = ic + GSB_L1_TEX_2D_READS;
    n += check(a, sm, GSB_L1_UNIT_TEX, 1, (uint64_t)wc, pattern(wc, key), oc, sm == a.hook_smid && ic == a.hook_index);
    n += check(a, sm, GSB_L1_UNIT_TEX, 2, (uint64_t)wc, wb < 0 ? make_uint4(0, 0, 0, 0) : pattern(wb, key), ob,
               sm == a.hook_smid && ib == a.hook_index);
  }
  add_words(a.log, n);
}

// ---- CONST and PARAM: the constant bank and the kernel parameters, uniform and per-thread indices -------------------
// Every word of a bank, the same word across the warp at each step (a broadcast from the constant cache). ptxas
// keeps these indices in vector registers (LDC), whatever the loop's shape; ULDC serves the kernel's scalar
// parameters.
template <uint32_t UNIT, uint32_t WORDS>
__device__ __forceinline__ uint32_t uniform(const gsb_l1_args &a, uint32_t sm, uint32_t key, const uint4 *bank) {
#pragma unroll 1
  for (uint32_t w = 0; w < WORDS; w++) check(a, sm, UNIT, 0, w, pattern(w, key), bank[w], false);
  return WORDS;
}

__global__ void __launch_bounds__(GSB_L1_THREADS, 1) l1_const(const gsb_l1_args a) {
  const uint32_t t = threadIdx.x, sm = smid(), key = gsb_seed_key(a.seed_expect);
  begin(a, sm);
  uint32_t n = 0;
  n += uniform<GSB_L1_UNIT_CONST, GSB_L1_CONST_WORDS>(a, sm, key, gsb_l1_bank);
#pragma unroll 1
  for (uint32_t k = 0; k < GSB_L1_CONST_WORDS / GSB_L1_THREADS; k++) {
    const uint32_t w = k * GSB_L1_THREADS + t;
    n += check(a, sm, GSB_L1_UNIT_CONST, 1, w, pattern(w, key), gsb_l1_bank[w], sm == a.hook_smid && w == a.hook_index);
  }
  add_words(a.log, n);
}

__global__ void __launch_bounds__(GSB_L1_THREADS, 1) l1_param(const __grid_constant__ gsb_l1_param p,
                                                               const gsb_l1_args a) {
  const uint32_t t = threadIdx.x, sm = smid(), key = gsb_seed_key(a.seed_expect);
  begin(a, sm);
  uint32_t n = 0;
  n += uniform<GSB_L1_UNIT_PARAM, GSB_L1_PARAM_WORDS>(a, sm, key, p.w);
#pragma unroll 1
  for (uint32_t w = t; w < GSB_L1_PARAM_WORDS; w += GSB_L1_THREADS)
    n += check(a, sm, GSB_L1_UNIT_PARAM, 1, w, pattern(w, key), p.w[w], sm == a.hook_smid && w == a.hook_index);
  add_words(a.log, n);
}

const void *kernel_of(uint32_t unit) {
  switch (unit) {
    case GSB_L1_UNIT_L1_LOAD: return (const void *)l1_load;
    case GSB_L1_UNIT_L1_STORE: return (const void *)l1_store;
    case GSB_L1_UNIT_NC: return (const void *)l1_nc;
    case GSB_L1_UNIT_TEX: return (const void *)l1_tex;
    case GSB_L1_UNIT_CONST: return (const void *)l1_const;
    case GSB_L1_UNIT_PARAM: return (const void *)l1_param;
    default: return nullptr;
  }
}

}  // namespace

int gsb_l1_kernel_launch(uint32_t unit, uint32_t grid, const gsb_l1_args *a, const uint4 *param, cudaStream_t stream) {
  switch (unit) {
    case GSB_L1_UNIT_L1_LOAD: l1_load<<<grid, GSB_L1_THREADS, 0, stream>>>(*a); break;
    case GSB_L1_UNIT_L1_STORE: l1_store<<<grid, GSB_L1_THREADS, 0, stream>>>(*a); break;
    case GSB_L1_UNIT_NC: l1_nc<<<grid, GSB_L1_THREADS, 0, stream>>>(*a); break;
    case GSB_L1_UNIT_TEX: l1_tex<<<grid, GSB_L1_THREADS, 0, stream>>>(*a); break;
    case GSB_L1_UNIT_CONST: l1_const<<<grid, GSB_L1_THREADS, 0, stream>>>(*a); break;
    case GSB_L1_UNIT_PARAM:
      if (!param) return (int)cudaErrorInvalidValue;
      l1_param<<<grid, GSB_L1_THREADS, 0, stream>>>(*reinterpret_cast<const gsb_l1_param *>(param), *a);
      break;
    default: return (int)cudaErrorInvalidValue;
  }
  return (int)cudaGetLastError();
}

int gsb_l1_const_upload(const uint4 *host, cudaStream_t stream) {
  return (int)cudaMemcpyToSymbolAsync(gsb_l1_bank, host, sizeof gsb_l1_bank, 0, cudaMemcpyHostToDevice, stream);
}

int gsb_l1_occupancy(uint32_t unit, int *ctas) {
  const void *fn = kernel_of(unit);
  if (!fn) return (int)cudaErrorInvalidValue;
  return (int)cudaOccupancyMaxActiveBlocksPerMultiprocessor(ctas, fn, GSB_L1_THREADS, 0);
}

int gsb_l1_kernel_preload(void) {
  for (uint32_t u = 0; u < GSB_L1_UNITS; u++) {
    cudaFuncAttributes attr;
    cudaError_t e = cudaFuncGetAttributes(&attr, kernel_of(u));
    // the units that read global memory ask for the largest L1: a hint the driver may round or ignore
    if (e == cudaSuccess && u <= GSB_L1_UNIT_TEX)
      e = cudaFuncSetAttribute(kernel_of(u), cudaFuncAttributePreferredSharedMemoryCarveout, 0);
    if (e != cudaSuccess) return (int)e;
  }
  return (int)cudaSuccess;
}
