/*
 * l1_table_sm90a.cu — the test-only twins l1_from_table<UNIT> of the L1 and constant-cache check's kernels
 * (gsb_test_l1_table, include/gpushare_b200.h): the shipped instructions (gsb_l1_isa.inc) on the reads and stores a
 * table chooses, compared on the SM with the pattern word or with the expected words the host uploads. Built into
 * libgpushare_b200_l1.so beside l1_check_sm90a.cu, as a translation unit of its own: without relocatable device code
 * each translation unit is a CUDA module of its own, so the CONST twin's 64 KiB bank fills this module's user bank as
 * gsb_l1_bank fills the shipped kernels'. Both banks hold the same pattern words, uploaded from the same host copy.
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "gsb_internal.h"
#include "gsb_l1.h"

namespace {

// the CONST twin's bank: the whole user constant bank of this module
__constant__ uint4 gsb_l1_table_bank[GSB_L1_CONST_WORDS];

// the PARAM twin's kernel parameter: 32000 bytes of pattern words, read in place from constant bank 0
struct table_param {
  uint4 w[GSB_L1_PARAM_WORDS];
};
static_assert(sizeof(table_param) == 32000, "the PARAM twin's parameter is 32000 bytes");

#include "gsb_l1_isa.inc"

// Table and expected entries are read with L1::no_allocate, so they do not take the lines a case is about.
__device__ __forceinline__ uint32_t entry(const uint32_t *p) {
  uint32_t v;
  asm volatile("ld.global.L1::no_allocate.u32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ uint4 entry4(const uint32_t *p) {
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}

// L1_LOAD and NC: the table's passes of region_words reads each, with one load form, timed as the shipped passes are
template <uint32_t UNIT, uint32_t FORM>
__device__ __forceinline__ uint32_t table_passes(const gsb_l1_args &a, const gsb_l1_table_args &tb, uint32_t sm,
                                                 uint32_t key) {
  const uint32_t t = threadIdx.x, form = UNIT == GSB_L1_UNIT_NC ? 0u : FORM;
  const uint32_t steps = tb.region_words / GSB_L1_THREADS, n_passes = tb.n / tb.region_words;
  const uint64_t base = (uint64_t)blockIdx.x * tb.region_words;
  uint32_t n = 0;
  unsigned long long cold = 0, warm = 0;
#pragma unroll 1
  for (uint32_t pass = 0; pass < n_passes; pass++) {
    __syncthreads();
    const long long t0 = clock64();
#pragma unroll 1
    for (uint32_t k = 0; k < steps; k++) {
      const uint32_t i = entry(tb.table + ((size_t)pass * steps + k) * GSB_L1_THREADS + t);
      const uint4 o = load<FORM>(a.buf + base + i);
      n += check(a, sm, UNIT, form, base + i, pattern(base + i, key), o, false);
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

// L1_STORE: the resident pass (flag), the rounds of stores (a writer's own read-back: flag), the read-back of the region
__device__ __forceinline__ uint32_t table_stores(const gsb_l1_args &a, const gsb_l1_table_args &tb, uint32_t sm,
                                                 uint32_t key) {
  const uint32_t t = threadIdx.x, flags = entry(tb.table), rounds = (tb.n - 1) / GSB_L1_THREADS;
  const uint32_t steps = tb.region_words / GSB_L1_THREADS;
  const uint64_t base = (uint64_t)blockIdx.x * tb.region_words;
  uint32_t n = 0;
  if (flags & GSB_L1_TABLE_RESIDENT) {
#pragma unroll 1
    for (uint32_t k = 0; k < steps; k++) {
      const uint32_t i = k * GSB_L1_THREADS + t;
      n += check(a, sm, GSB_L1_UNIT_L1_STORE, 0, base + i, pattern(base + i, key), ld_ca(a.buf + base + i), false);
    }
  }
#pragma unroll 1
  for (uint32_t r = 0; r < rounds; r++) {
    __syncthreads();
    const uint32_t e = entry(tb.table + 1 + (size_t)r * GSB_L1_THREADS + t), width = gsb_l1_entry_width(e);
    if (width == 0 || (sm == a.skip_smid && r + 1 == rounds)) continue;
    const uint32_t lo = gsb_l1_entry_lo(e);
    const uint64_t w = base + gsb_l1_entry_word(e);
    const uint4 g = pattern(w, gsb_seed_key(gsb_l1_table_seed(a.seed, gsb_l1_entry_gen(e))));
    store_bytes(a.buf + w, lo, width, g);
    if (flags & GSB_L1_TABLE_READ_OWN) {
      // the writer's own bytes only: the rest of the word may be another writer's in this round
      const uint4 o = ld_ca(a.buf + w);
      const uint32_t gv[4] = {g.x, g.y, g.z, g.w}, ov[4] = {o.x, o.y, o.z, o.w};
      uint32_t ev[4];
      gsb_copy_merge(gv, ov, lo, lo + width, ev);
      n += check(a, sm, GSB_L1_UNIT_L1_STORE, 2, w, make_uint4(ev[0], ev[1], ev[2], ev[3]), o, false);
    }
  }
  __syncthreads();
#pragma unroll 1
  for (uint32_t k = 0; k < steps; k++) {
    const uint32_t i = k * GSB_L1_THREADS + t;
    n += check(a, sm, GSB_L1_UNIT_L1_STORE, 1, base + i, entry4(tb.expected + (base + i) * 4), ld_ca(a.buf + base + i),
               false);
  }
  return n;
}

// TEX: 1-D fetches of region words, 2-D reads at texels of the CTA's band with clamp and border addressing
__device__ __forceinline__ uint32_t table_tex(const gsb_l1_args &a, const gsb_l1_table_args &tb, uint32_t sm,
                                              uint32_t key) {
  const uint32_t t = threadIdx.x, reads = tb.n / 2;
  const uint64_t base = (uint64_t)blockIdx.x * GSB_L1_REGION_WORDS;
  const int32_t band = (int32_t)(blockIdx.x * GSB_L1_TEX_ROWS);
  const uint32_t *ex = tb.expected + (size_t)blockIdx.x * tb.n;
  uint32_t n = 0;
#pragma unroll 1
  for (uint32_t k = 0; k < reads / GSB_L1_THREADS; k++) {
    const uint32_t r = k * GSB_L1_THREADS + t;
    const int32_t x = (int32_t)entry(tb.table + 2 * r), y = (int32_t)entry(tb.table + 2 * r + 1);
    const int32_t wc = (int32_t)entry(ex + 2 * r), wb = (int32_t)entry(ex + 2 * r + 1);
    if ((uint32_t)y == GSB_L1_TEX_1D) {
      const uint4 o = tex1Dfetch<uint4>(a.tex_linear, (int)(base + x));
      n += check(a, sm, GSB_L1_UNIT_TEX, 0, (uint64_t)wc, pattern(wc, key), o, false);
    } else {
      const uint4 oc = tex_at(a.tex_clamp, x, band + y), ob = tex_at(a.tex_border, x, band + y);
      n += check(a, sm, GSB_L1_UNIT_TEX, 1, (uint64_t)wc, pattern(wc, key), oc, false);
      n += check(a, sm, GSB_L1_UNIT_TEX, 2, (uint64_t)wc, wb < 0 ? make_uint4(0, 0, 0, 0) : pattern(wb, key), ob,
                 false);
    }
  }
  return n;
}

// CONST and PARAM: per-thread word indices into the bank or the parameter
template <uint32_t UNIT>
__device__ __forceinline__ uint32_t table_bank(const gsb_l1_args &a, const gsb_l1_table_args &tb, uint32_t sm,
                                               uint32_t key, const uint4 *bank) {
  uint32_t n = 0;
#pragma unroll 1
  for (uint32_t k = 0; k < tb.n / GSB_L1_THREADS; k++) {
    const uint32_t w = entry(tb.table + k * GSB_L1_THREADS + threadIdx.x);
    n += check(a, sm, UNIT, 1, w, pattern(w, key), bank[w], false);
  }
  return n;
}

template <uint32_t UNIT>
__global__ void __launch_bounds__(GSB_L1_THREADS, 1) l1_from_table(const gsb_l1_args a, const gsb_l1_table_args tb) {
  const uint32_t sm = smid(), key = gsb_seed_key(a.seed_expect);
  begin(a, sm);
  uint32_t n;
  if constexpr (UNIT == GSB_L1_UNIT_L1_LOAD) {
    n = table_passes<UNIT, GSB_L1_FORM_CA>(a, tb, sm, key);
    n += table_passes<UNIT, GSB_L1_FORM_PLAIN>(a, tb, sm, key);
    n += table_passes<UNIT, GSB_L1_FORM_EVICT_LAST>(a, tb, sm, key);
  } else if constexpr (UNIT == GSB_L1_UNIT_NC) {
    n = table_passes<UNIT, GSB_L1_FORM_NC>(a, tb, sm, key);
  } else if constexpr (UNIT == GSB_L1_UNIT_L1_STORE) {
    n = table_stores(a, tb, sm, key);
  } else if constexpr (UNIT == GSB_L1_UNIT_TEX) {
    n = table_tex(a, tb, sm, key);
  } else {
    n = table_bank<GSB_L1_UNIT_CONST>(a, tb, sm, key, gsb_l1_table_bank);
  }
  add_words(a.log, n);
}

template <uint32_t UNIT>
__global__ void __launch_bounds__(GSB_L1_THREADS, 1) l1_from_table(const __grid_constant__ table_param p,
                                                                    const gsb_l1_args a, const gsb_l1_table_args tb) {
  static_assert(UNIT == GSB_L1_UNIT_PARAM, "only PARAM takes the parameter");
  const uint32_t sm = smid();
  begin(a, sm);
  add_words(a.log, table_bank<GSB_L1_UNIT_PARAM>(a, tb, sm, gsb_seed_key(a.seed_expect), p.w));
}

}  // namespace

int gsb_l1_table_launch(uint32_t unit, uint32_t grid, const gsb_l1_args *a, const gsb_l1_table_args *t,
                        const uint4 *bank, const uint4 *param, cudaStream_t stream) {
  using Twin = void (*)(const gsb_l1_args, const gsb_l1_table_args);
  const Twin fn = unit == GSB_L1_UNIT_L1_LOAD    ? (Twin)l1_from_table<GSB_L1_UNIT_L1_LOAD>
                  : unit == GSB_L1_UNIT_L1_STORE ? (Twin)l1_from_table<GSB_L1_UNIT_L1_STORE>
                  : unit == GSB_L1_UNIT_NC       ? (Twin)l1_from_table<GSB_L1_UNIT_NC>
                  : unit == GSB_L1_UNIT_TEX      ? (Twin)l1_from_table<GSB_L1_UNIT_TEX>
                                                 : nullptr;
  // the buffer units ask for the largest L1, as the shipped kernels do
  if (fn) {
    const cudaError_t e = cudaFuncSetAttribute((const void *)fn, cudaFuncAttributePreferredSharedMemoryCarveout, 0);
    if (e != cudaSuccess) return (int)e;
  }
  switch (unit) {
    case GSB_L1_UNIT_L1_LOAD: l1_from_table<GSB_L1_UNIT_L1_LOAD><<<grid, GSB_L1_THREADS, 0, stream>>>(*a, *t); break;
    case GSB_L1_UNIT_L1_STORE: l1_from_table<GSB_L1_UNIT_L1_STORE><<<grid, GSB_L1_THREADS, 0, stream>>>(*a, *t); break;
    case GSB_L1_UNIT_NC: l1_from_table<GSB_L1_UNIT_NC><<<grid, GSB_L1_THREADS, 0, stream>>>(*a, *t); break;
    case GSB_L1_UNIT_TEX: l1_from_table<GSB_L1_UNIT_TEX><<<grid, GSB_L1_THREADS, 0, stream>>>(*a, *t); break;
    case GSB_L1_UNIT_CONST: {
      if (!bank) return (int)cudaErrorInvalidValue;
      const cudaError_t e = cudaMemcpyToSymbolAsync(gsb_l1_table_bank, bank, sizeof gsb_l1_table_bank, 0,
                                                    cudaMemcpyHostToDevice, stream);
      if (e != cudaSuccess) return (int)e;
      l1_from_table<GSB_L1_UNIT_CONST><<<grid, GSB_L1_THREADS, 0, stream>>>(*a, *t);
      break;
    }
    case GSB_L1_UNIT_PARAM:
      if (!param) return (int)cudaErrorInvalidValue;
      l1_from_table<GSB_L1_UNIT_PARAM>
          <<<grid, GSB_L1_THREADS, 0, stream>>>(*reinterpret_cast<const table_param *>(param), *a, *t);
      break;
    default: return (int)cudaErrorInvalidValue;
  }
  return (int)cudaGetLastError();
}
