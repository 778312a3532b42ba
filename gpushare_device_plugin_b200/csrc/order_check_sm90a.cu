/*
 * order_check_sm90a.cu — the memory-ordering check's kernel (gsb_order_probe): litmus tests of release/acquire,
 * fences and coherence at .gpu scope between SMs, through L2. Host code lives in gsb_device.cu (the probe) and
 * gsb_order.cc (conditions, text); the words, pairing and outcome classes are in gsb_order.h.
 *
 * One cooperative launch per (unit, distance), one CTA per SM: the kernel takes the device's opt-in maximum of dynamic
 * shared memory, more than half an SM's, so every CTA has an SM of its own and all of them are co-resident. Thread 0
 * plays the litmus role; warps 1-7 keep L2 busy with .cg loads and stores over the CTA's own scratch region until it
 * is done. Every shared location is one aligned u64 accessed with one instruction (single-copy atomic); a vector
 * access would be several accesses.
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "gsb_internal.h"
#include "gsb_order.h"

namespace {

constexpr unsigned kThreads = GSB_ORDER_THREADS;

__device__ __forceinline__ uint32_t smid() {
  uint32_t s;
  asm volatile("mov.u32 %0, %%smid;" : "=r"(s));
  return s;
}

__device__ __forceinline__ unsigned long long globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__device__ __forceinline__ void st_relaxed(unsigned long long *p, uint64_t v) {
  asm volatile("st.relaxed.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void st_release(unsigned long long *p, uint64_t v) {
  asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint64_t ld_relaxed(const unsigned long long *p) {
  uint64_t v;
  asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint64_t ld_acquire(const unsigned long long *p) {
  uint64_t v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void fence_acq_rel() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
__device__ __forceinline__ void fence_sc() { asm volatile("fence.sc.gpu;" ::: "memory"); }

// Arrive at the grid barrier and wait, for at most `wait_ns` of %globaltimer, until `target` CTAs have arrived: false
// when the bound ran out. Thread 0 only.
__device__ bool grid_barrier(unsigned int *counter, unsigned int target, unsigned long long wait_ns) {
  asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(counter) : "memory");
  const unsigned long long deadline = globaltimer() + wait_ns;
  for (;;) {
    unsigned int v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(counter) : "memory");
    if (v >= target) return true;
    if (globaltimer() > deadline) return false;
  }
}

// What thread 0 of one CTA tallies before it adds to the launch's log once.
struct Tally {
  unsigned long long words = 0, bad = 0, bits = 0, corrupt = 0, forbidden = 0, lost = 0, overlap = 0, weak = 0;
};

struct Litmus {
  const gsb_order_args &a;
  uint32_t sm, r, n;
  uint32_t ranks[3];
  int nr;
  Tally t;

  __device__ unsigned long long *loc(uint32_t rank, uint32_t slot) const {
    return a.locs + (size_t)rank * GSB_ORDER_LOC_WORDS + gsb_order_slot_word(slot);
  }

  // A record of a bad outcome: the consumer's %smid and those of the np ranks in prod whose stores its words show.
  __device__ __forceinline__ void record(uint32_t cls, uint32_t index, const uint64_t *w, uint32_t nw,
                                         const uint32_t *prod, int np) {
    if (sm < GSB_SM_MAX) atomicOr(&a.log->faulty[sm >> 5], 1u << (sm & 31u));
    const unsigned slot = atomicAdd(&a.log->count, 1u);
    if (slot >= GSB_ORDER_RECORDS) return;
    gsb_order_record &rec = a.log->rec[slot];
    rec.unit = a.unit;
    rec.distance = a.dist_index;
    rec.cls = cls;
    rec.smid = sm;
#pragma unroll
    for (int j = 0; j < 3; j++) rec.producer[j] = j < np ? a.smids[prod[j]] : GSB_SM_MAX;
    rec.index = index;
#pragma unroll
    for (uint32_t j = 0; j < GSB_ORDER_WORDS; j++) rec.words[j] = j < nw ? w[j] : 0ull;
  }

  // One observation's class into the tally, a record for a bad one.
  __device__ __forceinline__ void judge(uint32_t index, const uint32_t *keys, uint64_t *w, uint32_t iteration) {
    if (sm == a.inject_smid && index == a.inject_index)
      gsb_order_forbidden_words(a.unit, a.seed_expect, keys, iteration, w);  // test hook
    const uint32_t nw = gsb_order_obs_words(a.unit);
    const uint32_t cls = gsb_order_classify_words(a.unit, a.seed_expect, keys, w, iteration);
    switch (cls) {
      case GSB_ORDER_CLS_OVERLAP: t.overlap++; return;
      case GSB_ORDER_CLS_WEAK: t.weak++; return;
      case GSB_ORDER_CLS_FORBIDDEN: t.forbidden++; break;
      case GSB_ORDER_CLS_CORRUPT:
        t.corrupt++;
#pragma unroll
        for (uint32_t j = 0; j < GSB_ORDER_WORDS; j++)
          if (j < nw) t.bits += gsb_order_bad_bits(a.seed_expect, keys[j], w[j]);
        break;
      default: return;
    }
    t.bad++;
    // SB's words are this CTA's read of x_(r+d) and the partner r + d's read of x_r: the stores of r + d and of r
    const uint32_t sb[2] = {ranks[0], r};
    if (a.unit == GSB_ORDER_UNIT_SB_SC) record(cls, index, w, nw, sb, 2);
    else record(cls, index, w, nw, ranks, nr);
  }

  // MP_RELACQ, MP_FENCE and MP_RELAXED: store the own flag and data of iteration i, observe the producer's.
  template <uint32_t UNIT>
  __device__ void mp(bool skip) {
    const uint32_t m = a.observations;
    unsigned long long *own[GSB_ORDER_SLOTS], *src[GSB_ORDER_SLOTS];
    uint32_t own_key[GSB_ORDER_SLOTS], keys[GSB_ORDER_SLOTS];
#pragma unroll
    for (uint32_t s = 0; s < GSB_ORDER_SLOTS; s++) {
      own[s] = loc(r, s);
      src[s] = loc(ranks[0], s);
      own_key[s] = gsb_order_key(r, s);
      keys[s] = gsb_order_key(ranks[0], s);
    }
    for (uint32_t i = 1; i <= m; i++) {
      if (!skip) {
#pragma unroll
        for (uint32_t s = 1; s < GSB_ORDER_SLOTS; s++) st_relaxed(own[s], gsb_order_word(a.seed, own_key[s], i));
        if (UNIT == GSB_ORDER_UNIT_MP_RELACQ) {
          st_release(own[0], gsb_order_word(a.seed, own_key[0], i));
        } else {
          if (UNIT == GSB_ORDER_UNIT_MP_FENCE) fence_acq_rel();
          st_relaxed(own[0], gsb_order_word(a.seed, own_key[0], i));
        }
      }
      uint64_t w[GSB_ORDER_WORDS];
      if (UNIT == GSB_ORDER_UNIT_MP_RELACQ) {
        w[0] = ld_acquire(src[0]);
      } else {
        w[0] = ld_relaxed(src[0]);
        if (UNIT == GSB_ORDER_UNIT_MP_FENCE) fence_acq_rel();
      }
#pragma unroll
      for (uint32_t s = 1; s < GSB_ORDER_SLOTS; s++) w[s] = ld_relaxed(src[s]);
      judge(i - 1u, keys, w, i);
    }
  }

  __device__ void corr() {
    const uint32_t m = a.observations, own_key = gsb_order_key(r, 0), key = gsb_order_key(ranks[0], 0);
    unsigned long long *own = loc(r, 0), *src = loc(ranks[0], 0);
    const uint32_t keys[GSB_ORDER_WORDS] = {key, key, key, key, key};
    uint64_t prev = gsb_order_word(a.seed_expect, key, 0);
    for (uint32_t i = 1; i <= m; i++) {
      st_relaxed(own, gsb_order_word(a.seed, own_key, i));
      uint64_t w[GSB_ORDER_WORDS] = {prev, 0, 0, 0, 0};
      w[1] = ld_relaxed(src);
      w[2] = ld_relaxed(src);
      prev = w[2];
      judge(i - 1u, keys, w, i);
    }
  }

  // SB_SC: store x_r, fence.sc, read x_(r+d) and x_(r-d), fence.sc; the reads are published for the classification
  // after the barrier, where instance r takes CTA r + d's read of x_r.
  __device__ void sb() {
    const uint32_t m = a.observations, own_key = gsb_order_key(r, 0);
    unsigned long long *own = loc(r, 0), *fwd = loc(ranks[0], 0), *bwd = loc(ranks[1], 0);
    unsigned long long *obs = a.obs + (size_t)r * m * GSB_ORDER_OBS_WORDS;
    for (uint32_t i = 1; i <= m; i++) {
      st_relaxed(own, gsb_order_word(a.seed, own_key, i));
      fence_sc();
      const uint64_t f = ld_relaxed(fwd), b = ld_relaxed(bwd);
      fence_sc();
      obs[(size_t)(i - 1u) * GSB_ORDER_OBS_WORDS] = f;
      obs[(size_t)(i - 1u) * GSB_ORDER_OBS_WORDS + 1] = b;
    }
  }

  // IRIW_SC: store x_r; as reader A of instance r - 2e read x then y across fence.sc, as reader B of instance r - 3e
  // read its y then its x across fence.sc; published for the classification after the barrier.
  __device__ void iriw() {
    const uint32_t m = a.observations, own_key = gsb_order_key(r, 0);
    const uint32_t e = gsb_order_iriw_step(n, a.distance);
    unsigned long long *own = loc(r, 0), *x = loc(ranks[0], 0), *y = loc(ranks[1], 0);
    unsigned long long *bx = loc((r + 3u * n - 3u * e) % n, 0);
    unsigned long long *obs = a.obs + (size_t)r * m * GSB_ORDER_OBS_WORDS;
    for (uint32_t i = 1; i <= m; i++) {
      st_relaxed(own, gsb_order_word(a.seed, own_key, i));
      const uint64_t va = ld_relaxed(x);
      fence_sc();
      const uint64_t vb = ld_relaxed(y);
      const uint64_t vc = ld_relaxed(x);  // reader B's y is this CTA's x
      fence_sc();
      const uint64_t vd = ld_relaxed(bx);
      unsigned long long *o = obs + (size_t)(i - 1u) * GSB_ORDER_OBS_WORDS;
      o[0] = va;
      o[1] = vb;
      o[2] = vc;
      o[3] = vd;
    }
  }

  // After the barrier: SB's and IRIW's observations, each with its partner's half.
  __device__ void classify_published() {
    const uint32_t m = a.observations;
    const unsigned long long *mine = a.obs + (size_t)r * m * GSB_ORDER_OBS_WORDS;
    const unsigned long long *other =
        a.obs + (size_t)(a.unit == GSB_ORDER_UNIT_SB_SC ? ranks[0] : ranks[2]) * m * GSB_ORDER_OBS_WORDS;
    uint32_t keys[GSB_ORDER_WORDS] = {0, 0, 0, 0, 0};
    if (a.unit == GSB_ORDER_UNIT_SB_SC) {
      keys[0] = gsb_order_key(ranks[0], 0);
      keys[1] = gsb_order_key(r, 0);
    } else {
      keys[0] = keys[3] = gsb_order_key(ranks[0], 0);
      keys[1] = keys[2] = gsb_order_key(ranks[1], 0);
    }
    for (uint32_t k = 0; k < m; k++) {
      const unsigned long long *p = mine + (size_t)k * GSB_ORDER_OBS_WORDS, *q = other + (size_t)k * GSB_ORDER_OBS_WORDS;
      uint64_t w[GSB_ORDER_WORDS] = {0, 0, 0, 0, 0};
      if (a.unit == GSB_ORDER_UNIT_SB_SC) {
        w[0] = p[0];
        w[1] = q[1];  // the partner's read of x_r
      } else {
        w[0] = p[0];
        w[1] = p[1];
        w[2] = q[2];  // the other reader's c = ld y, d = ld x
        w[3] = q[3];
      }
      judge(k, keys, w, k + 1u);
    }
  }

  // After the barrier: every location the observations read, once more; it must hold the writer's last iteration.
  __device__ void final_reads() {
    const uint32_t nf = gsb_order_final_reads(a.unit);
#pragma unroll
    for (uint32_t j = 0; j < GSB_ORDER_SLOTS; j++) {
      if (j >= nf) break;
      const uint32_t rank = a.unit == GSB_ORDER_UNIT_IRIW_SC ? ranks[j] : ranks[0];
      const uint32_t slot = a.unit == GSB_ORDER_UNIT_IRIW_SC ? 0u : j, key = gsb_order_key(rank, slot);
      uint64_t w = ld_relaxed(loc(rank, slot));
      const uint32_t cls = gsb_order_final(a.seed_expect, key, w, a.observations);
      if (cls == GSB_ORDER_CLS_ALLOWED) continue;
      if (cls == GSB_ORDER_CLS_LOST) t.lost++;
      else {
        t.corrupt++;
        t.bits += gsb_order_bad_bits(a.seed_expect, key, w);
      }
      t.bad++;
      record(cls, j, &w, 1, &rank, 1);
    }
  }
};

__global__ void __launch_bounds__(kThreads, 1) order_check(const gsb_order_args a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];  // only to keep a second CTA off the SM
  volatile unsigned int *done = reinterpret_cast<volatile unsigned int *>(smem_raw);
  const uint32_t sm = smid(), r = blockIdx.x, n = gridDim.x;
  if (threadIdx.x == 0) {
    *done = 0u;
    a.smids[r] = sm;
    if (sm < GSB_SM_MAX) atomicOr(&a.log->covered[sm >> 5], 1u << (sm & 31u));
    unsigned long long *blk = a.locs + (size_t)r * GSB_ORDER_LOC_WORDS;
#pragma unroll
    for (uint32_t s = 0; s < GSB_ORDER_SLOTS; s++)
      st_relaxed(blk + gsb_order_slot_word(s), gsb_order_word(a.seed, gsb_order_key(r, s), 0u));
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    Litmus L{a, sm, r, n, {0, 0, 0}, 0, {}};
    L.nr = gsb_order_pairing_of(a.unit, n, a.distance, r, L.ranks);
    bool on_time = L.nr > 0 && grid_barrier(&a.log->barrier, n, GSB_ORDER_WAIT_NS);
    if (on_time) {
      const bool skip = a.unit == GSB_ORDER_UNIT_MP_RELACQ && sm == a.skip_smid;
      switch (a.unit) {
        case GSB_ORDER_UNIT_MP_RELACQ: L.mp<GSB_ORDER_UNIT_MP_RELACQ>(skip); break;
        case GSB_ORDER_UNIT_MP_FENCE: L.mp<GSB_ORDER_UNIT_MP_FENCE>(false); break;
        case GSB_ORDER_UNIT_MP_RELAXED: L.mp<GSB_ORDER_UNIT_MP_RELAXED>(false); break;
        case GSB_ORDER_UNIT_SB_SC: L.sb(); break;
        case GSB_ORDER_UNIT_IRIW_SC: L.iriw(); break;
        default: L.corr(); break;
      }
      L.t.words += (unsigned long long)gsb_order_reads(a.unit) * a.observations;
    }
    // the second barrier: every store of every CTA is in before the final reads and the published observations
    // Its bound also absorbs how far the slowest CTA's litmus loop trails this one's, which grows with observations.
    on_time = grid_barrier(&a.log->barrier, 2u * n, gsb_order_wait_ns(a.observations)) && on_time;
    *done = 1u;
    __threadfence_block();
    if (on_time) {
      if (a.unit == GSB_ORDER_UNIT_SB_SC || a.unit == GSB_ORDER_UNIT_IRIW_SC) L.classify_published();
      L.final_reads();
      L.t.words += gsb_order_final_reads(a.unit);
    }
    gsb_order_log *log = a.log;
    atomicAdd(&log->words, L.t.words);
    if (L.t.bad) atomicAdd(&log->mismatch_words, L.t.bad);
    if (L.t.bits) atomicAdd(&log->mismatch_bits, L.t.bits);
    if (L.t.corrupt) atomicAdd(&log->corrupt, L.t.corrupt);
    if (L.t.forbidden) atomicAdd(&log->forbidden, L.t.forbidden);
    if (L.t.lost) atomicAdd(&log->lost, L.t.lost);
    if (L.t.overlap) atomicAdd(&log->overlap, L.t.overlap);
    if (L.t.weak) atomicAdd(&log->weak, L.t.weak);
    if (!on_time) atomicAdd(&log->timeout, 1ull);
  } else if (threadIdx.x >= 32) {
    // stress: .cg loads and stores of the CTA's own scratch region until the litmus thread is done (not judged)
    uint4 *reg = a.scratch + (size_t)r * GSB_ORDER_SCRATCH_WORDS;
    const unsigned long long deadline =
        globaltimer() + 2ull * (GSB_ORDER_WAIT_NS + gsb_order_wait_ns(a.observations)) + 1000000000ull;
    uint32_t it = 0;
    for (uint32_t w = threadIdx.x - 32u; !*done; w += kThreads - 32u, it++) {
      uint4 *p = reg + w % GSB_ORDER_SCRATCH_WORDS;
      uint4 v;
      asm volatile("ld.global.cg.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
      asm volatile("st.global.cg.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x + 1u), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
      if ((it & 0xFFu) == 0u && globaltimer() > deadline) break;
    }
  }
  __syncthreads();
}

}  // namespace

int gsb_order_kernel_launch(uint32_t grid, const gsb_order_args *a, cudaStream_t stream) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kThreads);
  cfg.dynamicSmemBytes = a->smem_bytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, order_check, *a);
  // not all CTAs can be resident at once (another context holds SMs): the caller skips the launch, so it must not
  // stay this module's runtime's last error
  if (e == cudaErrorCooperativeLaunchTooLarge) cudaGetLastError();
  return (int)e;
}

int gsb_order_kernel_preload(int smem_bytes) {
  return (int)cudaFuncSetAttribute((const void *)order_check, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
}
