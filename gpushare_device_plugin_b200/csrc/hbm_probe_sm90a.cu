/*
 * hbm_probe_sm90a.cu — the per-device HBM probe kernels (sm_90a only).
 *
 * Replaces the reference's passive health half — nvml.WaitForEvent in watchXIDs
 * (pkg/gpu/nvidia/nvidia.go:100-152), which never touches HBM — with an active walk of the arena:
 * every 16-byte word of the window is loaded once (compared with the pattern of the generation
 * that last wrote it) and stored once (the next generation's pattern). Algorithmic traffic of a
 * VERIFY_REFILL launch = 2 * window bytes (SURVEY.md §8(d)); bound = HBM bandwidth. Integer only,
 * no tensor cores (this is not a contraction).
 *
 * Three data paths, same results bit for bit (tests/test_probe_gpu.py):
 *   DIRECT   ld.global.v4 -> registers -> st.global.v4          (control: no staging)
 *   CPASYNC  cp.async 16 B (LDGSTS) -> shared ring -> ld.shared.v4 -> st.global.v4
 *   BULK     cp.async.bulk (TMA 1-D, UBLKCP) + mbarrier -> shared ring -> ld.shared.v4 /
 *            st.shared.v4 -> cp.async.bulk shared->global
 * All are persistent kernels over fixed-size tiles, grid = resident CTAs/SM x #SMs.
 *
 * Kernels: the two GSB_VARIANT_AUTO launches — BULKD (FILL, VERIFY_REFILL) and BULK (VERIFY), 32 KiB x 3 stages —
 * plus one shape each of DIRECT, CPASYNC and BULKW, kept as independent data paths for the parity tests (five
 * implementations, one answer). BULK, BULKD and BULKW run one TMA ring protocol (bulk_ring): one ring per CTA with a
 * static or a claimed tile schedule, or, for BULKW, one ring per warp with the static schedule. Every shape is fixed
 * at compile time; the H100 tile-shape sweep behind the BULK / BULKD shape is in DESIGN.md §5. The BULKD refill runs
 * as a verify pass over the whole window and then a write pass, in one launch (HBM serves that faster than reads and
 * writes to the same rows at once); the other refills walk the window in place, each tile loaded and then stored.
 *
 * Reduction: per-thread registers -> warp shuffles -> one gsb_partial slot per CTA (plain stores,
 * no atomics on the data path) -> a self-resetting ticket elects the last CTA, which folds all
 * slots into the pinned host-mapped gsb_kernel_out. Checksums are XOR / wrapping-add, so the
 * result does not depend on CTA scheduling order.
 *
 * Fault log (cold path, see "fault log" below): a mismatching word also counts its flipped bit positions in a per-CTA
 * shared histogram and, while there is room, records itself in the device's fault log; the last CTA of a faulted
 * launch copies the log next to gsb_kernel_out and empties it. A clean launch pays one zeroed shared histogram per CTA.
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "gsb_internal.h"
#include "gsb_pattern.h"

namespace {

constexpr int kThreads = 256;
constexpr int kMaxWarps = 16;
constexpr unsigned long long kNoBad = ~0ull;

struct Acc {
  uint32_t mm_words = 0, mm_bits = 0, cxor = 0, csum = 0, words = 0;
  unsigned long long first_bad = kNoBad;
};

// ---------------------------------------------------------------- memory-op helpers (PTX)

__device__ __forceinline__ uint4 ld_stream(const uint4 *p) {
  uint4 v;
  asm volatile("ld.global.cs.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ void st_stream(uint4 *p, const uint4 v) {
  asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}
// A refill stores to the address it has just loaded from, and the stored value (the next generation's pattern) does
// not depend on the loaded one. Left alone, the four stores of a thread issue right behind its four loads, while
// those loads are still in flight, and the memory system then orders every same-line load/store pair one at a time,
// a fraction of the bandwidth VERIFY or FILL alone reach. tools/lab/direct_anomaly.cu isolates it: the same in-place
// walk runs near the copy peak when the stored value really depends on the loaded one or when the store trails its
// load by a tile, and far below it when it does not. Naming the loaded register as an input of an EMPTY inline-asm
// statement does nothing: a comment is not an instruction, so the dependency is gone before ptxas schedules the store.
// A real one costs two integer ops per word: the loaded lanes are AND-ed with a kernel argument that is always 0 (the
// compiler cannot know) and XOR-ed into the value to store.
__device__ __forceinline__ uint4 after_load(uint4 nw, uint32_t loaded, uint32_t opaque_zero) {
  nw.x ^= loaded & opaque_zero;
  return nw;
}
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void cp_async16(uint32_t dst_smem, const void *src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst_smem), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(bar),
      "r"(parity)
      : "memory");
}
// TMA 1-D bulk copy global -> shared, completion signalled on an mbarrier (SASS: UBLKCP)
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void *src, uint32_t bytes, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem),
      "l"(src), "r"(bytes), "r"(bar)
      : "memory");
}
// TMA 1-D bulk copy shared -> global, tracked by the thread's bulk async-group
__device__ __forceinline__ void bulk_s2g(void *dst, uint32_t src_smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(src_smem),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait_all() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ unsigned long long globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// ---------------------------------------------------------------- pattern + compare

__device__ __forceinline__ uint4 pattern_from_key(uint32_t m, uint32_t seed_key) {
  uint4 p;
  p.x = (m * GSB_PAT_K0 + GSB_PAT_C0) ^ seed_key;
  p.y = (m * GSB_PAT_K1 + GSB_PAT_C1) ^ seed_key;
  p.z = (m * GSB_PAT_K2 + GSB_PAT_C2) ^ seed_key;
  p.w = (m * GSB_PAT_K3 + GSB_PAT_C3) ^ seed_key;
  return p;
}

__device__ __forceinline__ void fold_checksum(const uint4 v, Acc &acc) {
  acc.cxor ^= v.x ^ v.y ^ v.z ^ v.w;
  acc.csum += v.x + v.y + v.z + v.w;
}

// ---------------------------------------------------------------- fault log (cold path)
//
// What a mismatching word leaves behind besides the three counters: its flipped bit positions in a per-CTA shared
// histogram (one shared atomic per flipped bit, so an all-wrong window costs what its flipped bits cost, never a global
// atomic per bit), and, while the device log has room, one record {word, observed, expected}. A CTA that saw a
// mismatch folds its histogram into the device log once, in finish(); the last CTA of a faulted launch copies the log
// to the host and empties it. A clean launch runs none of this beyond zeroing the shared histogram.

constexpr unsigned kFaultRecords = GSB_FAULT_RECORDS;

struct FaultSmem {
  uint32_t flips[2][128];  // [expected bit][32 * lane + bit]
  uint32_t log_full;       // this CTA has seen the device log full: claim no more slots
};
__shared__ FaultSmem fault_smem;

// every thread, before the CTA's first barrier
__device__ __forceinline__ void fault_smem_init() {
  uint32_t *h = &fault_smem.flips[0][0];
  for (unsigned i = threadIdx.x; i < 256u; i += blockDim.x) h[i] = 0u;
  if (threadIdx.x == 0) fault_smem.log_full = 0u;
}

__device__ __forceinline__ void record_fault(const uint4 v, const uint4 e, unsigned long long w, gsb_fault_log *log) {
  const uint32_t ov[4] = {v.x, v.y, v.z, v.w}, ev[4] = {e.x, e.y, e.z, e.w};
#pragma unroll
  for (int l = 0; l < 4; l++) {
    for (uint32_t d = ov[l] ^ ev[l]; d != 0u; d &= d - 1u) {
      const int b = __ffs(d) - 1;
      atomicAdd(&fault_smem.flips[(ev[l] >> b) & 1u][32 * l + b], 1u);
    }
  }
  // once the log is full no more atomics go to its counter: this CTA remembers it in shared memory
  volatile uint32_t *full = &fault_smem.log_full;
  if (*full) return;
  if (__ldcg(&log->count) >= kFaultRecords) {
    *full = 1u;
    return;
  }
  const unsigned slot = atomicAdd(&log->count, 1u);
  if (slot >= kFaultRecords) {
    *full = 1u;
    return;
  }
  gsb_fault_word &r = log->rec[slot];
  r.word = w;
#pragma unroll
  for (int l = 0; l < 4; l++) {
    r.observed[l] = ov[l];
    r.expected[l] = ev[l];
  }
}

__device__ __forceinline__ void compare_word(const uint4 v, const uint4 e, unsigned long long w, Acc &acc,
                                             gsb_fault_log *log) {
  const uint32_t dx = v.x ^ e.x, dy = v.y ^ e.y, dz = v.z ^ e.z, dw = v.w ^ e.w;
  if ((dx | dy | dz | dw) != 0u) {  // cold path: a healthy device never takes it
    acc.mm_words += 1u;
    acc.mm_bits += __popc(dx) + __popc(dy) + __popc(dz) + __popc(dw);
    acc.first_bad = w < acc.first_bad ? w : acc.first_bad;
    record_fault(v, e, w, log);
  }
}

// expected-seed key of the tile starting at absolute word w (tiles never straddle a granule when a
// table is in use: the shim enforces 64 KiB window alignment and granules are 64 MiB)
__device__ __forceinline__ uint32_t expect_key_of(const gsb_kernel_args &a, unsigned long long w) {
  const uint32_t s = a.seed_table ? __ldg(a.seed_table + (w >> a.granule_shift)) : a.seed_expect;
  return gsb_seed_key(s);
}

// What is done to one word, as compile-time flags:
//   kRead         `v` is the loaded word: fold it into the checksums and compare it with the expected pattern
//   kWrite        return the next generation's word (otherwise the return value is undefined)
//   kFoldWritten  fold the returned word into the checksums (FILL, which reads nothing)
//   kCount        count the word in words_done
constexpr unsigned kRead = 1u, kWrite = 2u, kFoldWritten = 4u, kCount = 8u;

// the flags of a launch that does OP (a compile-time GSB_OP_*) to every word once
__host__ __device__ constexpr unsigned op_words(int op) {
  return op == GSB_OP_FILL     ? kWrite | kFoldWritten | kCount
         : op == GSB_OP_VERIFY ? kRead | kCount
                               : kRead | kWrite | kCount;
}

template <unsigned F>
__device__ __forceinline__ uint4 process_word(const gsb_kernel_args &a, const uint4 v, unsigned long long w,
                                              uint32_t key_expect, uint32_t key_write, Acc &acc) {
  const uint32_t m = gsb_word_key(w);
  uint4 nw = make_uint4(0, 0, 0, 0);
  if (F & kRead) {
    fold_checksum(v, acc);
    compare_word(v, pattern_from_key(m, key_expect), w, acc, a.fault);
  }
  if (F & kWrite) {
    nw = pattern_from_key(m, key_write);
    if (F & kFoldWritten) fold_checksum(nw, acc);
  }
  if (F & kCount) acc.words += 1u;
  return nw;
}

// ---------------------------------------------------------------- CTA epilogue

__device__ __forceinline__ void warp_fold(gsb_partial &p) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    p.mismatch_words += __shfl_xor_sync(0xffffffffu, p.mismatch_words, off);
    p.mismatch_bits += __shfl_xor_sync(0xffffffffu, p.mismatch_bits, off);
    p.words += __shfl_xor_sync(0xffffffffu, p.words, off);
    const unsigned long long o = __shfl_xor_sync(0xffffffffu, p.first_bad_word, off);
    p.first_bad_word = o < p.first_bad_word ? o : p.first_bad_word;
    p.checksum_xor ^= __shfl_xor_sync(0xffffffffu, p.checksum_xor, off);
    p.checksum_sum += __shfl_xor_sync(0xffffffffu, p.checksum_sum, off);
  }
}

__device__ __forceinline__ void merge(gsb_partial &d, const gsb_partial &s) {
  d.mismatch_words += s.mismatch_words;
  d.mismatch_bits += s.mismatch_bits;
  d.words += s.words;
  d.first_bad_word = s.first_bad_word < d.first_bad_word ? s.first_bad_word : d.first_bad_word;
  d.checksum_xor ^= s.checksum_xor;
  d.checksum_sum += s.checksum_sum;
}

__device__ __forceinline__ gsb_partial block_fold(gsb_partial p, gsb_partial *wslots) {
  warp_fold(p);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int n_warps = (int)(blockDim.x >> 5);
  if (lane == 0) wslots[warp] = p;
  __syncthreads();
  gsb_partial r = wslots[0];
  if (threadIdx.x == 0) {
    for (int i = 1; i < n_warps; i++) merge(r, wslots[i]);
  }
  return r;  // valid in thread 0
}

__device__ __forceinline__ gsb_partial ld_partial_cg(const gsb_partial *p) {
  gsb_partial r;
  r.mismatch_words = __ldcg(&p->mismatch_words);
  r.mismatch_bits = __ldcg(&p->mismatch_bits);
  r.first_bad_word = __ldcg(&p->first_bad_word);
  r.words = __ldcg(&p->words);
  r.checksum_xor = __ldcg(&p->checksum_xor);
  r.checksum_sum = __ldcg(&p->checksum_sum);
  return r;
}

// after block_fold, in every thread: did any warp of the fold see a mismatch (uniform across the CTA)
__device__ __forceinline__ bool fold_saw_mismatch(const gsb_partial *wslots) {
  const int n_warps = (int)(blockDim.x >> 5);
  unsigned long long any = 0;
  for (int i = 0; i < n_warps; i++) any |= wslots[i].mismatch_words;
  return any != 0;
}

// a CTA that saw a mismatch: its shared histogram -> the device log (one global atomic per non-zero position)
__device__ __forceinline__ void fold_fault_hist(gsb_fault_log *log) {
  const uint32_t *h = &fault_smem.flips[0][0];
  unsigned long long *g = &log->flips[0][0];
  for (unsigned i = threadIdx.x; i < 256u; i += blockDim.x)
    if (h[i]) atomicAdd(g + i, (unsigned long long)h[i]);
  __threadfence();  // before thread 0's ticket: the last CTA must see these
}

// last CTA of a faulted launch, every thread: device log -> mapped host copy, then empty the device log
__device__ __forceinline__ void publish_faults(gsb_fault_log *log, gsb_fault_log *out, uint32_t launch_seq) {
  const unsigned claimed = __ldcg(&log->count);
  const unsigned n = claimed < kFaultRecords ? claimed : kFaultRecords;
  unsigned long long *g = &log->flips[0][0], *o = &out->flips[0][0];
  for (unsigned i = threadIdx.x; i < 256u; i += blockDim.x) {
    o[i] = __ldcg(g + i);
    g[i] = 0ull;
  }
  constexpr unsigned kRecWords = sizeof(gsb_fault_word) / sizeof(uint32_t);
  const uint32_t *rs = reinterpret_cast<const uint32_t *>(log->rec);
  uint32_t *rd = reinterpret_cast<uint32_t *>(out->rec);
  for (unsigned i = threadIdx.x; i < n * kRecWords; i += blockDim.x) rd[i] = __ldcg(rs + i);
  __syncthreads();  // every thread has read the count
  if (threadIdx.x == 0) {
    log->count = 0u;
    out->count = n;
    out->launch_seq = launch_seq;
  }
  __threadfence_system();
}

__device__ void finish(const gsb_kernel_args &a, const Acc &acc) {
  __shared__ gsb_partial wslots[kMaxWarps];
  __shared__ int is_last;
  gsb_partial p;
  p.mismatch_words = acc.mm_words;
  p.mismatch_bits = acc.mm_bits;
  p.first_bad_word = acc.first_bad;
  p.words = acc.words;
  p.checksum_xor = acc.cxor;
  p.checksum_sum = acc.csum;
  gsb_partial cta = block_fold(p, wslots);
  if (fold_saw_mismatch(wslots)) {  // cold: a clean CTA pays only the n_warps shared loads above
    fold_fault_hist(a.fault);
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    a.partials[blockIdx.x] = cta;
    __threadfence();
    const unsigned prev = atomicAdd(a.ticket, 1u);
    is_last = (prev == gridDim.x - 1u);
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  gsb_partial t;
  t.mismatch_words = 0;
  t.mismatch_bits = 0;
  t.first_bad_word = kNoBad;
  t.words = 0;
  t.checksum_xor = 0;
  t.checksum_sum = 0;
  for (unsigned i = threadIdx.x; i < gridDim.x; i += blockDim.x) merge(t, ld_partial_cg(a.partials + i));
  __syncthreads();  // wslots reuse
  gsb_partial all = block_fold(t, wslots);
  if (fold_saw_mismatch(wslots)) {  // every other CTA has folded its histogram and written its records
    publish_faults(a.fault, a.fault_out, a.launch_seq);
    __syncthreads();  // the host copy is complete before done_flag says the launch is
  }
  if (a.table_update) {
    // every other CTA has finished: record the generation now held by each granule this window
    // covered completely (plus the arena's ragged tail granule when the window reaches the end)
    const unsigned long long gw = 1ull << a.granule_shift;
    const unsigned long long end = a.first_word + a.n_words;
    const unsigned long long g0 = (a.first_word + gw - 1) >> a.granule_shift;
    unsigned long long g1 = end >> a.granule_shift;
    if (end == a.arena_words && (a.arena_words & (gw - 1))) g1 += 1;
    for (unsigned long long g = g0 + threadIdx.x; g < g1; g += blockDim.x) a.table_update[g] = a.seed_write;
  }
  if (threadIdx.x == 0) {
    *a.ticket = 0u;  // self-reset: the next launch on this stream starts from 0
    if (a.tile_counter) a.tile_counter[0] = a.tile_counter[1] = 0ull;  // every other CTA is past the refill's gate
    gsb_kernel_out *o = a.out;
    o->mismatch_words = all.mismatch_words;
    o->mismatch_bits = all.mismatch_bits;
    o->first_bad_word = all.first_bad_word;
    o->checksum_xor = all.checksum_xor;
    o->checksum_sum = all.checksum_sum;
    o->words_done = all.words;
    __threadfence_system();
    o->done_flag = a.launch_seq;
  }
}

// ---------------------------------------------------------------- DIRECT

template <int OP, int U>
__global__ void __launch_bounds__(kThreads) probe_direct(const gsb_kernel_args a) {
  constexpr unsigned long long TILE = (unsigned long long)kThreads * U;
  const unsigned long long n_tiles = (a.n_words + TILE - 1) / TILE;
  const uint32_t key_write = gsb_seed_key(a.seed_write);
  uint4 *__restrict__ win = a.base + a.first_word;
  Acc acc;
  fault_smem_init();
  __syncthreads();
  for (unsigned long long t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    const unsigned long long l0 = t * TILE + threadIdx.x;
    const uint32_t key_expect = (OP != GSB_OP_FILL) ? expect_key_of(a, a.first_word + t * TILE) : 0u;
    uint4 v[U];
    if ((t + 1) * TILE <= a.n_words) {
      if (OP != GSB_OP_FILL) {
#pragma unroll
        for (int u = 0; u < U; u++) v[u] = ld_stream(win + l0 + (unsigned long long)u * kThreads);
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
        const unsigned long long l = l0 + (unsigned long long)u * kThreads;
        uint4 nw = process_word<op_words(OP)>(a, v[u], a.first_word + l, key_expect, key_write, acc);
        if (OP == GSB_OP_VERIFY_REFILL) nw = after_load(nw, v[u].x ^ v[u].y ^ v[u].z ^ v[u].w, a.opaque_zero);
        if (OP != GSB_OP_VERIFY) st_stream(win + l, nw);
      }
    } else {  // ragged last tile
#pragma unroll
      for (int u = 0; u < U; u++) {
        const unsigned long long l = l0 + (unsigned long long)u * kThreads;
        if (l < a.n_words) {
          if (OP != GSB_OP_FILL) v[u] = ld_stream(win + l);
          uint4 nw = process_word<op_words(OP)>(a, v[u], a.first_word + l, key_expect, key_write, acc);
          if (OP == GSB_OP_VERIFY_REFILL) nw = after_load(nw, v[u].x ^ v[u].y ^ v[u].z ^ v[u].w, a.opaque_zero);
          if (OP != GSB_OP_VERIFY) st_stream(win + l, nw);
        }
      }
    }
  }
  finish(a, acc);
}

// ---------------------------------------------------------------- CPASYNC (LDGSTS ring)

template <int OP, int U, int S>
__global__ void __launch_bounds__(kThreads) probe_cpasync(const gsb_kernel_args a) {
  static_assert(OP != GSB_OP_FILL, "FILL has no loads to stage");
  constexpr unsigned long long TILE = (unsigned long long)kThreads * U;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  uint4 *ring = reinterpret_cast<uint4 *>(smem_raw);  // [S][TILE]
  const unsigned long long n_tiles = (a.n_words + TILE - 1) / TILE;
  const unsigned long long my_n =
      n_tiles > blockIdx.x ? (n_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0ull;
  const uint32_t key_write = gsb_seed_key(a.seed_write);
  uint4 *__restrict__ win = a.base + a.first_word;
  Acc acc;
  fault_smem_init();
  __syncthreads();

  auto issue = [&](unsigned long long k) {
    if (k < my_n) {
      const unsigned long long t = blockIdx.x + k * gridDim.x;
      const int s = (int)(k % S);
#pragma unroll
      for (int u = 0; u < U; u++) {
        const unsigned long long l = t * TILE + (unsigned long long)u * kThreads + threadIdx.x;
        if (l < a.n_words) cp_async16(smem_u32(ring + s * TILE + u * kThreads + threadIdx.x), win + l);
      }
    }
    cp_async_commit();  // always commit: keeps the group count uniform
  };

#pragma unroll
  for (int k = 0; k < S - 1; k++) issue(k);
  for (unsigned long long k = 0; k < my_n; k++) {
    issue(k + S - 1);
    cp_async_wait<S - 1>();  // tile k's copies (this thread's own 16 B slots) have landed
    const unsigned long long t = blockIdx.x + k * gridDim.x;
    const int s = (int)(k % S);
    const uint32_t key_expect = expect_key_of(a, a.first_word + t * TILE);
#pragma unroll
    for (int u = 0; u < U; u++) {
      const unsigned long long l = t * TILE + (unsigned long long)u * kThreads + threadIdx.x;
      if (l < a.n_words) {
        // each thread reads back only the slots it copied itself: no CTA barrier needed
        const uint4 v = ring[s * TILE + u * kThreads + threadIdx.x];
        const uint4 nw = process_word<op_words(OP)>(a, v, a.first_word + l, key_expect, key_write, acc);
        if (OP != GSB_OP_VERIFY) st_stream(win + l, nw);
      }
    }
  }
  cp_async_wait<0>();
  finish(a, acc);
}

// ---------------------------------------------------------------- BULK / BULKD / BULKW (TMA 1-D rings)
//
// A CTA runs RINGS rings: one for BULK and BULKD, one per warp for BULKW. Ring r has its own S stages of TILE words
// and its own mbarriers. Its leader (its first thread) starts the bulk load of slot k into stage k % S and completes
// it on the stage's mbarrier; the ring's threads process the tile in shared memory; the leader writes it back with a
// bulk store. A per-warp ring synchronises with __syncwarp only, so a warp waiting on HBM never holds the CTA's other
// warps at a barrier. Which tile slot k holds is the schedule's business; the schedule is a template argument, so
// nothing that differs between the two is decided at run time. Each schedule is built with its ring's index:
//   has(k)      slot k is issued at all: the loop stops before waiting on a slot whose load was never issued
//   next(k, s)  leader, once per slot in slot order: the tile slot k (stage s) holds, or the end of the walk
//   tile(k, s)  every thread of the ring, after slot k's barrier: the same tile
//   done(t)     t is the end of the walk
//   kPasses     1: every slot does OP to its tile; 2 (refill only): a slot tile t < n_tiles is verified, and
//               n_tiles + t writes tile t (the refill's two passes, below)

// BULK (RINGS = 1) and BULKW: ring r's slot k holds tile (blockIdx + k * grid) * RINGS + r while k < my_n, so the rings
// of a CTA take adjacent tiles, which keeps DRAM pages hot; every thread computes it.
template <int RINGS>
struct StaticSchedule {
  static constexpr int kPasses = 1;
  unsigned long long first, my_n;
  __device__ StaticSchedule(const gsb_kernel_args &, unsigned long long n_tiles, int r, unsigned long long *)
      : first((unsigned long long)blockIdx.x * RINGS + r) {
    const unsigned long long stride = (unsigned long long)gridDim.x * RINGS;
    my_n = n_tiles > first ? (n_tiles - first + stride - 1) / stride : 0ull;
  }
  __device__ bool has(unsigned long long k) const { return k < my_n; }
  __device__ unsigned long long next(unsigned long long k, int s) const { return tile(k, s); }
  __device__ unsigned long long tile(unsigned long long k, int) const { return first + k * gridDim.x * RINGS; }
  __device__ static bool done(unsigned long long) { return false; }
};

// BULKD: the leader claims the next tile from an atomic counter when it issues a slot, so CTAs that run ahead simply
// take more tiles and the kernel ends with every CTA busy (no straggler tail). Claims are made in time order, so
// concurrently processed tiles stay neighbours in memory. The claimed index travels to the consumers through
// tile_of[s] under the stage's mbarrier (arrive = release, wait = acquire); every slot is issued, and the first one
// past the last claim holds kDone. With two passes the counter runs over 2 * n_tiles claims, so claims are monotone:
// inside one CTA every slot of the verify pass comes before every slot of the write pass. The schedule is CTA-wide
// (RINGS = 1): its leader is thread 0, and the ring index is always 0.
template <int PASSES>
struct ClaimedSchedule {
  static constexpr int kPasses = PASSES;
  static constexpr unsigned long long kDone = ~0ull;
  unsigned long long n_claims, in_hand = 0;
  unsigned long long *counter, *tile_of;
  __device__ ClaimedSchedule(const gsb_kernel_args &a, unsigned long long n, int, unsigned long long *slots)
      : n_claims(PASSES * n), counter(a.tile_counter), tile_of(slots) {
    // the leader always holds one claim in hand: the atomic for the NEXT tile is issued when the current one is
    // consumed, so its ~L2 round trip overlaps the tile being processed instead of delaying the next load
    if (threadIdx.x == 0) in_hand = atomicAdd(counter, 1ull);
  }
  __device__ bool has(unsigned long long) const { return true; }
  __device__ unsigned long long next(unsigned long long, int s) {
    const unsigned long long t = in_hand;
    in_hand = atomicAdd(counter, 1ull);
    return tile_of[s] = t < n_claims ? t : kDone;
  }
  __device__ unsigned long long tile(unsigned long long, int s) const { return tile_of[s]; }
  __device__ static bool done(unsigned long long t) { return t == kDone; }
};

// The refill's two passes. A refill stores the next generation's pattern, which depends on the address and the seed
// only, so the window can be verified completely and then written completely: same memory image, same results, same
// 2 * W bytes. HBM serves a read pass and a write pass faster than it serves reads and writes to the same rows at
// once (DESIGN.md §5). One rule keeps it correct: the store of tile t must not reach HBM while another CTA's bulk load
// of tile t may still be reading it. So each CTA adds the verify tiles it has consumed (past their mbarrier) to the
// launch's count, tile_counter[1], once, when it leaves the verify pass: at its first write slot or at the end of the
// walk. A CTA with tiles to write then waits, before it writes any, until the count reaches n_tiles; it waits when it
// consumes its first write slot, never when its leader claims or issues one, since the leader is a consumer too. This
// cannot deadlock whatever the residency: verify tiles are claimed only by running CTAs, and such a CTA waits on
// nothing but its own loads until it has added its count. The wait is bounded: a CTA that has waited kGateTimeoutNs
// drops its write tiles, so words_done falls short of n_words and the host reports the launch as failed instead of
// the GPU spinning for ever.
constexpr unsigned long long kGateTimeoutNs = 1000000000ull;

// leader, once per CTA; false: the gate did not open in time
__device__ __forceinline__ bool leave_verify_pass(unsigned long long *verified, unsigned long long mine,
                                                  unsigned long long n_tiles, bool will_write) {
  asm volatile("red.release.gpu.global.add.u64 [%0], %1;" ::"l"(verified), "l"(mine) : "memory");
  if (!will_write) return true;
  const unsigned long long t0 = globaltimer();
  for (;;) {
    unsigned long long seen;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(seen) : "l"(verified) : "memory");
    if (seen >= n_tiles) break;
    if (globaltimer() - t0 > kGateTimeoutNs) return false;
    __nanosleep(64);
  }
  asm volatile("fence.proxy.async.global;" ::: "memory");  // the bulk stores that follow come after the acquire
  return true;
}

// one ring thread's words of a staged tile: n words from absolute word w0, the thread's words i = u * T + rt;
// F says what is done to each (process_word)
template <unsigned F, int U, int T>
__device__ __forceinline__ void process_stage(const gsb_kernel_args &a, uint4 *stage, unsigned long long w0,
                                              uint32_t n, uint32_t rt, uint32_t key_expect, uint32_t key_write,
                                              Acc &acc) {
#pragma unroll
  for (int u = 0; u < U; u++) {
    const uint32_t i = u * T + rt;
    if (i < n) {
      uint4 v = make_uint4(0, 0, 0, 0);
      if (F & kRead) v = stage[i];
      const uint4 nw = process_word<F>(a, v, w0 + i, key_expect, key_write, acc);
      if (F & kWrite) stage[i] = nw;
    }
  }
}

// RINGS rings per CTA, each of S stages of U words per ring thread
template <int OP, int U, int S, int RINGS, typename Schedule>
__device__ __forceinline__ void bulk_ring(const gsb_kernel_args &a) {
  constexpr bool kTwoPass = Schedule::kPasses == 2;
  static_assert(!kTwoPass || OP == GSB_OP_VERIFY_REFILL, "only a refill runs as a verify pass and a write pass");
  static_assert(RINGS == 1 || (kThreads == RINGS * 32 && !kTwoPass), "one ring per CTA, or one per warp");
  constexpr int kRingThreads = kThreads / RINGS;
  constexpr unsigned long long TILE = (unsigned long long)U * kRingThreads;
  const int r = RINGS == 1 ? 0 : (int)(threadIdx.x / kRingThreads);            // this thread's ring
  const uint32_t rt = RINGS == 1 ? threadIdx.x : threadIdx.x % kRingThreads;  // its thread in the ring
  auto ring_sync = [] {
    if (RINGS == 1) __syncthreads();
    else __syncwarp();
  };
  extern __shared__ __align__(128) unsigned char smem_raw[];
  uint4 *ring = reinterpret_cast<uint4 *>(smem_raw) + r * S * TILE;  // [S][TILE]
  __shared__ __align__(8) unsigned long long full_bars[RINGS][S];
  unsigned long long *full_bar = full_bars[r];
  __shared__ unsigned long long tile_of[S];  // ClaimedSchedule only
  __shared__ int gate_open;                  // two passes: this CTA may write its write-pass tiles
  const unsigned long long n_tiles = (a.n_words + TILE - 1) / TILE;
  Schedule sched(a, n_tiles, r, tile_of);
  const uint32_t key_write = gsb_seed_key(a.seed_write);
  uint4 *__restrict__ win = a.base + a.first_word;
  const bool leader = rt == 0;
  unsigned long long verified = 0;  // two passes, leader: verify-pass slots this CTA has consumed
  bool verifying = true;            // two passes, leader: this CTA has not yet left the verify pass
  Acc acc;

  auto words_of = [&](unsigned long long t) -> uint32_t {
    const unsigned long long left = a.n_words - t * TILE;
    return (uint32_t)(left < TILE ? left : TILE);
  };
  auto load = [&](unsigned long long k) {  // leader only: issue slot k
    if (!sched.has(k)) return;
    const int s = (int)(k % S);
    const unsigned long long t = sched.next(k, s);
    if (Schedule::done(t) || (kTwoPass && t >= n_tiles)) {
      // nothing to load (end of the walk, or a write-pass tile): the consumers still pass the barrier and read the slot
      mbar_arrive(smem_u32(&full_bar[s]));
      return;
    }
    const uint32_t bytes = words_of(t) * 16u;
    mbar_expect_tx(smem_u32(&full_bar[s]), bytes);
    bulk_g2s(smem_u32(ring + s * TILE), win + t * TILE, bytes, smem_u32(&full_bar[s]));
  };

  fault_smem_init();
  if (leader) {
#pragma unroll
    for (int s = 0; s < S; s++) mbar_init(smem_u32(&full_bar[s]), 1u);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    if (kTwoPass) gate_open = 1;
  }
  __syncthreads();  // the zeroed fault histogram and every ring's mbarriers

  // prologue: VERIFY and the two-pass refill can keep all S stages in flight (a consumed stage is reloaded at once);
  // the in-place VERIFY_REFILL keeps S-1 (a stage is reloaded one iteration after its store was issued)
  constexpr int kPrologue = (OP == GSB_OP_VERIFY || kTwoPass) ? S : S - 1;
  if (OP != GSB_OP_FILL && leader)
    for (int k = 0; k < kPrologue; k++) load(k);

  for (unsigned long long k = 0; sched.has(k); k++) {
    const int s = (int)(k % S);
    if (OP == GSB_OP_FILL) {
      if (leader) {
        bulk_wait_read<S - 1>();  // the bulk store that last read this stage (slot k-S) has drained it
        sched.next(k, s);
      }
      ring_sync();
    } else {
      mbar_wait(smem_u32(&full_bar[s]), (uint32_t)((k / S) & 1ull));
    }
    unsigned long long t = sched.tile(k, s);
    bool reads = OP != GSB_OP_FILL;  // two passes: a verify-pass slot reads and compares, a write-pass slot writes
    if (kTwoPass) {
      if (Schedule::done(t) || t >= n_tiles) {
        if (leader) {
          if (verifying) {
            verifying = false;
            gate_open = leave_verify_pass(a.tile_counter + 1, verified, n_tiles, !Schedule::done(t));
          }
          bulk_wait_read<S - 1>();  // the bulk store that last read this stage (slot k-S) has drained it
        }
        __syncthreads();
        if (!gate_open) break;  // uniform; only the leader writes gate_open, and only before this barrier
        if (!Schedule::done(t)) t -= n_tiles;
        reads = false;
      } else if (leader) {
        verified += 1;
      }
    }
    if (Schedule::done(t)) break;  // uniform: every thread reads the same slot after the same barrier
    const bool writes = kTwoPass ? !reads : OP != GSB_OP_VERIFY;
    const uint32_t nw_tile = words_of(t);
    uint4 *stage = ring + s * TILE;
    const unsigned long long w0 = a.first_word + t * TILE;
    const uint32_t key_expect = reads ? expect_key_of(a, w0) : 0u;
    if (!kTwoPass)
      process_stage<op_words(OP), U, kRingThreads>(a, stage, w0, nw_tile, rt, key_expect, key_write, acc);
    else if (reads)  // compare and fold what was read; its words are counted when they are written
      process_stage<kRead, U, kRingThreads>(a, stage, w0, nw_tile, rt, key_expect, key_write, acc);
    else  // the next generation; folds nothing (the checksums are of the words read)
      process_stage<kWrite | kCount, U, kRingThreads>(a, stage, w0, nw_tile, rt, key_expect, key_write, acc);
    if (writes) fence_proxy_async_smem();  // generic-proxy writes -> visible to the bulk engine
    ring_sync();  // every thread of the ring is done with this stage (reads, and writes + proxy fence)
    if (leader) {
      if (kTwoPass) {
        if (writes) {
          bulk_s2g(win + t * TILE, smem_u32(stage), nw_tile * 16u);
          bulk_commit();
        }
        load(k + S);  // same stage: a load once the barrier has released it, or (write pass) only the claim
      } else if (OP == GSB_OP_VERIFY) {
        load(k + S);  // same stage, just released by the barrier
      } else {
        bulk_s2g(win + t * TILE, smem_u32(stage), nw_tile * 16u);
        bulk_commit();
        if (OP == GSB_OP_VERIFY_REFILL && sched.has(k + S - 1)) {
          // refill stage (k-1)%S: its store (tile k-1) must have finished READING shared memory;
          // one group (tile k's store, just committed) may stay in flight
          if (k >= 1) bulk_wait_read<1>();
          load(k + S - 1);
        }
      }
    }
  }
  if (leader && OP != GSB_OP_VERIFY) bulk_wait_all<0>();  // shared memory must outlive the stores
  finish(a, acc);
}

template <int OP, int U, int S>
__global__ void __launch_bounds__(kThreads) probe_bulk(const gsb_kernel_args a) {
  bulk_ring<OP, U, S, 1, StaticSchedule<1>>(a);
}

template <int OP, int U, int S>
__global__ void __launch_bounds__(kThreads) probe_bulk_dyn(const gsb_kernel_args a) {
  bulk_ring<OP, U, S, 1, ClaimedSchedule<OP == GSB_OP_VERIFY_REFILL ? 2 : 1>>(a);
}

// BULKW: one ring per warp, WPL words per lane
template <int OP, int WPL, int S, int WARPS>
__global__ void __launch_bounds__(WARPS * 32) probe_bulk_warp(const gsb_kernel_args a) {
  bulk_ring<OP, WPL, S, WARPS, StaticSchedule<WARPS>>(a);
}

// ---------------------------------------------------------------- geometry + dispatch

constexpr int kDirectU = 4;
constexpr int kCpU = 4, kCpS = 4;  // 16 KiB tiles x 4 stages = 64 KiB / CTA
// 32 KiB tiles x 3 stages = 96 KiB / CTA: 2 CTAs per H100 SM (228 KiB); no other shape of the H100 sweep was more
// than ~1 % faster for any op (DESIGN.md §5)
constexpr int kBulkU = 8, kBulkS = 3;
constexpr int kBulkwWpl = 8, kBulkwS = 3, kBulkwWarps = 8;  // 4 KiB warp-tiles x 3 stages x 8 warps = 96 KiB / CTA
constexpr uint32_t kCpSmem = kCpU * kThreads * 16 * kCpS;
constexpr uint32_t kBulkSmem = kBulkU * kThreads * 16 * kBulkS;
constexpr uint32_t kBulkwSmem = kBulkwWpl * 512 * kBulkwS * kBulkwWarps;
constexpr int kMaxCtasPerSm = 8;

template <typename K>
int resident_ctas(K kernel, uint32_t smem, int threads) {
  int n = 0;
  if (smem > 32 * 1024) {  // dynamic + the kernel's static shared memory may cross the 48 KiB default
    if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
      return -1;
  }
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, threads, smem) != cudaSuccess) return -1;
  return n;
}

typedef void (*probe_fn)(const gsb_kernel_args);

probe_fn by_op(uint32_t op, probe_fn fill, probe_fn verify, probe_fn verify_refill) {
  if (op == GSB_OP_FILL) return fill;
  if (op == GSB_OP_VERIFY) return verify;
  if (op == GSB_OP_VERIFY_REFILL) return verify_refill;
  return nullptr;
}

// the kernel of (op, variant), its dynamic shared memory and block size; nullptr if there is none
probe_fn pick(uint32_t op, uint32_t variant, uint32_t *smem, uint32_t *threads) {
  *smem = 0;
  *threads = kThreads;
  switch (variant) {
    case GSB_VARIANT_DIRECT:
      return by_op(op, probe_direct<GSB_OP_FILL, kDirectU>, probe_direct<GSB_OP_VERIFY, kDirectU>,
                   probe_direct<GSB_OP_VERIFY_REFILL, kDirectU>);
    case GSB_VARIANT_CPASYNC:
      // FILL issues no loads, so there is nothing to stage: it takes the direct store path
      if (op != GSB_OP_FILL) *smem = kCpSmem;
      return by_op(op, probe_direct<GSB_OP_FILL, kDirectU>, probe_cpasync<GSB_OP_VERIFY, kCpU, kCpS>,
                   probe_cpasync<GSB_OP_VERIFY_REFILL, kCpU, kCpS>);
    case GSB_VARIANT_BULK:
      *smem = kBulkSmem;
      return by_op(op, probe_bulk<GSB_OP_FILL, kBulkU, kBulkS>, probe_bulk<GSB_OP_VERIFY, kBulkU, kBulkS>,
                   probe_bulk<GSB_OP_VERIFY_REFILL, kBulkU, kBulkS>);
    case GSB_VARIANT_BULKD:
      *smem = kBulkSmem;
      return by_op(op, probe_bulk_dyn<GSB_OP_FILL, kBulkU, kBulkS>, probe_bulk_dyn<GSB_OP_VERIFY, kBulkU, kBulkS>,
                   probe_bulk_dyn<GSB_OP_VERIFY_REFILL, kBulkU, kBulkS>);
    case GSB_VARIANT_BULKW:
      *smem = kBulkwSmem;
      *threads = kBulkwWarps * 32;
      return by_op(op, probe_bulk_warp<GSB_OP_FILL, kBulkwWpl, kBulkwS, kBulkwWarps>,
                   probe_bulk_warp<GSB_OP_VERIFY, kBulkwWpl, kBulkwS, kBulkwWarps>,
                   probe_bulk_warp<GSB_OP_VERIFY_REFILL, kBulkwWpl, kBulkwS, kBulkwWarps>);
    default:
      return nullptr;
  }
}

// test hook (gsb_test_stall): hold the stream for `ns` nanoseconds
__global__ void stall_kernel(unsigned long long ns) {
  const unsigned long long t0 = globaltimer();
  do {
    __nanosleep(1000);
  } while (globaltimer() - t0 < ns);
}

}  // namespace

int gsb_kernel_stall(unsigned long long ns, cudaStream_t stream) {
  stall_kernel<<<1, 1, 0, stream>>>(ns);
  return (int)cudaGetLastError();
}

// Under lazy module loading (the CUDA 12 default) a kernel's code reaches the device at its first launch or attribute
// query. Once an arena has mapped (almost) all free HBM such a load fails for lack of memory, and the kernel stays
// unusable in this process; so every kernel is loaded when the device is first made ready, before any arena exists.
int gsb_kernel_preload(void) {
  cudaFuncAttributes attr;
  for (uint32_t op = GSB_OP_FILL; op <= GSB_OP_VERIFY_REFILL; op++) {
    for (uint32_t v = GSB_VARIANT_DIRECT; v <= GSB_VARIANT_BULKD; v++) {
      uint32_t smem = 0, threads = 0;
      const probe_fn fn = pick(op, v, &smem, &threads);
      if (!fn) continue;
      const cudaError_t e = cudaFuncGetAttributes(&attr, fn);
      if (e != cudaSuccess) return (int)e;
    }
  }
  return (int)cudaFuncGetAttributes(&attr, stall_kernel);
}

uint32_t gsb_kernel_max_grid(int sm_count) { return (uint32_t)(sm_count * kMaxCtasPerSm); }

int gsb_kernel_geometry(uint32_t op, uint32_t variant, uint32_t grid_request, int sm_count,
                        gsb_launch_geom *geom) {
  // shipped choice per op (H100 lab sweep, DESIGN.md §5): the writing ops take the dynamic tile scheduler (full-arena
  // refill 56.0 vs 57.7 ms, fill 25.6 vs 26.0 ms against the static one); VERIFY runs as fast on the static one
  if (variant == GSB_VARIANT_AUTO) variant = op == GSB_OP_VERIFY ? GSB_VARIANT_BULK : GSB_VARIANT_BULKD;
  uint32_t smem = 0, threads = 0;
  probe_fn fn = pick(op, variant, &smem, &threads);
  if (!fn) return (int)cudaErrorInvalidValue;
  int per_sm = resident_ctas(fn, smem, (int)threads);
  if (per_sm <= 0) return (int)cudaErrorInvalidDeviceFunction;
  if (per_sm > kMaxCtasPerSm) per_sm = kMaxCtasPerSm;
  uint32_t grid = (uint32_t)(per_sm * sm_count);  // one full wave of resident CTAs: persistent
  if (grid_request) grid = grid_request < gsb_kernel_max_grid(sm_count) ? grid_request : gsb_kernel_max_grid(sm_count);
  geom->variant = variant;
  geom->grid = grid;
  geom->block = threads;
  geom->smem_bytes = smem;
  return 0;
}

int gsb_kernel_launch(uint32_t op, const gsb_launch_geom *geom, const gsb_kernel_args *args,
                      cudaStream_t stream) {
  uint32_t smem = 0, threads = 0;
  probe_fn fn = pick(op, geom->variant, &smem, &threads);
  if (!fn) return (int)cudaErrorInvalidValue;
  gsb_kernel_args a = *args;
  a.opaque_zero = 0u;
  fn<<<geom->grid, threads, smem, stream>>>(a);
  return (int)cudaGetLastError();
}
