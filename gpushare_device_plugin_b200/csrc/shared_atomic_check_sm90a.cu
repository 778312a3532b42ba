/*
 * shared_atomic_check_sm90a.cu — the shared-memory atomic check's kernels (gsb_shared_atomic_probe): atomics on every
 * SM's shared memory, whose final words, returned tickets, exchanged values and compare-and-swap pairs are checked bit
 * for bit. Host code lives in gsb_device.cu (the probe) and gsb_shared_atomic.cc (expected words, policy, text); the
 * geometry and the values are in gsb_shared_atomic.h. Built into a module of its own, libgpushare_b200_shared_atomic.so.
 *
 * One CTA per SM, with the opt-in maximum of dynamic shared memory, so at most one CTA fits on an SM. Each CTA records
 * its %smid, writes the unit's starting words into its area, issues the unit's atomics (spread, then hot), and after a
 * barrier compares its area with the expected words uploaded by the host. Every atomic is inline PTX on a shared-window
 * address with a per-lane operand, so the instruction is the one named and never a warp-aggregated form.
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "gsb_internal.h"
#include "gsb_shared_atomic.h"

namespace {

constexpr uint32_t kThreads = GSB_SHARED_ATOMIC_THREADS;
constexpr uint32_t kCount = GSB_SHARED_ATOMIC_COUNT;

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

__device__ __noinline__ void record(gsb_shared_atomic_log *log, uint32_t sm, uint32_t unit, uint32_t kind,
                                    uint32_t index, uint64_t e, uint64_t o) {
  if (sm < GSB_SM_MAX) atomicOr(&log->faulty[sm >> 5], 1u << (sm & 31u));
  const unsigned slot = atomicAdd(&log->count, 1u);
  if (slot < GSB_SHARED_ATOMIC_RECORDS) {
    gsb_shared_atomic_record &r = log->rec[slot];
    r.smid = sm;
    r.unit = unit;
    r.kind = kind;
    r.index = index;
    r.expected = e;
    r.observed = o;
  }
}

// ---- the atomics, one PTX instruction each, on a shared-window address

__device__ __forceinline__ void red_int32(uint32_t p, uint32_t kind, uint32_t v) {
  switch (kind) {
    case 0: asm volatile("red.shared.add.u32 [%0], %1;" ::"r"(p), "r"(v) : "memory"); break;
    case 1: asm volatile("red.shared.and.b32 [%0], %1;" ::"r"(p), "r"(v) : "memory"); break;
    case 2: asm volatile("red.shared.or.b32 [%0], %1;" ::"r"(p), "r"(v) : "memory"); break;
    case 3: asm volatile("red.shared.xor.b32 [%0], %1;" ::"r"(p), "r"(v) : "memory"); break;
    case 4: asm volatile("red.shared.min.s32 [%0], %1;" ::"r"(p), "r"(v) : "memory"); break;
    case 5: asm volatile("red.shared.max.s32 [%0], %1;" ::"r"(p), "r"(v) : "memory"); break;
    case 6: asm volatile("red.shared.min.u32 [%0], %1;" ::"r"(p), "r"(v) : "memory"); break;
    case 7: asm volatile("red.shared.max.u32 [%0], %1;" ::"r"(p), "r"(v) : "memory"); break;
    case 8: asm volatile("red.shared.inc.u32 [%0], %1;" ::"r"(p), "r"(v) : "memory"); break;
    default: asm volatile("red.shared.dec.u32 [%0], %1;" ::"r"(p), "r"(v) : "memory"); break;
  }
}
__device__ __forceinline__ void red_wide(uint32_t p, uint32_t kind, uint64_t v) {
  switch (kind) {
    case 0: asm volatile("red.shared.add.u64 [%0], %1;" ::"r"(p), "l"(v) : "memory"); break;
    case 1: asm volatile("red.shared.and.b64 [%0], %1;" ::"r"(p), "l"(v) : "memory"); break;
    case 2: asm volatile("red.shared.or.b64 [%0], %1;" ::"r"(p), "l"(v) : "memory"); break;
    case 3: asm volatile("red.shared.xor.b64 [%0], %1;" ::"r"(p), "l"(v) : "memory"); break;
    case 4: asm volatile("red.shared.min.s64 [%0], %1;" ::"r"(p), "l"(v) : "memory"); break;
    default: asm volatile("red.shared.max.u64 [%0], %1;" ::"r"(p), "l"(v) : "memory"); break;
  }
}
__device__ __forceinline__ void red_float(uint32_t p, uint32_t kind, uint64_t h, uint32_t phase) {
  switch (kind) {
    case 0: {
      const float v = (float)gsb_atomic_ival(GSB_ATOMIC_OP_FADD32, phase, h);
      asm volatile("red.shared.add.f32 [%0], %1;" ::"r"(p), "f"(v) : "memory");
      break;
    }
    case 1: {
      const double v = (double)gsb_atomic_ival(GSB_ATOMIC_OP_FADD64, phase, h);
      asm volatile("red.shared.add.f64 [%0], %1;" ::"r"(p), "d"(v) : "memory");
      break;
    }
    default: {
      const uint32_t v = gsb_atomic_half2(kind - 2u, gsb_atomic_ival(GSB_ATOMIC_OP_HADD2, phase, h & 0xFFFFu),
                                          gsb_atomic_ival(GSB_ATOMIC_OP_HADD2, phase, (h >> 16) & 0xFFFFu));
      if (kind == 2u) asm volatile("red.shared.add.noftz.f16x2 [%0], %1;" ::"r"(p), "r"(v) : "memory");
      else asm volatile("red.shared.add.noftz.bf16x2 [%0], %1;" ::"r"(p), "r"(v) : "memory");
      break;
    }
  }
}
__device__ __forceinline__ uint32_t atom_add_u32(uint32_t p, uint32_t v) {
  uint32_t old;
  asm volatile("atom.shared.add.u32 %0, [%1], %2;" : "=r"(old) : "r"(p), "r"(v) : "memory");
  return old;
}
__device__ __forceinline__ uint32_t atom_exch_b32(uint32_t p, uint32_t v) {
  uint32_t old;
  asm volatile("atom.shared.exch.b32 %0, [%1], %2;" : "=r"(old) : "r"(p), "r"(v) : "memory");
  return old;
}
__device__ __forceinline__ uint64_t atom_exch_b64(uint32_t p, uint64_t v) {
  uint64_t old;
  asm volatile("atom.shared.exch.b64 %0, [%1], %2;" : "=l"(old) : "r"(p), "l"(v) : "memory");
  return old;
}
__device__ __forceinline__ void atom_exch_b128(uint32_t p, uint64_t lo, uint64_t hi, uint64_t *olo, uint64_t *ohi) {
  asm volatile(
      "{\n\t.reg .b128 d, v;\n\tmov.b128 v, {%2, %3};\n\tatom.shared.exch.b128 d, [%4], v;\n\t"
      "mov.b128 {%0, %1}, d;\n\t}"
      : "=l"(*olo), "=l"(*ohi)
      : "l"(lo), "l"(hi), "r"(p)
      : "memory");
}
__device__ __forceinline__ uint32_t atom_cas_b32(uint32_t p, uint32_t cmp, uint32_t v) {
  uint32_t old;
  asm volatile("atom.shared.cas.b32 %0, [%1], %2, %3;" : "=r"(old) : "r"(p), "r"(cmp), "r"(v) : "memory");
  return old;
}
__device__ __forceinline__ uint64_t atom_cas_b64(uint32_t p, uint64_t cmp, uint64_t v) {
  uint64_t old;
  asm volatile("atom.shared.cas.b64 %0, [%1], %2, %3;" : "=l"(old) : "r"(p), "l"(cmp), "l"(v) : "memory");
  return old;
}
__device__ __forceinline__ void atom_cas_b128(uint32_t p, uint64_t clo, uint64_t chi, uint64_t lo, uint64_t hi,
                                              uint64_t *olo, uint64_t *ohi) {
  asm volatile(
      "{\n\t.reg .b128 d, c, v;\n\tmov.b128 c, {%2, %3};\n\tmov.b128 v, {%4, %5};\n\t"
      "atom.shared.cas.b128 d, [%6], c, v;\n\tmov.b128 {%0, %1}, d;\n\t}"
      : "=l"(*olo), "=l"(*ohi)
      : "l"(clo), "l"(chi), "l"(lo), "l"(hi), "r"(p)
      : "memory");
}

// One contribution of thread t (phase, round or repetition r) to unit u of an INT32, WIDE or FLOAT area at `area`.
template <uint32_t UNIT>
__device__ __forceinline__ void contribute(uint32_t area, uint32_t seed, uint32_t phase, uint32_t t, uint32_t r,
                                           uint32_t u) {
  constexpr uint32_t ub = UNIT == GSB_SHARED_ATOMIC_UNIT_INT32 ? 4u : 8u;
  const uint32_t p = area + u * ub, kind = gsb_shared_atomic_kind(UNIT, u);
  const uint64_t h = gsb_shared_atomic_key(UNIT, seed, phase, t, r);
  if constexpr (UNIT == GSB_SHARED_ATOMIC_UNIT_INT32)
    red_int32(p, kind, (uint32_t)gsb_shared_atomic_operand(UNIT, seed, kind, u, h));
  if constexpr (UNIT == GSB_SHARED_ATOMIC_UNIT_WIDE) red_wide(p, kind, gsb_shared_atomic_operand(UNIT, seed, kind, u, h));
  if constexpr (UNIT == GSB_SHARED_ATOMIC_UNIT_FLOAT) red_float(p, kind, h, phase);
}

// An add or CAS ticket: the id goes to its entry; a ticket out of range is recorded instead.
__device__ __forceinline__ void take_ticket(const gsb_shared_atomic_args &a, uint32_t *slots, uint32_t unit, uint32_t f,
                                            uint32_t l, uint32_t ticket, uint32_t id, uint32_t sm) {
  if (ticket < kCount) {
    slots[gsb_shared_atomic_slot(0, f, l, ticket)] = id;
  } else {
    atomicAdd(&a.log->faults, 1u);
    record(a.log, sm, unit, GSB_SHARED_ATOMIC_REC_TICKET, l, kCount, ticket);
  }
}

template <uint32_t UNIT>
__global__ void __launch_bounds__(kThreads, 1) shared_atomic_check(const gsb_shared_atomic_args a) {
  extern __shared__ __align__(16) uint32_t smem[];
  const uint32_t b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31u, sm = smid();
  const uint32_t area = (uint32_t)__cvta_generic_to_shared(smem);
  constexpr bool kSlots = UNIT == GSB_SHARED_ATOMIC_UNIT_TICKET || UNIT == GSB_SHARED_ATOMIC_UNIT_CAS;
  uint32_t *slots = kSlots ? a.slots + gsb_shared_atomic_slot(b, 0, 0, 0) : nullptr;
  if (tid == 0) {
    if (sm < GSB_SM_MAX) atomicOr(&a.log->covered[sm >> 5], 1u << (sm & 31u));
    if (b < GSB_SM_MAX) a.log->cta_smid[b] = sm;
  }
  for (uint32_t w = tid; w < GSB_SHARED_ATOMIC_AREA_WORDS; w += kThreads)
    smem[w] = gsb_shared_atomic_init_word(UNIT, a.seed, w);
  if constexpr (kSlots)
    for (uint32_t i = tid; i < GSB_SHARED_ATOMIC_SLOT_WORDS; i += kThreads) slots[i] = GSB_SHARED_ATOMIC_NO_ID;
  __syncthreads();
  const bool skip = sm == a.skip_smid;  // test hook: this CTA issues none of its atomics
  if (skip && tid == 0) a.log->skipped_cta = b + 1u;
  uint32_t issued = 0, longest = 0;
  if (!skip) {
    if constexpr (!kSlots) {
      for (uint32_t r = 0; r < gsb_shared_atomic_rounds(UNIT); r++, issued++)
        contribute<UNIT>(area, a.seed, GSB_ATOMIC_PHASE_SPREAD, tid, r, gsb_shared_atomic_spread_unit(UNIT, tid, r));
      for (uint32_t r = 0; r < GSB_SHARED_ATOMIC_HOT_REPS; r++, issued++)
        contribute<UNIT>(area, a.seed, GSB_ATOMIC_PHASE_HOT, tid, r, gsb_shared_atomic_hot_unit(UNIT, lane));
    }
    const uint32_t hot = area + GSB_SHARED_ATOMIC_SPREAD_BYTES + lane * GSB_SHARED_ATOMIC_HOT_STRIDE;
    if constexpr (UNIT == GSB_SHARED_ATOMIC_UNIT_TICKET) {
      for (uint32_t r = 0; r < GSB_SHARED_ATOMIC_HOT_REPS; r++) {
        const uint32_t id = warp * GSB_SHARED_ATOMIC_HOT_REPS + r;
        take_ticket(a, slots, UNIT, 0u, lane, atom_add_u32(hot, 1u), id, sm);
        uint32_t *e = slots + gsb_shared_atomic_slot(0, 1u, lane, id);
        e[0] = atom_exch_b32(hot + GSB_SHARED_ATOMIC_TICKET_EXCH32, gsb_shared_atomic_exch(a.seed, 1u, lane, id, 0u));
        const uint64_t v64 = (uint64_t)gsb_shared_atomic_exch(a.seed, 2u, lane, id, 0u) |
                             (uint64_t)gsb_shared_atomic_exch(a.seed, 2u, lane, id, 1u) << 32;
        const uint64_t o64 = atom_exch_b64(hot + GSB_SHARED_ATOMIC_TICKET_EXCH64, v64);
        e = slots + gsb_shared_atomic_slot(0, 2u, lane, id);
        e[0] = (uint32_t)o64;
        e[1] = (uint32_t)(o64 >> 32);
        const uint64_t lo = (uint64_t)gsb_shared_atomic_exch(a.seed, 3u, lane, id, 0u) |
                            (uint64_t)gsb_shared_atomic_exch(a.seed, 3u, lane, id, 1u) << 32;
        const uint64_t hi = (uint64_t)gsb_shared_atomic_exch(a.seed, 3u, lane, id, 2u) |
                            (uint64_t)gsb_shared_atomic_exch(a.seed, 3u, lane, id, 3u) << 32;
        uint64_t olo, ohi;
        atom_exch_b128(hot + GSB_SHARED_ATOMIC_TICKET_EXCH128, lo, hi, &olo, &ohi);
        e = slots + gsb_shared_atomic_slot(0, 3u, lane, id);
        e[0] = (uint32_t)olo;
        e[1] = (uint32_t)(olo >> 32);
        e[2] = (uint32_t)ohi;
        e[3] = (uint32_t)(ohi >> 32);
        issued += 4u;
      }
    }
    if constexpr (UNIT == GSB_SHARED_ATOMIC_UNIT_CAS) {
      // each returned value is the next compare; the swap that succeeds returns this thread's ticket
      // one deadline bounds all of a thread's loops, so no thread spins past GSB_SHARED_ATOMIC_CAS_WAIT_NS
      const uint64_t start64 = gsb_shared_atomic_cas64_start(a.seed, lane);
      const unsigned long long t0 = globaltimer(), deadline = t0 + GSB_SHARED_ATOMIC_CAS_WAIT_NS;
      bool late = false;
      for (uint32_t r = 0; r < GSB_SHARED_ATOMIC_HOT_REPS && !late; r++) {
        const uint32_t id = warp * GSB_SHARED_ATOMIC_HOT_REPS + r;
        uint32_t c32 = 0;
        for (;;) {
          const uint32_t old = atom_cas_b32(hot, c32, c32 + 1u);
          if (old == c32) break;
          c32 = old;
          if ((late = globaltimer() > deadline)) break;
        }
        if (!late) take_ticket(a, slots, UNIT, 0u, lane, c32, id, sm), issued++;
        uint64_t c64 = start64;
        while (!late) {
          const uint64_t old = atom_cas_b64(hot + GSB_SHARED_ATOMIC_CAS64, c64, c64 + 1u);
          if (old == c64) break;
          c64 = old;
          late = globaltimer() > deadline;
        }
        if (!late) take_ticket(a, slots, UNIT, 1u, lane, (uint32_t)(c64 - start64), id, sm), issued++;
        uint64_t clo = 0, chi = gsb_shared_atomic_pair(a.seed, lane, 0u);
        while (!late) {
          uint64_t olo, ohi;
          atom_cas_b128(hot + GSB_SHARED_ATOMIC_CAS128, clo, chi, clo + 1u, gsb_shared_atomic_pair(a.seed, lane, clo + 1u),
                        &olo, &ohi);
          if (olo == clo && ohi == chi) break;
          if (ohi != gsb_shared_atomic_pair(a.seed, lane, olo)) {  // a torn pair
            atomicAdd(&a.log->faults, 1u);
            record(a.log, sm, UNIT, GSB_SHARED_ATOMIC_REC_TORN, lane, gsb_shared_atomic_pair(a.seed, lane, olo), ohi);
          }
          clo = olo;
          chi = ohi;
          late = globaltimer() > deadline;
        }
        if (!late) take_ticket(a, slots, UNIT, 2u, lane, (uint32_t)clo, id, sm), issued++;
      }
      longest = (uint32_t)min(globaltimer() - t0, 0xFFFFFFFFull);
      if (late) atomicAdd(&a.log->timeouts, 1u);
    }
  }
  __syncthreads();
  if constexpr (UNIT == GSB_SHARED_ATOMIC_UNIT_TICKET) {  // the final exchange words go to their entries
    if (tid < GSB_SHARED_ATOMIC_HOT_WORDS) {
      const uint32_t *hw = smem + (GSB_SHARED_ATOMIC_SPREAD_BYTES + tid * GSB_SHARED_ATOMIC_HOT_STRIDE) / 4u;
      slots[gsb_shared_atomic_slot(0, 1u, tid, kCount)] = hw[GSB_SHARED_ATOMIC_TICKET_EXCH32 / 4u];
      for (uint32_t c = 0; c < 2u; c++)
        slots[gsb_shared_atomic_slot(0, 2u, tid, kCount) + c] = hw[GSB_SHARED_ATOMIC_TICKET_EXCH64 / 4u + c];
      for (uint32_t c = 0; c < 4u; c++)
        slots[gsb_shared_atomic_slot(0, 3u, tid, kCount) + c] = hw[GSB_SHARED_ATOMIC_TICKET_EXCH128 / 4u + c];
    }
  }
  uint32_t checked = 0;
  for (uint32_t w = tid; w < GSB_SHARED_ATOMIC_AREA_WORDS; w += kThreads) {
    if (!gsb_shared_atomic_compared(UNIT, w)) continue;
    uint32_t o = smem[w];
    const uint32_t e = a.expected[w];
    if (sm == a.hook_smid && w == a.hook_index) o ^= (uint32_t)a.hook_xr;  // test hook
    checked++;
    if (o != e) {
      atomicAdd(&a.log->mismatch_words, 1ull);
      atomicAdd(&a.log->mismatch_bits, (unsigned long long)__popc(o ^ e));
      record(a.log, sm, UNIT, GSB_SHARED_ATOMIC_REC_WORD, w, e, o);
    }
  }
  checked = __reduce_add_sync(0xFFFFFFFFu, checked);
  issued = __reduce_add_sync(0xFFFFFFFFu, issued);
  if (lane == 0) {
    atomicAdd(&a.log->words, (unsigned long long)checked);
    atomicAdd(&a.log->issued, (unsigned long long)issued);
  }
  if constexpr (UNIT == GSB_SHARED_ATOMIC_UNIT_CAS) {
    longest = __reduce_max_sync(0xFFFFFFFFu, longest);
    if (lane == 0) atomicMax(&a.log->cas_max_ns, longest);
  }
}

// ---- DSMEM and REDAS: atomics over the SM-to-SM network into every other rank's area

__device__ __forceinline__ uint32_t cluster_rank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ uint32_t cluster_size() {
  uint32_t n;
  asm volatile("mov.u32 %0, %%cluster_nctarank;" : "=r"(n));
  return n;
}
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t mapa(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
__device__ __forceinline__ void red_cluster_add_u32(uint32_t p, uint32_t v) {
  asm volatile("red.shared::cluster.add.u32 [%0], %1;" ::"r"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void red_cluster_add_u64(uint32_t p, uint64_t v) {
  asm volatile("red.shared::cluster.add.u64 [%0], %1;" ::"r"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void red_cluster_add_f32(uint32_t p, float v) {
  asm volatile("red.shared::cluster.add.f32 [%0], %1;" ::"r"(p), "f"(v) : "memory");
}
__device__ __forceinline__ uint32_t atom_cluster_cas_b32(uint32_t p, uint32_t cmp, uint32_t v) {
  uint32_t old;
  asm volatile("atom.shared::cluster.cas.b32 %0, [%1], %2, %3;" : "=r"(old) : "r"(p), "r"(cmp), "r"(v) : "memory");
  return old;
}
// red.async into a peer's word, completing `bytes` on the peer's mbarrier `bar` (both shared::cluster addresses)
__device__ __forceinline__ void redas(uint32_t j, uint32_t p, uint64_t v, uint32_t bar) {
  switch (j) {
    case 0:
      asm volatile("red.async.relaxed.cluster.shared::cluster.mbarrier::complete_tx::bytes.add.u32 [%0], %1, [%2];"
                   ::"r"(p), "r"((uint32_t)v), "r"(bar) : "memory");
      break;
    case 1:
      asm volatile("red.async.relaxed.cluster.shared::cluster.mbarrier::complete_tx::bytes.add.u64 [%0], %1, [%2];"
                   ::"r"(p), "l"(v), "r"(bar) : "memory");
      break;
    case 2:
      asm volatile("red.async.relaxed.cluster.shared::cluster.mbarrier::complete_tx::bytes.xor.b32 [%0], %1, [%2];"
                   ::"r"(p), "r"((uint32_t)v), "r"(bar) : "memory");
      break;
    case 3:
      asm volatile("red.async.relaxed.cluster.shared::cluster.mbarrier::complete_tx::bytes.max.s32 [%0], %1, [%2];"
                   ::"r"(p), "r"((uint32_t)v), "r"(bar) : "memory");
      break;
    default:
      asm volatile("red.async.relaxed.cluster.shared::cluster.mbarrier::complete_tx::bytes.inc.u32 [%0], %1, [%2];"
                   ::"r"(p), "r"((uint32_t)v), "r"(bar) : "memory");
      break;
  }
}
// a bounded wait for phase 0 of this CTA's mbarrier: false when the deadline passed first
__device__ __forceinline__ bool mbar_wait(uint32_t bar, unsigned long long deadline) {
  for (;;) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], 0;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar)
        : "memory");
    if (done) return true;
    if (globaltimer() > deadline) return false;
  }
}

template <uint32_t UNIT>
__global__ void __launch_bounds__(kThreads, 1) shared_atomic_cluster(const gsb_shared_atomic_args a) {
  // the area, then (in the dynamic allocation too: the CTA takes the whole opt-in maximum, with no static shared
  // memory beside it) REDAS's mbarrier, which completes when every peer's bytes have landed
  extern __shared__ __align__(16) uint32_t smem[];
  const uint32_t b = blockIdx.x, tid = threadIdx.x, lane = tid & 31u, sm = smid();
  const uint32_t rank = cluster_rank(), n = cluster_size();
  const uint32_t area = (uint32_t)__cvta_generic_to_shared(smem), bar = area + GSB_SHARED_ATOMIC_AREA_BYTES;
  if (tid == 0) {
    if (sm < GSB_SM_MAX) atomicOr(&a.log->covered[sm >> 5], 1u << (sm & 31u));
    if (b < GSB_SM_MAX) a.log->cta_smid[b] = sm;
  }
  for (uint32_t w = tid; w < GSB_SHARED_ATOMIC_AREA_WORDS; w += kThreads)
    smem[w] = gsb_shared_atomic_cluster_init_word(UNIT, a.seed, w);
  if constexpr (UNIT == GSB_SHARED_ATOMIC_UNIT_REDAS) {
    if (tid == 0) {  // armed with exactly the bytes the peers send, before the barrier lets any of them issue
      asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar) : "memory");
      asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar),
                   "r"((n - 1u) * kThreads * GSB_SHARED_ATOMIC_REDAS_BYTES)
                   : "memory");
    }
  }
  cluster_sync();  // every area written and every mbarrier armed before any peer sends
  const bool skip = sm == a.skip_smid;  // test hook: this CTA sends nothing, and takes part in every barrier
  if (skip && tid == 0) a.log->skipped_cta = b + 1u;
  uint32_t issued = 0, longest = 0;
  bool late = false;
  const unsigned long long t0 = globaltimer(), deadline = t0 + GSB_SHARED_ATOMIC_CAS_WAIT_NS;
  for (uint32_t k = 1; k < n && !skip; k++) {
    const uint32_t q = (rank + k) % n, peer = mapa(area, q);  // another rank only: its own would take the ATOMS path
    if constexpr (UNIT == GSB_SHARED_ATOMIC_UNIT_DSMEM) {
      for (uint32_t j = 0; j < GSB_SHARED_ATOMIC_DSMEM_OPS; j++, issued++) {
        const uint32_t p = peer + 4u * gsb_shared_atomic_peer_word(UNIT, tid, j);
        const uint64_t v = gsb_shared_atomic_peer_operand(UNIT, a.seed, rank, tid, j);
        if (j < 4u) red_cluster_add_u32(p, (uint32_t)v);
        else if (j < 6u) red_cluster_add_u64(p, v);
        else red_cluster_add_f32(p, __uint_as_float((uint32_t)v));
      }
      // a cas.b32 increment loop on the peer's counter `lane`, each returned value the next compare
      const uint32_t p = peer + 4u * gsb_shared_atomic_peer_word(UNIT, tid, GSB_SHARED_ATOMIC_DSMEM_OPS);
      uint32_t cmp = 0;
      while (!late) {
        const uint32_t old = atom_cluster_cas_b32(p, cmp, cmp + 1u);
        if (old == cmp) {
          issued++;
          break;
        }
        cmp = old;
        late = globaltimer() > deadline;
      }
    } else {
      const uint32_t pbar = mapa(bar, q);
      for (uint32_t j = 0; j < GSB_SHARED_ATOMIC_REDAS_OPS; j++, issued++)
        redas(j, peer + 4u * gsb_shared_atomic_peer_word(UNIT, tid, j),
              gsb_shared_atomic_peer_operand(UNIT, a.seed, rank, tid, j), pbar);
    }
  }
  if constexpr (UNIT == GSB_SHARED_ATOMIC_UNIT_DSMEM) {
    longest = (uint32_t)min(globaltimer() - t0, 0xFFFFFFFFull);
    if (late) atomicAdd(&a.log->timeouts, 1u);
    cluster_sync();  // every peer's atomics done before this rank reads its area
  } else {
    if (tid == 0 && !mbar_wait(bar, globaltimer() + GSB_SHARED_ATOMIC_CAS_WAIT_NS))
      atomicAdd(&a.log->timeouts, 1u);  // counted, and the area checked anyway
    __syncthreads();
  }
  uint32_t checked = 0;
  for (uint32_t w = tid; w < GSB_SHARED_ATOMIC_AREA_WORDS; w += kThreads) {
    uint32_t o = smem[w];
    const uint32_t e = a.expected[rank * GSB_SHARED_ATOMIC_AREA_WORDS + w];
    if (sm == a.hook_smid && w == a.hook_index) o ^= (uint32_t)a.hook_xr;  // test hook
    checked++;
    if (o != e) {
      atomicAdd(&a.log->mismatch_words, 1ull);
      atomicAdd(&a.log->mismatch_bits, (unsigned long long)__popc(o ^ e));
      record(a.log, sm, UNIT, GSB_SHARED_ATOMIC_REC_WORD, rank * GSB_SHARED_ATOMIC_AREA_WORDS + w, e, o);
    }
  }
  checked = __reduce_add_sync(0xFFFFFFFFu, checked);
  issued = __reduce_add_sync(0xFFFFFFFFu, issued);
  longest = __reduce_max_sync(0xFFFFFFFFu, longest);
  if (lane == 0) {
    atomicAdd(&a.log->words, (unsigned long long)checked);
    atomicAdd(&a.log->issued, (unsigned long long)issued);
    atomicMax(&a.log->cas_max_ns, longest);
  }
  cluster_sync();  // no CTA exits while a peer of its cluster may still reach its shared memory
}

template <uint32_t UNIT>
cudaLaunchConfig_t cluster_config(uint32_t n, uint32_t clusters, uint32_t smem, cudaStream_t stream,
                                  cudaLaunchAttribute *attr) {
  cudaLaunchConfig_t c = {};
  c.gridDim = dim3(clusters * n, 1, 1);
  c.blockDim = dim3(kThreads, 1, 1);
  c.dynamicSmemBytes = smem;
  c.stream = stream;
  attr->id = cudaLaunchAttributeClusterDimension;
  attr->val.clusterDim.x = n;
  attr->val.clusterDim.y = 1;
  attr->val.clusterDim.z = 1;
  c.attrs = attr;
  c.numAttrs = 1;
  return c;
}

}  // namespace

int gsb_shared_atomic_kernel_launch(uint32_t unit, uint32_t grid, const gsb_shared_atomic_args *a, cudaStream_t stream) {
  if (!grid || grid > GSB_SM_MAX) return (int)cudaErrorInvalidValue;
  const size_t smem = a->smem_bytes;
  switch (unit) {
    case GSB_SHARED_ATOMIC_UNIT_INT32:
      shared_atomic_check<GSB_SHARED_ATOMIC_UNIT_INT32><<<grid, kThreads, smem, stream>>>(*a);
      break;
    case GSB_SHARED_ATOMIC_UNIT_WIDE: shared_atomic_check<GSB_SHARED_ATOMIC_UNIT_WIDE><<<grid, kThreads, smem, stream>>>(*a); break;
    case GSB_SHARED_ATOMIC_UNIT_FLOAT:
      shared_atomic_check<GSB_SHARED_ATOMIC_UNIT_FLOAT><<<grid, kThreads, smem, stream>>>(*a);
      break;
    case GSB_SHARED_ATOMIC_UNIT_TICKET:
      shared_atomic_check<GSB_SHARED_ATOMIC_UNIT_TICKET><<<grid, kThreads, smem, stream>>>(*a);
      break;
    case GSB_SHARED_ATOMIC_UNIT_CAS: shared_atomic_check<GSB_SHARED_ATOMIC_UNIT_CAS><<<grid, kThreads, smem, stream>>>(*a); break;
    default: return (int)cudaErrorInvalidValue;
  }
  return (int)cudaGetLastError();
}

int gsb_shared_atomic_cluster_launch(uint32_t unit, uint32_t n, uint32_t clusters, const gsb_shared_atomic_args *a,
                                     cudaStream_t stream) {
  if (n < 2u || n > 16u || (n & (n - 1u)) || !clusters || clusters * n > GSB_SM_MAX) return (int)cudaErrorInvalidValue;
  cudaLaunchAttribute attr;
  cudaError_t e;
  switch (unit) {
    case GSB_SHARED_ATOMIC_UNIT_DSMEM: {
      const cudaLaunchConfig_t c = cluster_config<GSB_SHARED_ATOMIC_UNIT_DSMEM>(n, clusters, a->smem_bytes, stream, &attr);
      e = cudaLaunchKernelEx(&c, shared_atomic_cluster<GSB_SHARED_ATOMIC_UNIT_DSMEM>, *a);
      break;
    }
    case GSB_SHARED_ATOMIC_UNIT_REDAS: {
      const cudaLaunchConfig_t c = cluster_config<GSB_SHARED_ATOMIC_UNIT_REDAS>(n, clusters, a->smem_bytes, stream, &attr);
      e = cudaLaunchKernelEx(&c, shared_atomic_cluster<GSB_SHARED_ATOMIC_UNIT_REDAS>, *a);
      break;
    }
    default: return (int)cudaErrorInvalidValue;
  }
  return (int)(e != cudaSuccess ? e : cudaGetLastError());
}

int gsb_shared_atomic_max_clusters(uint32_t unit, uint32_t n, int smem_bytes, int *clusters) {
  cudaLaunchAttribute attr;
  *clusters = 0;
  const cudaLaunchConfig_t c = cluster_config<GSB_SHARED_ATOMIC_UNIT_DSMEM>(n, 1, (uint32_t)smem_bytes, nullptr, &attr);
  const void *fn = unit == GSB_SHARED_ATOMIC_UNIT_REDAS ? (const void *)shared_atomic_cluster<GSB_SHARED_ATOMIC_UNIT_REDAS>
                                                        : (const void *)shared_atomic_cluster<GSB_SHARED_ATOMIC_UNIT_DSMEM>;
  return (int)cudaOccupancyMaxActiveClusters(clusters, fn, &c);
}

int gsb_shared_atomic_kernel_preload(int smem_bytes) {
  const void *fns[5] = {(const void *)shared_atomic_check<GSB_SHARED_ATOMIC_UNIT_INT32>,
                                              (const void *)shared_atomic_check<GSB_SHARED_ATOMIC_UNIT_WIDE>,
                                              (const void *)shared_atomic_check<GSB_SHARED_ATOMIC_UNIT_FLOAT>,
                                              (const void *)shared_atomic_check<GSB_SHARED_ATOMIC_UNIT_TICKET>,
                                              (const void *)shared_atomic_check<GSB_SHARED_ATOMIC_UNIT_CAS>};
  for (const void *fn : fns) {
    const cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
    if (e != cudaSuccess) return (int)e;
  }
  const void *cluster_fns[2] = {(const void *)shared_atomic_cluster<GSB_SHARED_ATOMIC_UNIT_DSMEM>,
                                (const void *)shared_atomic_cluster<GSB_SHARED_ATOMIC_UNIT_REDAS>};
  for (const void *fn : cluster_fns) {
    cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(fn, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    if (e != cudaSuccess) return (int)e;
  }
  return (int)cudaSuccess;
}
