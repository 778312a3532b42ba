/*
 * gsb_sparse_mma.h — the sparse tensor-core check's kernel body (gsb_sparse_probe): one 64 x 128 D per CTA through the
 * unit's 2:4-sparse instruction (1:2 for TF32), every D word compared bit for bit. The shipped kernels
 * (sparse_check<UNIT>, sparse_check_sm90a.cu) generate their operands and patterns from a.seed; the test-only twins
 * (sparse_from_table<UNIT>, sparse_operands_sm90a.cu, gsb_test_sparse_operands) read them from the table after the
 * 8192 expected words. Everything after an operand or pattern is taken is the same code. Device code only.
 *
 * Shared memory: the compressed A' (64 x K/2) and B stored as 128 x K, both in the K-major, no-swizzle core-matrix
 * layout of the tensor-core format check (8 rows x 16 bytes per core matrix), which wgmma.sp reads through descriptors
 * and ldmatrix reads one 16-byte row per lane. The metadata is computed per thread into registers
 * (gsb_sparse_kat.h).
 */
#ifndef GSB_SPARSE_MMA_H_
#define GSB_SPARSE_MMA_H_

#include <stdint.h>

#include <type_traits>

#include "gsb_sparse_kat.h"
#include "gsb_tensor_mma.h"

namespace {

// ------------------------------------------------------------------ instructions

#define GSB_SP_D64                                                                                                   \
  "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30," \
  "%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,"   \
  "%59,%60,%61,%62,%63}"
#define GSB_SP_OUT(c)                                                                                                 \
  c(d[0]), c(d[1]), c(d[2]), c(d[3]), c(d[4]), c(d[5]), c(d[6]), c(d[7]), c(d[8]), c(d[9]), c(d[10]), c(d[11]),       \
      c(d[12]), c(d[13]), c(d[14]), c(d[15]), c(d[16]), c(d[17]), c(d[18]), c(d[19]), c(d[20]), c(d[21]), c(d[22]),   \
      c(d[23]), c(d[24]), c(d[25]), c(d[26]), c(d[27]), c(d[28]), c(d[29]), c(d[30]), c(d[31]), c(d[32]), c(d[33]),   \
      c(d[34]), c(d[35]), c(d[36]), c(d[37]), c(d[38]), c(d[39]), c(d[40]), c(d[41]), c(d[42]), c(d[43]), c(d[44]),   \
      c(d[45]), c(d[46]), c(d[47]), c(d[48]), c(d[49]), c(d[50]), c(d[51]), c(d[52]), c(d[53]), c(d[54]), c(d[55]),   \
      c(d[56]), c(d[57]), c(d[58]), c(d[59]), c(d[60]), c(d[61]), c(d[62]), c(d[63])

// D += A B through wgmma.sp with metadata register m and sparsity selector SEL; the caller seeds D with +0.0 (0).
template <uint32_t UNIT, int SEL, typename T>
__device__ __forceinline__ void wgmma_sp(T (&d)[64], uint64_t da, uint64_t db, uint32_t m) {
  if constexpr (UNIT == GSB_SPARSE_UNIT_F16_SP)
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %68, 0;\nwgmma.mma_async.sp.sync.aligned.m64n128k32.f32.f16.f16 "
                 GSB_SP_D64 ", %64, %65, %66, %67, p, 1, 1, 0, 0;\n}\n"
                 : GSB_SP_OUT("+f") : "l"(da), "l"(db), "r"(m), "n"(SEL), "r"(1));
  if constexpr (UNIT == GSB_SPARSE_UNIT_BF16_SP)
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %68, 0;\nwgmma.mma_async.sp.sync.aligned.m64n128k32.f32.bf16.bf16 "
                 GSB_SP_D64 ", %64, %65, %66, %67, p, 1, 1, 0, 0;\n}\n"
                 : GSB_SP_OUT("+f") : "l"(da), "l"(db), "r"(m), "n"(SEL), "r"(1));
  if constexpr (UNIT == GSB_SPARSE_UNIT_TF32_SP)
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %68, 0;\nwgmma.mma_async.sp.sync.aligned.m64n128k16.f32.tf32.tf32 "
                 GSB_SP_D64 ", %64, %65, %66, %67, p, 1, 1;\n}\n"
                 : GSB_SP_OUT("+f") : "l"(da), "l"(db), "r"(m), "n"(SEL), "r"(1));
  if constexpr (UNIT == GSB_SPARSE_UNIT_E4M3_SP)
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %68, 0;\nwgmma.mma_async.sp.sync.aligned.m64n128k64.f32.e4m3.e4m3 "
                 GSB_SP_D64 ", %64, %65, %66, %67, p, 1, 1;\n}\n"
                 : GSB_SP_OUT("+f") : "l"(da), "l"(db), "r"(m), "n"(SEL), "r"(1));
  if constexpr (UNIT == GSB_SPARSE_UNIT_E5M2_SP)
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %68, 0;\nwgmma.mma_async.sp.sync.aligned.m64n128k64.f32.e5m2.e5m2 "
                 GSB_SP_D64 ", %64, %65, %66, %67, p, 1, 1;\n}\n"
                 : GSB_SP_OUT("+f") : "l"(da), "l"(db), "r"(m), "n"(SEL), "r"(1));
  if constexpr (UNIT == GSB_SPARSE_UNIT_S8_SP)
    asm volatile("{\n.reg .pred p;\nsetp.ne.b32 p, %68, 0;\nwgmma.mma_async.sp.sync.aligned.m64n128k64.s32.s8.s8 "
                 GSB_SP_D64 ", %64, %65, %66, %67, p;\n}\n"
                 : GSB_SP_OUT("+r") : "l"(da), "l"(db), "r"(m), "n"(SEL), "r"(1));
}

// D (16 x 8 FP32) += A (16 x 32 FP16, stored 16 x 16) B (32 x 8 FP16). a[] as hmma_16816's A fragment over the
// compressed K; b[m] = B k (8m + 2t, + 1), column g; d as hmma_16816's.
template <int SEL>
__device__ __forceinline__ void hmma_sp_16832(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[4],
                                              uint32_t m) {
  asm volatile(
      "mma.sp::ordered_metadata.sync.aligned.m16n8k32.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, "
      "{%8, %9, %10, %11}, {%0, %1, %2, %3}, %12, %13;\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]), "r"(b[2]), "r"(b[3]), "r"(m), "n"(SEL));
}

// ------------------------------------------------------------------ operands

template <uint32_t UNIT>
struct SparseUnit {
  static constexpr bool b8 =
      UNIT == GSB_SPARSE_UNIT_E4M3_SP || UNIT == GSB_SPARSE_UNIT_E5M2_SP || UNIT == GSB_SPARSE_UNIT_S8_SP;
  static constexpr uint32_t esz = UNIT == GSB_SPARSE_UNIT_TF32_SP ? 4 : b8 ? 1 : 2;
  // = gsb_sparse_shape(UNIT).k
  static constexpr uint32_t k = UNIT == GSB_SPARSE_UNIT_TF32_SP                                ? 256
                                : UNIT == GSB_SPARSE_UNIT_E4M3_SP || UNIT == GSB_SPARSE_UNIT_E5M2_SP ? 128
                                                                                              : 512;
  static constexpr uint32_t kc = k / 2;            // stored values per row of A'
  static constexpr uint32_t e = 16 / esz;          // elements per 16-byte core-matrix row
  static constexpr uint32_t steps = k / (64 / esz);  // instructions along K: each takes 32 bytes of A', 64 of B
  // byte offset of element (row r, k) of a K-major operand with `kk_total` elements along K
  static __device__ __forceinline__ uint32_t at(uint32_t r, uint32_t kk, uint32_t kk_total) {
    return ((r / 8) * (kk_total / e) + kk / e) * 128 + (r % 8) * 16 + (kk % e) * esz;
  }
};

// v * 2^s in the unit's operand type, exactly (gsb_sparse_kat.h keeps every value representable and normal)
template <uint32_t UNIT>
__device__ __forceinline__ void store_sparse(unsigned char *p, int32_t v, int32_t s) {
  if constexpr (UNIT == GSB_SPARSE_UNIT_F16_SP || UNIT == GSB_SPARSE_UNIT_HMMA_SP) store_operand<GSB_SM_UNIT_F16>(p, v, s);
  if constexpr (UNIT == GSB_SPARSE_UNIT_BF16_SP) store_operand<GSB_SM_UNIT_BF16>(p, v, s);
  if constexpr (UNIT == GSB_SPARSE_UNIT_TF32_SP) store_elem<kFmtTF32>(p, v, s);
  if constexpr (UNIT == GSB_SPARSE_UNIT_E4M3_SP) store_operand<GSB_SM_UNIT_E4M3>(p, v, s);
  if constexpr (UNIT == GSB_SPARSE_UNIT_E5M2_SP) store_elem<kFmtE5M2>(p, v, s);
  if constexpr (UNIT == GSB_SPARSE_UNIT_S8_SP) store_operand<GSB_SM_UNIT_S8>(p, v, s);
}

// The metadata register of this thread at K step `step`: the seed's patterns, or the table's
template <uint32_t UNIT, bool FROM_TABLE>
__device__ __forceinline__ uint32_t sparse_meta(uint32_t key, const int32_t *table, uint32_t w, uint32_t l,
                                                uint32_t step) {
  if constexpr (!FROM_TABLE) {
    return gsb_sparse_meta(UNIT, key, w, l, step);
  } else {
    uint32_t m = 0;
#pragma unroll
    for (uint32_t n = 0; n < 8; n++) {
      uint32_t row, q;
      gsb_sparse_slot(UNIT, l, step, n, &row, &q);
      m |= gsb_sparse_code(UNIT, (uint32_t)table[gsb_sparse_table_p(UNIT, 16 * w + row, q)]) << (4 * n);
    }
    return m;
  }
}

// ------------------------------------------------------------------ the kernel body

template <uint32_t UNIT, bool FROM_TABLE>
__device__ __forceinline__ void sparse_check_body(const gsb_sm_args &a) {
  using U = SparseUnit<UNIT>;
  constexpr uint32_t K = U::k, KC = U::kc;
  extern __shared__ __align__(1024) unsigned char sparse_smem[];
  const uint32_t sm = smid();
  if (threadIdx.x == 0) cover(a.log, sm);
  const uint32_t key = gsb_sparse_key(UNIT, a.seed);
  const int32_t *table =
      reinterpret_cast<const int32_t *>(static_cast<const char *>(a.expected) + GSB_SPARSE_WORDS * sizeof(uint32_t));
  unsigned char *A = sparse_smem, *B = sparse_smem + GSB_SM_M * KC * U::esz;
  for (uint32_t e = threadIdx.x; e < GSB_SM_M * KC; e += kMmaThreads) {
    const uint32_t i = e / KC, c = e % KC;
    store_sparse<UNIT>(A + U::at(i, c, KC),
                       FROM_TABLE ? table[gsb_sparse_table_a(UNIT, i, c)] : gsb_sparse_a(UNIT, key, i, c),
                       FROM_TABLE ? table[gsb_sparse_table_sa(UNIT, i)] : gsb_sparse_sa(UNIT, key, i));
  }
  for (uint32_t e = threadIdx.x; e < GSB_SM_N * K; e += kMmaThreads) {
    const uint32_t j = e / K, k = e % K;
    store_sparse<UNIT>(B + U::at(j, k, K), FROM_TABLE ? table[gsb_sparse_table_b(UNIT, k, j)] : gsb_sparse_b(UNIT, key, k, j),
                       FROM_TABLE ? table[gsb_sparse_table_sb(UNIT, j)] : gsb_sparse_sb(UNIT, key, j));
  }
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy stores -> wgmma's reads
  __syncthreads();
  const uint32_t w = threadIdx.x / 32, l = threadIdx.x % 32, g = l / 4, t = l % 4;
  const uint32_t *expected = static_cast<const uint32_t *>(a.expected);
  const uint32_t a0 = (uint32_t)__cvta_generic_to_shared(A), b0 = (uint32_t)__cvta_generic_to_shared(B);

  if constexpr (UNIT == GSB_SPARSE_UNIT_HMMA_SP) {
    // warp w computes rows 16w..16w+15, all sixteen 8-column tiles; K steps of 32 alternate selector 0 and 1
    float d[16][4];
#pragma unroll
    for (int n = 0; n < 16; n++)
#pragma unroll
      for (int i = 0; i < 4; i++) d[n][i] = 0.f;
    const uint32_t row = 16 * w + l % 8 + 8 * ((l / 8) % 2);  // the A' row this lane addresses
#pragma unroll 1
    for (uint32_t kk = 0; kk < U::steps; kk += 2) {
      const uint32_t m = sparse_meta<UNIT, FROM_TABLE>(key, table, w, l, kk);  // carries steps kk and kk + 1
#pragma unroll
      for (uint32_t s = 0; s < 2; s++) {
        uint32_t af[4];
        ldmatrix_x4(af, a0 + U::at(row, 16 * (kk + s) + 8 * (l / 16), KC));
#pragma unroll
        for (uint32_t n = 0; n < 16; n++) {
          uint32_t bf[4];  // tile n, K blocks 0-3 of the step
          ldmatrix_x4(bf, b0 + U::at(8 * n + l % 8, 32 * (kk + s) + 8 * (l / 8), K));
          if (s == 0) hmma_sp_16832<0>(d[n], af, bf, m);
          else hmma_sp_16832<1>(d[n], af, bf, m);
        }
      }
    }
#pragma unroll
    for (int n = 0; n < 16; n++)
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const uint32_t idx = (16 * w + g + 8 * (i / 2)) * GSB_SM_N + 8 * n + 2 * t + (i % 2);
        check(a, sm, UNIT, idx, expected[idx], __float_as_uint(d[n][i]));
      }
  } else {
    // the m64n128 accumulator fragment: register r holds D[16w + g + 8 ((r / 2) mod 2)][8 (r / 4) + 2t + (r mod 2)]
    using T = typename std::conditional<UNIT == GSB_SPARSE_UNIT_S8_SP, uint32_t, float>::type;
    T d[64];
#pragma unroll
    for (int r = 0; r < 64; r++) d[r] = 0;
    // every metadata register is made before the first wgmma.sp, so none is written while one is in flight
    constexpr uint32_t NM = U::b8 ? U::steps : U::steps / 2;  // 8-bit: selector 0 only, one register per step
    uint32_t m[NM];
#pragma unroll
    for (uint32_t i = 0; i < NM; i++) m[i] = sparse_meta<UNIT, FROM_TABLE>(key, table, w, l, U::b8 ? i : 2 * i);
    // per step: two core matrices of A' (32 bytes of each row), four of B (64 bytes)
    const uint32_t sbo_a = KC / U::e * 128, sbo_b = K / U::e * 128;
    asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
#pragma unroll
    for (uint32_t kk = 0; kk < U::steps; kk++) {
      const uint64_t da = smem_desc(a0 + kk * 256, 128, sbo_a), db = smem_desc(b0 + kk * 512, 128, sbo_b);
      if constexpr (U::b8) {
        wgmma_sp<UNIT, 0>(d, da, db, m[kk]);  // the 8-bit forms take selector 0 only
      } else {
        if (kk % 2 == 0) wgmma_sp<UNIT, 0>(d, da, db, m[kk / 2]);  // the register carries steps kk and kk + 1
        else wgmma_sp<UNIT, 1>(d, da, db, m[kk / 2]);
      }
    }
    asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
    asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
#pragma unroll
    for (int r = 0; r < 64; r++) {
      const uint32_t idx = (16 * w + g + 8 * ((r / 2) % 2)) * GSB_SM_N + 8 * (r / 4) + 2 * t + (r % 2);
      uint32_t bits;
      if constexpr (UNIT == GSB_SPARSE_UNIT_S8_SP) bits = d[r];
      else bits = __float_as_uint(d[r]);
      check(a, sm, UNIT, idx, expected[idx], bits);
    }
  }
  add_words(a.log, 64);
}

}  // namespace

#endif /* GSB_SPARSE_MMA_H_ */
