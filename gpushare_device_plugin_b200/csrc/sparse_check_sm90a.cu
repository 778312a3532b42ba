/*
 * sparse_check_sm90a.cu — the sparse tensor-core check's kernels (gsb_sparse_probe): one 64 x 128 D per CTA, one CTA
 * per SM, through the 2:4-sparse wgmma.sp forms (F16, BF16, TF32 1:2, E4M3, E5M2, S8) and warp-level
 * mma.sp::ordered_metadata. The body is gsb_sparse_mma.h; host code lives in gsb_device.cu (the probe) and
 * gsb_sparse.cc (the expected answers). Built into a module of its own, libgpushare_b200_sparse.so, with its
 * test-only twins (sparse_operands_sm90a.cu).
 *
 * Every kernel is launched with the device's opt-in maximum of dynamic shared memory, more than half an SM's, so at
 * most one CTA fits on an SM; thread 0 of each CTA sets bit %smid of the launch's coverage bitmap. A wrong D word is
 * counted in the launch's gsb_sm_log (words, bits, faulty-SM bitmap, the first GSB_SM_RECORDS records).
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "gsb_sparse_mma.h"

namespace {

template <uint32_t UNIT>
__global__ void __launch_bounds__(kMmaThreads) sparse_check(const gsb_sm_args a) {
  sparse_check_body<UNIT, false>(a);  // operands and patterns of a.seed
}

}  // namespace

int gsb_sparse_kernel_launch(uint32_t unit, uint32_t grid, const gsb_sm_args *a, cudaStream_t stream) {
  const size_t smem = a->smem_bytes;
  switch (unit) {
    case GSB_SPARSE_UNIT_F16_SP: sparse_check<GSB_SPARSE_UNIT_F16_SP><<<grid, kMmaThreads, smem, stream>>>(*a); break;
    case GSB_SPARSE_UNIT_BF16_SP: sparse_check<GSB_SPARSE_UNIT_BF16_SP><<<grid, kMmaThreads, smem, stream>>>(*a); break;
    case GSB_SPARSE_UNIT_TF32_SP: sparse_check<GSB_SPARSE_UNIT_TF32_SP><<<grid, kMmaThreads, smem, stream>>>(*a); break;
    case GSB_SPARSE_UNIT_E4M3_SP: sparse_check<GSB_SPARSE_UNIT_E4M3_SP><<<grid, kMmaThreads, smem, stream>>>(*a); break;
    case GSB_SPARSE_UNIT_E5M2_SP: sparse_check<GSB_SPARSE_UNIT_E5M2_SP><<<grid, kMmaThreads, smem, stream>>>(*a); break;
    case GSB_SPARSE_UNIT_S8_SP: sparse_check<GSB_SPARSE_UNIT_S8_SP><<<grid, kMmaThreads, smem, stream>>>(*a); break;
    case GSB_SPARSE_UNIT_HMMA_SP: sparse_check<GSB_SPARSE_UNIT_HMMA_SP><<<grid, kMmaThreads, smem, stream>>>(*a); break;
    default: return (int)cudaErrorInvalidValue;
  }
  return (int)cudaGetLastError();
}

int gsb_sparse_kernel_preload(int smem_bytes) {
  const void *fns[GSB_SPARSE_UNITS] = {
      (const void *)sparse_check<GSB_SPARSE_UNIT_F16_SP>,  (const void *)sparse_check<GSB_SPARSE_UNIT_BF16_SP>,
      (const void *)sparse_check<GSB_SPARSE_UNIT_TF32_SP>, (const void *)sparse_check<GSB_SPARSE_UNIT_E4M3_SP>,
      (const void *)sparse_check<GSB_SPARSE_UNIT_E5M2_SP>, (const void *)sparse_check<GSB_SPARSE_UNIT_S8_SP>,
      (const void *)sparse_check<GSB_SPARSE_UNIT_HMMA_SP>};
  for (const void *fn : fns) {
    const cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
    if (e != cudaSuccess) return (int)e;
  }
  return (int)cudaSuccess;
}
