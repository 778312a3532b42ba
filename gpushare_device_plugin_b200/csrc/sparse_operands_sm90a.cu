/*
 * sparse_operands_sm90a.cu — test-only twins of the sparse tensor-core check's kernels (gsb_test_sparse_operands): the
 * same instruction, layout, metadata packing and compare as sparse_check<UNIT> (the body is gsb_sparse_mma.h), on
 * integers, patterns and scales a test chose, read from the table after the 8192 expected words instead of generated
 * from the seed. The probe (gsb_device.cu) launches a twin for every launch of a unit whose chosen operands are armed.
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "gsb_sparse_mma.h"

namespace {

template <uint32_t UNIT>
__global__ void __launch_bounds__(kMmaThreads) sparse_from_table(const gsb_sm_args a) {
  sparse_check_body<UNIT, true>(a);  // operands and patterns from the table after the expected words
}

}  // namespace

int gsb_sparse_operands_launch(uint32_t unit, uint32_t grid, const gsb_sm_args *a, cudaStream_t stream) {
  const size_t smem = a->smem_bytes;
  switch (unit) {
    case GSB_SPARSE_UNIT_F16_SP: sparse_from_table<GSB_SPARSE_UNIT_F16_SP><<<grid, kMmaThreads, smem, stream>>>(*a); break;
    case GSB_SPARSE_UNIT_BF16_SP: sparse_from_table<GSB_SPARSE_UNIT_BF16_SP><<<grid, kMmaThreads, smem, stream>>>(*a); break;
    case GSB_SPARSE_UNIT_TF32_SP: sparse_from_table<GSB_SPARSE_UNIT_TF32_SP><<<grid, kMmaThreads, smem, stream>>>(*a); break;
    case GSB_SPARSE_UNIT_E4M3_SP: sparse_from_table<GSB_SPARSE_UNIT_E4M3_SP><<<grid, kMmaThreads, smem, stream>>>(*a); break;
    case GSB_SPARSE_UNIT_E5M2_SP: sparse_from_table<GSB_SPARSE_UNIT_E5M2_SP><<<grid, kMmaThreads, smem, stream>>>(*a); break;
    case GSB_SPARSE_UNIT_S8_SP: sparse_from_table<GSB_SPARSE_UNIT_S8_SP><<<grid, kMmaThreads, smem, stream>>>(*a); break;
    case GSB_SPARSE_UNIT_HMMA_SP: sparse_from_table<GSB_SPARSE_UNIT_HMMA_SP><<<grid, kMmaThreads, smem, stream>>>(*a); break;
    default: return (int)cudaErrorInvalidValue;
  }
  return (int)cudaGetLastError();
}

int gsb_sparse_operands_preload(int smem_bytes) {
  const void *fns[GSB_SPARSE_UNITS] = {
      (const void *)sparse_from_table<GSB_SPARSE_UNIT_F16_SP>,  (const void *)sparse_from_table<GSB_SPARSE_UNIT_BF16_SP>,
      (const void *)sparse_from_table<GSB_SPARSE_UNIT_TF32_SP>, (const void *)sparse_from_table<GSB_SPARSE_UNIT_E4M3_SP>,
      (const void *)sparse_from_table<GSB_SPARSE_UNIT_E5M2_SP>, (const void *)sparse_from_table<GSB_SPARSE_UNIT_S8_SP>,
      (const void *)sparse_from_table<GSB_SPARSE_UNIT_HMMA_SP>};
  for (const void *fn : fns) {
    const cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
    if (e != cudaSuccess) return (int)e;
  }
  return (int)cudaSuccess;
}
