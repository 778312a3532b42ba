/*
 * cluster_script_sm90a.cu — test-only twins of the SM-to-SM check's kernels (gsb_test_cluster_script): the shipped body
 * (gsb_cluster_body.inc) in the shipped launch geometry, with the region size and the routes of a gsb_cluster_script
 * read from device memory. Kept out of cluster_check_sm90a.cu so the shipped kernels and their symbols stay as they are,
 * and built as a module of its own (libgpushare_b200_cluster_script.so, with its own static CUDA runtime), which
 * libgpushare_b200.so loads, so the main library's kernel set stays the one its golden SASS records.
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "gsb_cluster.h"
#include "gsb_internal.h"
#include "gsb_pattern.h"

namespace {

#include "gsb_cluster_body.inc"

template <uint32_t P>
__global__ void __launch_bounds__(kThreads, 1) cluster_from_script(const gsb_cluster_args a,
                                                                   const gsb_cluster_script *s) {
  cluster_body<P, true>(a, s);
}

template <uint32_t P>
int launch(uint32_t n, uint32_t clusters, const gsb_cluster_args *a, const gsb_cluster_script *s,
           cudaStream_t stream) {
  cudaLaunchAttribute attr;
  const cudaLaunchConfig_t c = config<P>(n, clusters, a->smem_bytes, stream, &attr);
  const cudaError_t e = cudaLaunchKernelEx(&c, cluster_from_script<P>, *a, s);
  return (int)(e != cudaSuccess ? e : cudaGetLastError());
}

}  // namespace

int gsb_cluster_script_launch(uint32_t path, uint32_t n, uint32_t clusters, const gsb_cluster_args *a,
                              const gsb_cluster_script *s, cudaStream_t stream) {
  if (n < 2 || n > GSB_CLUSTER_MAX_N || (n & (n - 1)) || !clusters || !s) return (int)cudaErrorInvalidValue;
  switch (path) {
    case GSB_CLUSTER_PATH_DSMEM_ST: return launch<GSB_CLUSTER_PATH_DSMEM_ST>(n, clusters, a, s, stream);
    case GSB_CLUSTER_PATH_DSMEM_LD: return launch<GSB_CLUSTER_PATH_DSMEM_LD>(n, clusters, a, s, stream);
    case GSB_CLUSTER_PATH_ST_ASYNC: return launch<GSB_CLUSTER_PATH_ST_ASYNC>(n, clusters, a, s, stream);
    case GSB_CLUSTER_PATH_BULK_S2S: return launch<GSB_CLUSTER_PATH_BULK_S2S>(n, clusters, a, s, stream);
    case GSB_CLUSTER_PATH_MULTICAST: return launch<GSB_CLUSTER_PATH_MULTICAST>(n, clusters, a, s, stream);
    default: return (int)cudaErrorInvalidValue;
  }
}

int gsb_cluster_script_preload(int smem_bytes) {
  const void *fns[GSB_CLUSTER_PATHS] = {
      (const void *)cluster_from_script<GSB_CLUSTER_PATH_DSMEM_ST>,
      (const void *)cluster_from_script<GSB_CLUSTER_PATH_DSMEM_LD>,
      (const void *)cluster_from_script<GSB_CLUSTER_PATH_ST_ASYNC>,
      (const void *)cluster_from_script<GSB_CLUSTER_PATH_BULK_S2S>,
      (const void *)cluster_from_script<GSB_CLUSTER_PATH_MULTICAST>};
  for (const void *fn : fns) {
    cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(fn, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    if (e != cudaSuccess) return (int)e;
  }
  return (int)cudaSuccess;
}
