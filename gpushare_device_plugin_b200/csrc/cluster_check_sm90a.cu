/*
 * cluster_check_sm90a.cu — the SM-to-SM check's kernels (gsb_cluster_probe): bit-exact transfers between the CTAs of a
 * thread-block cluster over the SM-to-SM network, one kernel per path. Host code lives in gsb_device.cu (the probe) and
 * gsb_cluster.cc (policy, classification, text); the geometry and the words are defined in gsb_cluster.h.
 *
 * The kernel body and its device helpers are in gsb_cluster_body.inc, which the test-only twins
 * (cluster_script_sm90a.cu) share.
 */
#include <cuda_runtime.h>
#include <stdint.h>

#include "gsb_cluster.h"
#include "gsb_internal.h"
#include "gsb_pattern.h"

namespace {

#include "gsb_cluster_body.inc"

template <uint32_t P>
__global__ void __launch_bounds__(kThreads, 1) cluster_check(const gsb_cluster_args a) {
  cluster_body<P, false>(a, nullptr);
}

template <uint32_t P>
int launch(uint32_t n, uint32_t clusters, const gsb_cluster_args *a, cudaStream_t stream) {
  cudaLaunchAttribute attr;
  const cudaLaunchConfig_t c = config<P>(n, clusters, a->smem_bytes, stream, &attr);
  const cudaError_t e = cudaLaunchKernelEx(&c, cluster_check<P>, *a);
  return (int)(e != cudaSuccess ? e : cudaGetLastError());
}

}  // namespace

int gsb_cluster_kernel_launch(uint32_t path, uint32_t n, uint32_t clusters, const gsb_cluster_args *a,
                              cudaStream_t stream) {
  if (n < 2 || n > GSB_CLUSTER_MAX_N || (n & (n - 1)) || !clusters) return (int)cudaErrorInvalidValue;
  switch (path) {
    case GSB_CLUSTER_PATH_DSMEM_ST: return launch<GSB_CLUSTER_PATH_DSMEM_ST>(n, clusters, a, stream);
    case GSB_CLUSTER_PATH_DSMEM_LD: return launch<GSB_CLUSTER_PATH_DSMEM_LD>(n, clusters, a, stream);
    case GSB_CLUSTER_PATH_ST_ASYNC: return launch<GSB_CLUSTER_PATH_ST_ASYNC>(n, clusters, a, stream);
    case GSB_CLUSTER_PATH_BULK_S2S: return launch<GSB_CLUSTER_PATH_BULK_S2S>(n, clusters, a, stream);
    case GSB_CLUSTER_PATH_MULTICAST: return launch<GSB_CLUSTER_PATH_MULTICAST>(n, clusters, a, stream);
    default: return (int)cudaErrorInvalidValue;
  }
}

int gsb_cluster_max_active(uint32_t n, int smem_bytes, int *clusters) {
  cudaLaunchAttribute attr;
  const cudaLaunchConfig_t c = config<GSB_CLUSTER_PATH_DSMEM_ST>(n, 1, (uint32_t)smem_bytes, nullptr, &attr);
  *clusters = 0;
  return (int)cudaOccupancyMaxActiveClusters(clusters, (const void *)cluster_check<GSB_CLUSTER_PATH_DSMEM_ST>, &c);
}

int gsb_cluster_kernel_preload(int smem_bytes) {
  const void *fns[GSB_CLUSTER_PATHS] = {
      (const void *)cluster_check<GSB_CLUSTER_PATH_DSMEM_ST>, (const void *)cluster_check<GSB_CLUSTER_PATH_DSMEM_LD>,
      (const void *)cluster_check<GSB_CLUSTER_PATH_ST_ASYNC>, (const void *)cluster_check<GSB_CLUSTER_PATH_BULK_S2S>,
      (const void *)cluster_check<GSB_CLUSTER_PATH_MULTICAST>};
  for (const void *fn : fns) {
    cudaError_t e = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(fn, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
    if (e != cudaSuccess) return (int)e;
  }
  return (int)cudaSuccess;
}
