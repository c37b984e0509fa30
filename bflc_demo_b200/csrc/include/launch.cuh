// Kernel launch helper: cudaLaunchKernelEx with the programmatic-stream-serialization attribute
// (PDL).  A kernel launched this way may begin while its predecessor in the stream is still
// running; it must execute ptx::pdl_wait() before touching memory the predecessor produces
// (all kernels of this library do).  Works under stream capture (programmatic graph edges).
//
// If the runtime rejects a programmatic launch (observed: cudaErrorInvalidValue for some
// launches issued from PyTorch's autograd worker thread), the launch is retried as a plain
// stream-ordered launch and counted in pdl_fallbacks().
#pragma once
#include <cuda_runtime.h>

#include <utility>

#include "bflc_kernels.h"

namespace bflc {

void note_pdl_fallback();

// cluster > 1: the grid is launched as clusters of `cluster` CTAs along x (grid.x a multiple of it)
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl_cluster(unsigned cluster, void (*kernel)(KArgs...), dim3 grid, dim3 block,
                                      size_t smem, cudaStream_t stream, Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  int n = 0;
  if (cluster > 1) {
    attr[n].id = cudaLaunchAttributeClusterDimension;
    attr[n].val.clusterDim.x = cluster; attr[n].val.clusterDim.y = 1; attr[n].val.clusterDim.z = 1;
    ++n;
  }
  const int n_base = n;
  if (pdl_enabled()) {
    attr[n].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[n].val.programmaticStreamSerializationAllowed = 1;
    ++n;
  }
  cfg.attrs = attr;
  cfg.numAttrs = n;
  cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, args...);
  if (e == cudaErrorInvalidValue && cfg.numAttrs != n_base) {
    (void)cudaGetLastError();  // clear, then retry without the PDL attribute
    cfg.numAttrs = n_base;
    note_pdl_fallback();
    e = cudaLaunchKernelEx(&cfg, kernel, args...);
  }
  return e;
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem,
                              cudaStream_t stream, Args&&... args) {
  return launch_pdl_cluster(1u, kernel, grid, block, smem, stream, std::forward<Args>(args)...);
}

}  // namespace bflc
