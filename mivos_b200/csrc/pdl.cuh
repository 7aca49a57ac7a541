// Programmatic dependent launch (PDL).  The per-frame step is a dependent chain of ~70 short
// kernels; with plain stream order kernel N+1 is only scheduled after kernel N has drained and
// its completion has been processed.  Every kernel of this library is launched with
// cudaLaunchAttributeProgrammaticStreamSerialization and
//   * executes griddepcontrol.launch_dependents first, so the NEXT kernel's CTAs are scheduled as
//     soon as this grid's CTAs have all started and SMs free up, and run their prologue
//     (barrier init, tensor-map prefetch) under this grid's tail;
//   * executes griddepcontrol.wait before its first access to global memory, which blocks until
//     the PREVIOUS grid has completed and its writes are visible — so the data dependences (and
//     the write-after-read ones) of plain stream order are kept.
// Stream capture turns the attribute into programmatic dependency edges of the CUDA graph.
// MIVOS_PDL=0 launches without the attribute (griddepcontrol.* are then no-ops).
#pragma once
#include <cuda_runtime.h>

#include <utility>

namespace mivos {

bool pdl_enabled();  // host_util.cu

__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_prologue() {
  pdl_launch_dependents();
  pdl_wait();
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args&&... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

}  // namespace mivos
