// Programmatic dependent launch (PDL) for the engine's one-stream kernel chain.
//
// An iteration is ~450 dependent launches on ONE stream; with plain
// stream order kernel N+1 is only scheduled once kernel N has fully drained, and its own prologue (block scheduling,
// barrier init, tensor-map prefetch, parameter loads) then runs on an idle GPU.  With the
// programmatic-serialization launch attribute the blocks of kernel N+1 are scheduled as soon as every block of kernel N
// has STARTED (each kernel issues griddepcontrol.launch_dependents first thing) and SM resources free up; they run
// their prologue and park at griddepcontrol.wait, which returns when kernel N has completed and flushed its memory.
//
// Rules every kernel launched through launch_pdl() follows:
//   * pdl_launch_dependents() at the top (the dependents' own griddepcontrol.wait keeps them correct);
//   * pdl_wait() before the first access (read OR write) to memory another kernel of the chain produces or consumes;
//     only kernel parameters, constant weights and the kernel's own shared memory may be touched before it.
// Kernels that are launched the plain way interoperate: they simply serialise fully.  PXR_PDL=0 turns the attribute off.
#pragma once
#include <cuda_runtime.h>
#include <cstdlib>
#include <utility>

namespace pxr {

inline bool pdl_enabled() {
  static const bool on = [] {
    const char* e = getenv("PXR_PDL");
    return !(e && atoi(e) == 0);
  }();
  return on;
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
                              Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = pdl_enabled() ? 1 : 0;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}

#ifdef __CUDACC__
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
// the common case: no prologue worth overlapping beyond block scheduling itself
__device__ __forceinline__ void pdl_prologue() {
  pdl_launch_dependents();
  pdl_wait();
}
#endif

}  // namespace pxr
