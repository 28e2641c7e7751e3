// launch.cuh -- programmatic dependent launch (PDL) helpers.
//
// Every kernel of the library begins with pdl_wait() (griddepcontrol.wait: returns once the preceding grid in the
// stream has completed and its writes are visible; a no-op for ordinary launches) placed after any prologue that
// touches no global memory, and calls pdl_trigger() right after it so that the NEXT kernel may be scheduled and run
// its own prologue (barrier init, shared-memory tables) while this one is still computing.
// With ~25 short kernels per SGD step the launch gaps are a large fraction of the step.  XTB_PDL=0 disables it.
#pragma once
#include <cuda_runtime.h>
#include <cstdlib>

namespace xtb {

__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

inline int g_pdl = [] { const char* e = getenv("XTB_PDL"); return e ? atoi(e) : 1; }();

template <class... KArgs, class... Args>
static inline cudaError_t pdl_launch(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = g_pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

}  // namespace xtb

#define XLAUNCH(kernel, grid, block, smem, stream, ...) \
  (void)::xtb::pdl_launch(kernel, dim3(grid), dim3(block), (size_t)(smem), stream, __VA_ARGS__)
