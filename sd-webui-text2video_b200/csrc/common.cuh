// Shared host-side helpers of the library.
#pragma once
#include <cuda_runtime.h>

namespace t2v {
void set_error(const char* fmt, ...);
int num_sms();
// 0, or -2 after recording what failed and the CUDA error string (so t2v_last_error() never shows a stale message)
int launch_status(const char* what);
// Called at the entry of the public entry points: a non-sticky CUDA error left behind by ANOTHER library of the process (or an
// unchecked call of ours) must not be blamed on the first kernel this call launches.  Reports it on stderr and clears it.
void clear_pending_error(const char* where);

// ---- programmatic dependent launch (PDL), opt-in with T2V_PDL=1
// Every kernel of the library executes griddep_wait() (all prerequisite grids complete, their writes visible) once its
// input-independent prologue is done; the GEMM / attention producers signal griddep_launch() when they have issued their
// last load, so the NEXT kernel of the stream may be scheduled onto SMs as they drain and run ITS prologue (barrier init,
// tensor-map prefetch, index math) under this kernel's tail.  The attribute is NOT set by default (it has not been shown
// to shorten the CUDA-graphed forward); without it the device-side instructions are no-ops.
bool pdl_enabled();
#ifdef __CUDACC__
__device__ __forceinline__ void griddep_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void griddep_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
// short kernels (norms, elementwise, glue): where they release their dependents is a build-time choice for A/B runs
#ifndef T2V_PDL_SMALL_EARLY
#define T2V_PDL_SMALL_EARLY 1
#endif
__device__ __forceinline__ void griddep_launch_small() {
#if T2V_PDL_SMALL_EARLY
    griddep_launch();
#endif
}

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream, Args&&... args) {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid;
    cfg.blockDim = block;
    cfg.dynamicSmemBytes = smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = pdl_enabled() ? 1 : 0;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
#endif
}  // namespace t2v
