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
}  // namespace t2v
