// common.cuh -- shared helpers for the sm_90a kernels and the C-ABI glue.
#pragma once

#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>

#include <nvtx3/nvToolsExt.h>

#include "../../include/b200vslam.h"

namespace b200 {

void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what, const char* file, int line);

#define B200_CUDA(expr)                                                          \
    do {                                                                         \
        cudaError_t _e = (expr);                                                 \
        if (_e != cudaSuccess) return ::b200::cuda_fail(_e, #expr, __FILE__, __LINE__); \
    } while (0)

template <typename T>
__host__ __device__ constexpr T ceil_div(T a, T b) {
    return (a + b - 1) / b;
}
template <typename T>
__host__ __device__ constexpr T round_up(T a, T b) {
    return ceil_div(a, b) * b;
}

// NVTX ranges around the host-side phases of every entry point (header-only NVTX 3: a no-op unless a tool is attached; `ncu --nvtx
// --nvtx-include "b200:lba:batch/"` filters a capture by them).  Names: b200:<orb|match|lba|track>:<phase>.
struct NvtxRange {
    explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
    ~NvtxRange() { nvtxRangePop(); }
    NvtxRange(const NvtxRange&) = delete;
    NvtxRange& operator=(const NvtxRange&) = delete;
};
#define B200_CAT2(a, b) a##b
#define B200_CAT(a, b) B200_CAT2(a, b)
#define B200_RANGE(name) ::b200::NvtxRange B200_CAT(b200_nvtx_range_, __LINE__)(name)

// Require a Hopper-class (compute capability 9.x) device; there is no fallback path.
int require_device(int device);

struct StagingArena;  // staging.cuh

namespace lba {
// With the handle's device set: its stream and its staging arena, grown to at least the given sizes (lba_kernels.cu).
int staging(b200_lba_t h, size_t dev_bytes, size_t host_bytes, cudaStream_t* stream, StagingArena** arena);
}

}  // namespace b200
