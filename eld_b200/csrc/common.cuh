// common.cuh - shared host-side plumbing of libeld_b200.so (error channel, context).
#pragma once
#include <cstdlib>
#include <cuda_runtime.h>
#include <cuda.h>
#include <cstdint>
#include <cstdio>
#include <cstdarg>
#include <atomic>

#include "../../include/eld_b200.h"

namespace eld {

void set_error(const char* fmt, ...);

#define ELD_CHECK_CUDA(expr)                                                                   \
    do {                                                                                       \
        cudaError_t _e = (expr);                                                               \
        if (_e != cudaSuccess) {                                                               \
            ::eld::set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr,                \
                             cudaGetErrorString(_e));                                          \
            return ELD_E_CUDA;                                                                 \
        }                                                                                      \
    } while (0)

#define ELD_REQUIRE(cond, ...)                                                                 \
    do {                                                                                       \
        if (!(cond)) {                                                                         \
            ::eld::set_error(__VA_ARGS__);                                                     \
            return ELD_E_ARG;                                                                  \
        }                                                                                      \
    } while (0)

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                    const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                    const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

}  // namespace eld

struct eld_ctx {
    int device;
    int num_sms;
    int smem_optin;
    eld::PFN_encodeTiled encode_tiled;
    std::atomic<int64_t> launches;
};

namespace eld {
inline void count_launch(eld_ctx* ctx, int n = 1) { ctx->launches.fetch_add(n, std::memory_order_relaxed); }

// whether the byte ranges [a, a + a_bytes) and [b, b + b_bytes) share an address
inline bool ranges_overlap(const void* a, size_t a_bytes, const void* b, size_t b_bytes)
{
    const uintptr_t x = reinterpret_cast<uintptr_t>(a), y = reinterpret_cast<uintptr_t>(b);
    return a_bytes > 0 && b_bytes > 0 && x < y + b_bytes && y < x + a_bytes;
}

// max / clamp that keep NaN, as torch.clamp and np.clip do (fmaxf / fminf return the other operand for a NaN)
__device__ __forceinline__ float fmax_nan(float x, float lo) { return x != x ? x : fmaxf(x, lo); }
__device__ __forceinline__ float clamp_nan(float x, float lo, float hi) { return x != x ? x : fminf(fmaxf(x, lo), hi); }

// Launch with programmatic stream serialization (PDL): the kernel may start while its predecessor drains; it blocks in
// griddepcontrol.wait before touching anything the predecessor writes.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), int grid, int block, size_t smem, cudaStream_t st, Args... args)
{
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3((unsigned)block); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}


// device side of PDL (see wgmma.cuh for the wgmma tiles): wait for the predecessor, then release the successor
__device__ __forceinline__ void pdl_wait_and_release()
{
    asm volatile("griddepcontrol.wait;" ::: "memory");
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
}
}
