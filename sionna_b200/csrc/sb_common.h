// sb_common.h -- error slot, CUDA checks, launch-size helpers and small device helpers shared by all translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <algorithm>
#include <type_traits>
#include "../../include/sionna_b200.h"

// thread-local error message (defined in common.cu)
void sb_set_error(const char* fmt, ...);
void sb_count_launch(void);

#define SB_CHECK_ARG(cond, ...)                  \
    do {                                         \
        if (!(cond)) {                           \
            sb_set_error(__VA_ARGS__);           \
            return SB_EINVAL;                    \
        }                                        \
    } while (0)

#define SB_CUDA(call)                                                                   \
    do {                                                                                \
        cudaError_t e_ = (call);                                                        \
        if (e_ != cudaSuccess) {                                                        \
            sb_set_error("%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
            return SB_ECUDA;                                                            \
        }                                                                               \
    } while (0)

#define SB_LAUNCH_CHECK()                                                                \
    do {                                                                                 \
        cudaError_t e_ = cudaGetLastError();                                             \
        if (e_ != cudaSuccess) {                                                         \
            sb_set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(e_), __FILE__, __LINE__); \
            return SB_ECUDA;                                                             \
        }                                                                                \
        sb_count_launch();                                                               \
    } while (0)

static inline int sb_num_sms(void) {
    int dev = 0, n = 132;
    if (cudaGetDevice(&dev) == cudaSuccess) cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    return n;
}

// Grid of a grid-stride kernel: ceil(items / per_cta) CTAs, at least 1 and at most ctas_per_sm per SM.
static inline int sb_grid(long long items, int per_cta, int ctas_per_sm) {
    const long long ctas = (items + per_cta - 1) / per_cta;
    return (int)std::max<long long>(1, std::min<long long>(ctas, (long long)sb_num_sms() * ctas_per_sm));
}

// Compile-time dispatch of a small runtime integer: f(std::integral_constant<int, v>{}) for v in [LO, HI], whose int
// result is returned; SB_EUNSUPPORTED for any other v.
template <int LO, int HI, class F>
static inline int sb_dispatch(int v, F&& f) {
    if constexpr (LO > HI) {
        return SB_EUNSUPPORTED;
    } else {
        if (v == LO) return f(std::integral_constant<int, LO>{});
        return sb_dispatch<LO + 1, HI>(v, f);
    }
}

// Row-wise element kernels: blockDim = (tx, ty) with tx = row length rounded up to a warp (<= 256) and ty rows per CTA;
// a CTA walks rows (64-bit row index once per row), threads walk columns with 32-bit arithmetic only.
struct RowLaunch { dim3 block; int grid; };
static inline RowLaunch row_launch(long long rows, int cols) {
    const int tx = std::min(256, std::max(32, (cols + 31) / 32 * 32));
    const int ty = std::max(1, 256 / tx);
    return RowLaunch{dim3((unsigned)tx, (unsigned)ty, 1), sb_grid(rows, ty, 16)};
}

// complex float arithmetic
__device__ __forceinline__ float2 cmul(float2 a, float2 b) { return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
__device__ __forceinline__ float2 cmulc(float2 a, float2 b) {   // a * conj(b)
    return make_float2(a.x * b.x + a.y * b.y, a.y * b.x - a.x * b.y);
}
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 cscale(float2 a, float s) { return make_float2(a.x * s, a.y * s); }
__device__ __forceinline__ float2 cdiv(float2 a, float2 b) {
    float d = b.x * b.x + b.y * b.y;
    return make_float2((a.x * b.x + a.y * b.y) / d, (a.y * b.x - a.x * b.y) / d);
}
