// sb_common.h -- error slot, CUDA checks, launch-size helpers and small device helpers shared by all translation units.
#pragma once
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <algorithm>
#include <memory>
#include <mutex>
#include <type_traits>
#include <vector>
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

// Device copies of a handle's host tables, one per device that has used the handle. The first get() on a device
// allocates and copies every table there: the library's only device allocation and synchronous copy. A copy never
// changes once built, and all copies are freed together, by set() or by the destructor (the handle's *_destroy). So a
// call on one device never frees tables that a kernel on another device may still read, and returning to a device does
// not upload again. Handles hold the store as a `mutable` member, so that decode and encode calls take them const.
class DeviceTables {
  public:
    struct Copy {
        int device = -1, smem_optin = 0, num_sms = 0;
        std::vector<void*> ptr;   // device copy of each table, in the order given to set()
        template <typename T>
        const T* at(size_t i) const { return static_cast<const T*>(ptr[i]); }
    };
    DeviceTables() = default;
    DeviceTables(const DeviceTables&) = delete;
    DeviceTables& operator=(const DeviceTables&) = delete;
    ~DeviceTables() { set(); }

    // Registers the handle's host tables, which must outlive the registration unchanged, and frees every device copy.
    template <typename... T>
    void set(const std::vector<T>&... h) {
        std::lock_guard<std::mutex> lock(mu_);
        for (const auto& c : copies_) free_copy(*c);
        copies_.clear();
        tables_ = {Table{h.data(), h.size() * sizeof(T)}...};
    }

    // The copy on the current device, built on first use. If an allocation or copy fails, whatever that attempt
    // allocated is freed, nothing is recorded and SB_ECUDA is returned; the next call tries again.
    int get(const Copy** out) {
        int dev = 0;
        SB_CUDA(cudaGetDevice(&dev));
        std::lock_guard<std::mutex> lock(mu_);
        if ((*out = lookup(dev))) return SB_OK;
        auto c = std::make_unique<Copy>();
        c->device = dev;
        if (int rc = build(*c)) {
            free_copy(*c);
            return rc;
        }
        copies_.push_back(std::move(c));
        *out = copies_.back().get();
        return SB_OK;
    }

    // The copy on the current device if one has been built, else nullptr.
    const Copy* find() {
        int dev = 0;
        if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
        std::lock_guard<std::mutex> lock(mu_);
        return lookup(dev);
    }

  private:
    struct Table { const void* data; size_t bytes; };

    const Copy* lookup(int dev) const {
        for (const auto& c : copies_)
            if (c->device == dev) return c.get();
        return nullptr;
    }
    int build(Copy& c) const {
        SB_CUDA(cudaDeviceGetAttribute(&c.smem_optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, c.device));
        SB_CUDA(cudaDeviceGetAttribute(&c.num_sms, cudaDevAttrMultiProcessorCount, c.device));
        for (const Table& t : tables_) {
            void* d = nullptr;   // at least one byte, so that an empty table still gets a valid pointer
            SB_CUDA(cudaMalloc(&d, std::max<size_t>(1, t.bytes)));
            c.ptr.push_back(d);
            if (t.bytes) SB_CUDA(cudaMemcpy(d, t.data, t.bytes, cudaMemcpyHostToDevice));
        }
        return SB_OK;
    }
    static void free_copy(const Copy& c) {
        for (void* p : c.ptr) cudaFree(p);
    }

    std::mutex mu_;
    std::vector<Table> tables_;
    std::vector<std::unique_ptr<Copy>> copies_;   // one per device; never moved, so get()'s pointer stays valid
};

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
