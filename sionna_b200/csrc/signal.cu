// signal.cu -- direct-form FIR convolution with on-chip tap preparation (signal/utils.py:11-159, Filter.call
// signal/filter.py:268-285), window scaling (Window.call signal/window.py:145-163) and the row mean of |X|^2 behind
// empirical_psd (signal/utils.py:251-311), DESIGN §3.14.
//
// Convolution. y[r, m] = sum_k h'[k] x[r, m + offset - k], x = 0 outside [0, N), for m in [0, out_len). One CTA
// computes a tile of W = tpr * R consecutive outputs for each of G rows (G * tpr = kThreads): thread t owns R
// consecutive outputs of its row and keeps R samples of x in a register window that slides by one sample per tap, so
// each shared load of x feeds R FMAs (2 R for complex x or h, 4 R for both). R is odd, so the lanes' shared addresses
// (stride R) fall in distinct banks. Taps are processed in chunks, so any K works: a step (tile, chunk) needs the
// chunk's prepared taps (reversed) and, per row, the W + chunk - 1 samples of x they touch. Steps run through two
// shared-memory stages: while one step computes, the next step's x arrives by cp.async and its taps are written. Rows
// are int64 and tiles are handed out by a grid-stride loop, so the grid never depends on the row count.
//
// Tap preparation. Every CTA builds h' itself from the raw coefficients: h w~ (w~ = w / sqrt(mean(w^2)) when the
// window is normalised), divided by sqrt(sum |h w~|^2) when normalised, conjugated on request. Both sums are reduced in
// one fixed order (thread t sums k = t, t + kThreads, ..., then a fixed tree), so every CTA holds bit-identical taps.
#include "sb_common.h"
#include <math.h>
#include <stdint.h>

namespace {

constexpr int kThreads = 256;
constexpr int kR = 9;                    // outputs per thread (odd: conflict-free shared loads)
constexpr int kStageBytes = 40960;       // staged x per pipeline stage (all rows of a step)
constexpr int kRowsPerChunk = 1024;      // power mean: rows summed by one partial
constexpr int kFlags = SB_CONV_WINDOW_NORMALIZE | SB_CONV_NORMALIZE | SB_CONV_CONJUGATE;

template <typename T> struct Vec2;
template <> struct Vec2<float> { using type = float2; };
template <> struct Vec2<double> { using type = double2; };

template <typename T, bool C> struct Elem { using type = T; };
template <typename T> struct Elem<T, true> { using type = typename Vec2<T>::type; };

template <typename T> __device__ __forceinline__ T re(T v) { return v; }
template <typename T> __device__ __forceinline__ T im(T) { return T(0); }
__device__ __forceinline__ float re(float2 v) { return v.x; }
__device__ __forceinline__ float im(float2 v) { return v.y; }
__device__ __forceinline__ double re(double2 v) { return v.x; }
__device__ __forceinline__ double im(double2 v) { return v.y; }

template <typename E> __device__ __forceinline__ E zero() { return E{}; }

// sum over the CTA of v, in a fixed order: per thread as given, then a binary tree over kThreads values.
template <typename T>
__device__ T cta_sum(T v, T* red) {
    red[threadIdx.x] = v;
    __syncthreads();
    for (int s = kThreads / 2; s > 0; s >>= 1) {
        if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
    }
    const T out = red[0];
    __syncthreads();
    return out;
}

// 1 / sqrt(mean(w^2)) of the window, 1 if not normalised. (Scales are applied as products with one reciprocal: a
// division per element would be a slow-path call that costs registers.)
template <typename T>
__device__ T window_inv_rms(const T* __restrict__ w, int k, bool normalize, T* red) {
    if (!w || !normalize) return T(1);
    T s = T(0);
    for (int i = threadIdx.x; i < k; i += kThreads) s += w[i] * w[i];
    return T(1) / sqrt(cta_sum(s, red) / T(k));
}

// Raw tap i times the (normalised) window, in the reference's order: w~ = w / rms, then h w~.
template <typename T, bool HC>
__device__ __forceinline__ typename Elem<T, HC>::type windowed_tap(const typename Elem<T, HC>::type* __restrict__ h,
                                                                   const T* __restrict__ w, T winv, int i) {
    typename Elem<T, HC>::type v = h[i];
    if (w) {
        const T wi = w[i] * winv;
        if constexpr (HC) { v.x *= wi; v.y *= wi; } else { v *= wi; }
    }
    return v;
}

// Asynchronous copy of one element to shared memory; src_bytes = 0 writes zeros (the padding outside x).
template <typename X>
__device__ __forceinline__ void cp_async(X* dst, const X* src, bool valid) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], %2, %3;\n" ::"r"(d), "l"(src), "n"((int)sizeof(X)),
                 "r"(valid ? (int)sizeof(X) : 0));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
__device__ __forceinline__ void cp_async_wait_prev() { asm volatile("cp.async.wait_group 1;\n" ::); }

template <typename T, bool XC, bool HC>
__global__ void __launch_bounds__(kThreads, 2) conv_kernel(const typename Elem<T, XC>::type* __restrict__ x,
                                                        const typename Elem<T, HC>::type* __restrict__ h,
                                                        const T* __restrict__ w,
                                                        typename Elem<T, XC || HC>::type* __restrict__ y,
                                                        long long rows, int n, int k, int offset, int out_len,
                                                        int flags, int tpr, int kcp_max, int buf_bytes) {
    using X = typename Elem<T, XC>::type;
    using H = typename Elem<T, HC>::type;
    using Y = typename Elem<T, XC || HC>::type;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __shared__ T red[kThreads];
    const int g_rows = kThreads / tpr;                         // rows per CTA
    const int w_out = tpr * kR;                                // outputs per row per tile
    const int ls = w_out + ((kcp_max + 31) & ~31);             // row stride of staged x (== w_out mod 32: no conflicts)
    const size_t tap_bytes = ((size_t)kcp_max * sizeof(H) + 15) & ~(size_t)15;
    // two stages, each: [kcp_max] reversed prepared taps of a chunk, then the x rows (later the output tile)
    const size_t stage_bytes = tap_bytes + buf_bytes;
    auto sh = [&](int b) { return reinterpret_cast<H*>(smem_raw + b * stage_bytes); };
    auto sx = [&](int b) { return reinterpret_cast<X*>(smem_raw + b * stage_bytes + tap_bytes); };

    // ---- prologue: normalisation constants of h' (identical in every CTA) ----
    const T winv = window_inv_rms(w, k, (flags & SB_CONV_WINDOW_NORMALIZE) != 0, red);
    T hinv = T(1);
    if (flags & SB_CONV_NORMALIZE) {
        T s = T(0);
        for (int i = threadIdx.x; i < k; i += kThreads) {
            const H v = windowed_tap<T, HC>(h, w, winv, i);
            s += re(v) * re(v) + im(v) * im(v);
        }
        hinv = T(1) / sqrt(cta_sum(s, red));
    }
    const bool conj = HC && (flags & SB_CONV_CONJUGATE);

    const int g = threadIdx.x / tpr, tl = threadIdx.x % tpr;   // row in the CTA, thread in the row
    const int p0 = tl * kR;                                    // first output of this thread in the tile
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    constexpr int kWarps = kThreads / 32;
    const int wpr = g_rows >= kWarps ? 1 : kWarps / g_rows;   // warps per row when staging / storing
    const long long groups = (rows + g_rows - 1) / g_rows;
    const long long tiles_per_row = (out_len + w_out - 1) / w_out;
    const long long tiles = groups * tiles_per_row;
    const int chunks = (k + kcp_max - 1) / kcp_max;

    // Stage step (tile, chunk c) into buffer b: its taps (plain stores) and its x samples (asynchronous copies).
    auto stage = [&](long long tile, int c, int b) {
        const int k0 = c * kcp_max, kc = min(kcp_max, k - k0), kcp = (kc + kR - 1) / kR * kR;
        for (int q = threadIdx.x; q < kcp; q += kThreads) {
            const int kk = k0 + kcp - 1 - q;                   // tap of reversed slot q
            H v = zero<H>();
            if (kk < k0 + kc) {
                v = windowed_tap<T, HC>(h, w, winv, kk);
                if constexpr (HC) {
                    v.x *= hinv;
                    v.y = conj ? -(v.y * hinv) : v.y * hinv;
                } else {
                    v *= hinv;
                }
            }
            sh(b)[q] = v;
        }
        const long long row0 = (tile / tiles_per_row) * g_rows;
        const int m0 = (int)(tile % tiles_per_row) * w_out;
        const long long base = (long long)m0 + offset - k0 - kcp + 1;   // x index of row 0 of sx(b)
        const int seg = w_out + kcp;
        for (int gg = warp / wpr; gg < g_rows; gg += kWarps / wpr) {
            const long long row = row0 + gg;
            for (int j = (warp % wpr) * 32 + lane; j < seg; j += wpr * 32) {
                const long long i = base + j;
                const bool valid = row < rows && i >= 0 && i < n;
                cp_async(&sx(b)[gg * ls + j], valid ? x + row * (long long)n + i : x, valid);
            }
        }
        cp_async_commit();
    };

    Y acc[kR];
    long long tile = blockIdx.x;
    int c = 0, b = 0;
    if (tile < tiles) stage(tile, 0, 0);
    while (tile < tiles) {
        long long next = tile;                                 // the step after this one: next chunk, or next tile
        int nc = c + 1;
        if (nc == chunks) {
            nc = 0;
            next += gridDim.x;
        }
        if (next < tiles) stage(next, nc, b ^ 1);
        else cp_async_commit();                                // an empty group keeps the wait below uniform
        cp_async_wait_prev();                                  // this step's copies have landed (the next may not)
        __syncthreads();
        if (c == 0) {
#pragma unroll
            for (int r = 0; r < kR; ++r) acc[r] = zero<Y>();
        }
        const int kcp = (min(kcp_max, k - c * kcp_max) + kR - 1) / kR * kR;
        const H* sht = sh(b);
        const X* sxt = sx(b) + g * ls + p0;
        X win[kR];
#pragma unroll
        for (int r = 0; r < kR; ++r) win[r] = sxt[r];
        for (int q0 = 0; q0 < kcp; q0 += kR) {
#pragma unroll
            for (int u = 0; u < kR; ++u) {
                const H t = sht[q0 + u];
#pragma unroll
                for (int r = 0; r < kR; ++r) {
                    const X xv = win[(u + r) % kR];
                    if constexpr (XC && HC) {
                        acc[r].x = fma(re(t), xv.x, acc[r].x);
                        acc[r].x = fma(-im(t), xv.y, acc[r].x);
                        acc[r].y = fma(re(t), xv.y, acc[r].y);
                        acc[r].y = fma(im(t), xv.x, acc[r].y);
                    } else if constexpr (XC) {
                        acc[r].x = fma(t, xv.x, acc[r].x);
                        acc[r].y = fma(t, xv.y, acc[r].y);
                    } else if constexpr (HC) {
                        acc[r].x = fma(t.x, xv, acc[r].x);
                        acc[r].y = fma(t.y, xv, acc[r].y);
                    } else {
                        acc[r] = fma(t, xv, acc[r]);
                    }
                }
                win[u] = sxt[q0 + u + kR];                     // slot u now holds the sample after the window
            }
        }
        if (c == chunks - 1) {                                 // tile done: out through shared memory, coalesced
            Y* sy = reinterpret_cast<Y*>(sx(b));
            __syncthreads();                                   // everyone done reading sx[b] before it becomes sy
#pragma unroll
            for (int r = 0; r < kR; ++r) sy[g * w_out + p0 + r] = acc[r];
            __syncthreads();
            const long long row0 = (tile / tiles_per_row) * g_rows;
            const int m0 = (int)(tile % tiles_per_row) * w_out;
            const int wn = min(w_out, out_len - m0);
            for (int gg = warp / wpr; gg < g_rows; gg += kWarps / wpr) {
                const long long row = row0 + gg;
                if (row >= rows) break;
                Y* yr = y + row * (long long)out_len + m0;
                for (int j = (warp % wpr) * 32 + lane; j < wn; j += wpr * 32) yr[j] = sy[gg * w_out + j];
            }
        }
        __syncthreads();                                       // buffer b is free for the step after next
        tile = next;
        c = nc;
        b ^= 1;
    }
}

template <typename T, bool XC>
__global__ void __launch_bounds__(kThreads) scale_last_kernel(const typename Elem<T, XC>::type* __restrict__ x,
                                                              const T* __restrict__ w,
                                                              typename Elem<T, XC>::type* __restrict__ y,
                                                              long long rows, int n, int normalize) {
    __shared__ T red[kThreads];
    const T winv = window_inv_rms(w, n, normalize != 0, red);
    for (long long r = blockIdx.y; r < rows; r += gridDim.y)
        for (int j = blockIdx.x * kThreads + threadIdx.x; j < n; j += gridDim.x * kThreads) {
            const T wj = w[j] * winv;
            auto v = x[r * n + j];
            if constexpr (XC) { v.x *= wj; v.y *= wj; } else { v *= wj; }
            y[r * n + j] = v;
        }
}

// Partial sums of |x|^2 over row chunk blockIdx.y (kRowsPerChunk rows) for 32 columns: lane = column, warp w sums rows
// w, w + 8, ... of the chunk in order, then warps are added in order. One chunk: the mean is written directly.
__global__ void __launch_bounds__(kThreads) power_partial_kernel(const float2* __restrict__ x, float* __restrict__ out,
                                                                 long long rows, int n, int chunks) {
    __shared__ float part[kThreads / 32][32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int col = blockIdx.x * 32 + lane;
    for (long long c = blockIdx.y; c < chunks; c += gridDim.y) {
        const long long r0 = c * kRowsPerChunk, r1 = min(rows, r0 + kRowsPerChunk);
        float s = 0.f;
        if (col < n)
            for (long long r = r0 + warp; r < r1; r += kThreads / 32) {
                const float2 v = x[r * n + col];
                s += v.x * v.x + v.y * v.y;
            }
        part[warp][lane] = s;
        __syncthreads();
        if (warp == 0 && col < n) {
            float t = part[0][lane];
#pragma unroll
            for (int i = 1; i < kThreads / 32; ++i) t += part[i][lane];
            if (chunks == 1) out[col] = t / (float)rows;
            else out[c * n + col] = t;
        }
        __syncthreads();
    }
}

__global__ void power_final_kernel(const float* __restrict__ part, float* __restrict__ psd, long long rows, int n,
                                   int chunks) {
    for (int col = blockIdx.x * blockDim.x + threadIdx.x; col < n; col += gridDim.x * blockDim.x) {
        float t = 0.f;
        for (int c = 0; c < chunks; ++c) t += part[(long long)c * n + col];
        psd[col] = t / (float)rows;
    }
}

// Host plan of a convolution launch: threads per row (power of two), the tap chunk and the shared memory of one stage.
struct ConvPlan {
    int tpr, kcp_max, buf_bytes;
    size_t smem;
};

ConvPlan conv_plan(int k, int out_len, size_t xs, size_t hs, size_t ys) {
    const int budget = (int)(kStageBytes / xs);              // staged x elements per stage (all rows)
    int tpr = 1;
    while (tpr < kThreads && tpr * kR < out_len) tpr <<= 1;
    const int kpad = (k + kR - 1) / kR * kR;
    for (;; tpr <<= 1) {
        const int g = kThreads / tpr, w = tpr * kR;
        const int avail = (budget / g - w) & ~31;              // per-row room for the chunk, multiple of 32
        const int kcp = std::min(kpad, avail / kR * kR);
        if (kcp >= kR || tpr == kThreads) {
            const int ls = w + ((kcp + 31) & ~31);
            const size_t buf = (std::max((size_t)g * ls * xs, (size_t)kThreads * kR * ys) + 15) & ~(size_t)15;
            const size_t taps = ((size_t)kcp * hs + 15) & ~(size_t)15;
            return ConvPlan{tpr, kcp, (int)buf, 2 * (taps + buf)};
        }
    }
}

template <typename T, bool XC, bool HC>
int launch_conv(const void* x, const void* h, const void* w, void* y, long long rows, int n, int k, int offset,
                int out_len, int flags, cudaStream_t st) {
    using X = typename Elem<T, XC>::type;
    using H = typename Elem<T, HC>::type;
    using Y = typename Elem<T, XC || HC>::type;
    const ConvPlan p = conv_plan(k, out_len, sizeof(X), sizeof(H), sizeof(Y));
    auto kern = conv_kernel<T, XC, HC>;
    SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem));
    const long long g = kThreads / p.tpr, w_out = (long long)p.tpr * kR;
    const long long tiles = (rows + g - 1) / g * ((out_len + w_out - 1) / w_out);
    kern<<<sb_grid(tiles, 1, 16), kThreads, p.smem, st>>>((const X*)x, (const H*)h, (const T*)w, (Y*)y, rows, n, k,
                                                          offset, out_len, flags, p.tpr, p.kcp_max, p.buf_bytes);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

template <typename T>
int launch_conv_t(int xc, int hc, const void* x, const void* h, const void* w, void* y, long long rows, int n, int k,
                  int offset, int out_len, int flags, cudaStream_t st) {
    if (xc && hc) return launch_conv<T, true, true>(x, h, w, y, rows, n, k, offset, out_len, flags, st);
    if (xc) return launch_conv<T, true, false>(x, h, w, y, rows, n, k, offset, out_len, flags, st);
    if (hc) return launch_conv<T, false, true>(x, h, w, y, rows, n, k, offset, out_len, flags, st);
    return launch_conv<T, false, false>(x, h, w, y, rows, n, k, offset, out_len, flags, st);
}

int power_chunks(long long rows) { return (int)std::max<long long>(1, (rows + kRowsPerChunk - 1) / kRowsPerChunk); }

}  // namespace

extern "C" int sb_convolve(const void* d_x, int32_t x_complex, const void* d_h, int32_t h_complex, const void* d_w,
                           void* d_y, int32_t precision, int64_t rows, int32_t n, int32_t k, int32_t offset,
                           int32_t out_len, int32_t flags, void* stream) {
    const char* who = "sb_convolve";
    SB_CHECK_ARG(rows >= 0 && n >= 1 && k >= 1 && out_len >= 0, "%s: bad shape (rows >= 0, n >= 1, k >= 1, "
                 "out_len >= 0; got rows %lld, n %d, k %d, out_len %d)", who, (long long)rows, n, k, out_len);
    SB_CHECK_ARG(offset >= 0 && offset <= k - 1, "%s: offset = %d outside [0, k - 1 = %d]", who, offset, k - 1);
    SB_CHECK_ARG((long long)out_len <= (long long)n + k - 1 - offset, "%s: out_len = %d > n + k - 1 - offset = %lld",
                 who, out_len, (long long)n + k - 1 - offset);
    SB_CHECK_ARG((flags & ~kFlags) == 0, "%s: unknown flag bits 0x%x", who, flags & ~kFlags);
    SB_CHECK_ARG(precision == 0 || precision == 1, "%s: precision = %d, supported are 0 float32, 1 float64", who,
                 precision);
    SB_CHECK_ARG((x_complex == 0 || x_complex == 1) && (h_complex == 0 || h_complex == 1),
                 "%s: x_complex and h_complex must be 0 or 1", who);
    SB_CHECK_ARG(!(flags & SB_CONV_WINDOW_NORMALIZE) || d_w, "%s: window normalisation without a window", who);
    if (rows == 0) return SB_OK;
    SB_CHECK_ARG(d_x && d_h && d_y, "%s: missing input, taps or output", who);
    if (out_len == 0) return SB_OK;
    cudaStream_t st = (cudaStream_t)stream;
    return precision ? launch_conv_t<double>(x_complex, h_complex, d_x, d_h, d_w, d_y, rows, n, k, offset, out_len,
                                             flags, st)
                     : launch_conv_t<float>(x_complex, h_complex, d_x, d_h, d_w, d_y, rows, n, k, offset, out_len,
                                            flags, st);
}

extern "C" int sb_scale_last(const void* d_x, int32_t x_complex, const void* d_w, void* d_y, int32_t precision,
                             int64_t rows, int32_t n, int32_t normalize, void* stream) {
    const char* who = "sb_scale_last";
    SB_CHECK_ARG(rows >= 0 && n >= 1, "%s: bad shape (rows >= 0, n >= 1; got rows %lld, n %d)", who,
                 (long long)rows, n);
    SB_CHECK_ARG(precision == 0 || precision == 1, "%s: precision = %d, supported are 0 float32, 1 float64", who,
                 precision);
    SB_CHECK_ARG(x_complex == 0 || x_complex == 1, "%s: x_complex must be 0 or 1", who);
    SB_CHECK_ARG(normalize == 0 || normalize == 1, "%s: normalize must be 0 or 1", who);
    if (rows == 0) return SB_OK;
    SB_CHECK_ARG(d_x && d_w && d_y, "%s: missing input, window or output", who);
    const unsigned gx = (unsigned)std::min((n + kThreads - 1) / kThreads, 64);
    const dim3 grid(gx, (unsigned)std::max<long long>(1, std::min<long long>(rows, sb_num_sms() * 16LL / gx)));
    cudaStream_t st = (cudaStream_t)stream;
    if (precision == 0 && x_complex == 0)
        scale_last_kernel<float, false><<<grid, kThreads, 0, st>>>((const float*)d_x, (const float*)d_w, (float*)d_y,
                                                                  rows, n, normalize);
    else if (precision == 0)
        scale_last_kernel<float, true><<<grid, kThreads, 0, st>>>((const float2*)d_x, (const float*)d_w, (float2*)d_y,
                                                                 rows, n, normalize);
    else if (x_complex == 0)
        scale_last_kernel<double, false><<<grid, kThreads, 0, st>>>((const double*)d_x, (const double*)d_w,
                                                                   (double*)d_y, rows, n, normalize);
    else
        scale_last_kernel<double, true><<<grid, kThreads, 0, st>>>((const double2*)d_x, (const double*)d_w,
                                                                  (double2*)d_y, rows, n, normalize);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" size_t sb_power_mean_workspace_bytes(int64_t rows, int32_t n) {
    if (rows <= 0 || n <= 0) return 0;
    const int chunks = power_chunks(rows);
    return chunks == 1 ? 0 : (size_t)chunks * (size_t)n * sizeof(float);
}

extern "C" int sb_power_mean(const float* d_x, float* d_psd, int64_t rows, int32_t n, void* d_workspace,
                             size_t workspace_bytes, void* stream) {
    const char* who = "sb_power_mean";
    SB_CHECK_ARG(rows >= 1 && n >= 1, "%s: bad shape (rows >= 1, n >= 1; got rows %lld, n %d)", who,
                 (long long)rows, n);
    SB_CHECK_ARG(d_x && d_psd, "%s: missing input or output", who);
    const size_t need = sb_power_mean_workspace_bytes(rows, n);
    if (workspace_bytes < need || (need && !d_workspace)) {
        sb_set_error("%s: workspace of %zu bytes, %zu needed", who, workspace_bytes, need);
        return SB_ENOMEM;
    }
    const int chunks = power_chunks(rows);
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned cols = (unsigned)((n + 31) / 32);
    const unsigned ychunks = (unsigned)std::min<long long>(chunks, 65535);
    power_partial_kernel<<<dim3(cols, ychunks), kThreads, 0, st>>>((const float2*)d_x,
                                                                   chunks == 1 ? d_psd : (float*)d_workspace, rows, n,
                                                                   chunks);
    SB_LAUNCH_CHECK();
    if (chunks > 1) {
        power_final_kernel<<<(n + kThreads - 1) / kThreads, kThreads, 0, st>>>((const float*)d_workspace, d_psd, rows,
                                                                              n, chunks);
        SB_LAUNCH_CHECK();
    }
    return SB_OK;
}
