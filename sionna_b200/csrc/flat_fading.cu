// flat_fading.cu -- flat-fading MIMO channels for sm_90a: draw, spatially correlate and apply a channel matrix in one
// launch, and the Cholesky factors of the correlation matrices. Replaces (paths under the reference's
// src/sionna/phy/channel/):
//   sb_flat_fading   GenerateFlatFadingChannel.call   flat_fading_channel.py:63-72
//                    ApplyFlatFadingChannel.call      flat_fading_channel.py:123-131
//                    FlatFadingChannel.call           flat_fading_channel.py:235-246
//                    KroneckerModel.__call__          spatial_correlation.py:113-122
//                    PerColumnModel.__call__          spatial_correlation.py:185-195
//   sb_chol_lower    tf.linalg.cholesky of the correlation matrices (the models above)
//
// Randomness. h is drawn with sb_awgn's counter convention over the flat [num, M, K] index: element i takes Philox block
// i / 2 and the Box-Muller pair of words (x, y) for an even i, (z, w) for an odd one, scaled as sb_awgn scales unit
// noise (0 + (g * sqrt(1/2)) * sqrt(1)). The noise of y takes the same convention over the flat [num, M] index with
// sqrt(no) as the scale. This file is built with -fmad=false, as phy_kernels.cu is, so that
//   drawn h          == complex_normal([num, M, K])             bit for bit (same seed and offset),
//   y with noise     == sb_awgn(y without noise, no)            bit for bit,
// and every path that forms y = h x (drawn or given h, correlated in shared memory or not) sums the K products in the
// same order with the same roundings.
#include "sb_common.h"
#include "rng.cuh"
#include "dense_mimo.cuh"

namespace {

constexpr float kHalfStd = 0.70710678118654752f;     // sqrt(1/2): CN(0, 1) has variance 1/2 per real dimension
constexpr int kMaxCorrDim = 128;                     // M with an rx factor, K with a tx factor (as sb_spatial_corr)
constexpr int kTileElems = 4096;                     // elements of h staged per CTA when a tile holds several problems
constexpr int kPerThread = 16;                       // elements of h one thread updates per correlation step
constexpr int kInRegs = 8;                           // of which held in registers; the rest wait in shared memory
constexpr int kMaxTileElems = 1024 * kPerThread;     // 16384 = 128 x 128: one problem per CTA at the largest shape

struct FfArgs {
    const float2* h_in;  long long h_stride;         // given h [*, M, K] (stride 0 or 1 matrix per problem), or NULL
    unsigned long long seed_h, off_h;                // draw of h when h_in is NULL
    const float2* l_tx;  long long tx_stride;        // L_tx [*, K, K], or NULL
    const float2* l_rx;  long long rx_stride;        // L_rx [*, M, M] or, per_column, [*, K, M, M]; or NULL
    int per_column;
    float2* h_out;                                   // [num, M, K] or NULL
    const float2* x;     long long x_stride;         // [*, K] or NULL
    const float* no;     long long no_inner;         // noise variance of y element i: no[i / no_inner]; NULL: none
    unsigned long long seed_n, off_n;
    float2* y;                                       // [num, M] when x is given
    long long num;
    int M, K;
};

// element i of the unit-variance complex normal stream (seed, off), given the Philox block of i / 2
__device__ __forceinline__ float2 cn_from_block(uint4 r, unsigned long long i) {
    const float2 g = (i & 1) ? box_muller(r.z, r.w) : box_muller(r.x, r.y);
    return make_float2(0.f + g.x * kHalfStd, 0.f + g.y * kHalfStd);   // sb_awgn on x = 0, no = 1
}

// a / b for a >= 0, b >= 1 with a 32-bit division when both fit (a 64-bit one costs several times more instructions)
__device__ __forceinline__ long long idx_div(long long a, long long b) {
    return ((a | b) >> 32) == 0 ? (long long)((unsigned)a / (unsigned)b) : a / b;
}

// y[row] = acc (+ noise), acc = sum_k h[k] x[k] accumulated with `mac` in k order: the one order of operations of
// every path
__device__ __forceinline__ float2 mac(float2 acc, float2 h, float2 x) { return cadd(acc, cmul(h, x)); }
__device__ __forceinline__ void store_y(const FfArgs& a, long long row, float2 acc) {
    if (a.no) {
        const uint4 r = philox4x32_10(a.seed_n, a.off_n, (unsigned long long)row >> 1);
        const float2 g = (row & 1) ? box_muller(r.z, r.w) : box_muller(r.x, r.y);
        const float s = sqrtf(a.no[idx_div(row, a.no_inner)]);
        acc = make_float2(acc.x + (g.x * kHalfStd) * s, acc.y + (g.y * kHalfStd) * s);
    }
    a.y[row] = acc;
}

// Uncorrelated channels, any M and K: one thread per row (problem, rx antenna) draws or reads its K coefficients,
// writes them if asked and forms y. No shared memory.
__global__ void __launch_bounds__(256) flat_fading_rows_kernel(FfArgs a) {
    const long long rows = a.num * a.M;
    for (long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x; row < rows;
         row += (long long)gridDim.x * blockDim.x) {
        const long long p = idx_div(row, a.M);
        const long long e0 = row * a.K;                          // flat index of h[p, m, 0]
        const float2* hp = a.h_in ? a.h_in + (p * a.h_stride * a.M + (row - p * a.M)) * a.K : nullptr;
        const float2* xp = a.x ? a.x + p * a.x_stride * a.K : nullptr;
        unsigned long long blk = ~0ull;
        uint4 r = make_uint4(0u, 0u, 0u, 0u);
        float2 acc = make_float2(0.f, 0.f);
        for (int k = 0; k < a.K; ++k) {
            float2 hk;
            if (hp) {
                hk = hp[k];
            } else {
                const unsigned long long i = (unsigned long long)(e0 + k);
                if ((i >> 1) != blk) { blk = i >> 1; r = philox4x32_10(a.seed_h, a.off_h, blk); }
                hk = cn_from_block(r, i);
            }
            if (a.h_out) a.h_out[e0 + k] = hk;
            if (xp) acc = mac(acc, hk, xp[k]);
        }
        if (xp) store_y(a, row, acc);
    }
}

// Correlated channels: a CTA stages `tile` whole problems of h in shared memory ([tile, M, K]) and runs
//   1. h = h0 (drawn: one thread per Philox block; given: a coalesced copy),
//   2. tx factor:  h[m, k] = sum_{j <= k} h[m, j] conj(L_tx[k, j])           (h L_tx^H)
//   3. rx factor:  h[m, k] = sum_{i <= m} L[m, i] h[i, k], L = L_rx or, per column, L_rx[k]   (L_rx h)
//   4. h written once if asked, 5. y = h x (+ noise), one thread per row.
// The reference's order (tx first, then rx). Steps 2 and 3 give each thread up to kPerThread elements: it computes
// them all (the first kInRegs into registers, the others into a staging area after the tile), then the CTA
// synchronises and writes them back, so the update is in place with at most half a second buffer (128 x 128: 128 KB
// tile + 64 KB staging). The factors are read through the read-only cache (shared across problems they stay in L1).
__global__ void __launch_bounds__(1024) flat_fading_tile_kernel(FfArgs a, int tile) {
    extern __shared__ float2 s_h[];
    const int M = a.M, K = a.K, MK = M * K;
    float2* s_stage = s_h + (size_t)tile * MK;                   // [kPerThread - kInRegs][blockDim.x], if needed
    for (long long p0 = (long long)blockIdx.x * tile; p0 < a.num; p0 += (long long)gridDim.x * tile) {
        const int np = (int)min((long long)tile, a.num - p0);
        const int n_el = np * MK;
        const long long e0 = p0 * MK;                            // flat index of the tile's first element
        __syncthreads();                                         // previous tile's readers are done
        if (a.h_in) {
            for (int e = threadIdx.x; e < n_el; e += blockDim.x) {
                const int p = e / MK;
                s_h[e] = a.h_in[((p0 + p) * a.h_stride) * MK + (e - p * MK)];
            }
        } else {
            const unsigned long long b0 = (unsigned long long)e0 >> 1, b1 = (unsigned long long)(e0 + n_el + 1) >> 1;
            for (unsigned long long b = b0 + threadIdx.x; b < b1; b += blockDim.x) {
                const uint4 r = philox4x32_10(a.seed_h, a.off_h, b);
                for (int h = 0; h < 2; ++h) {
                    const long long i = (long long)(2 * b + h);
                    if (i >= e0 && i < e0 + n_el) s_h[i - e0] = cn_from_block(r, (unsigned long long)i);
                }
            }
        }
        __syncthreads();
        for (int step = 0; step < 2; ++step) {
            const bool tx = step == 0;
            if (tx ? !a.l_tx : !a.l_rx) continue;
            float2 res[kInRegs];
#pragma unroll
            for (int u = 0; u < kPerThread; ++u) {
                const int e = threadIdx.x + u * blockDim.x;
                if (e >= n_el) break;
                const int p = e / MK, mk = e - p * MK, m = mk / K, k = mk - m * K;
                const float2* hp = s_h + p * MK;
                float2 acc = make_float2(0.f, 0.f);
                if (tx) {
                    const float2* l = a.l_tx + ((p0 + p) * a.tx_stride * K + k) * K;
#pragma unroll 1
                    for (int j = 0; j <= k; ++j) acc = cadd(acc, cmulc(hp[m * K + j], __ldg(l + j)));
                } else {
                    const float2* l = a.l_rx + (((p0 + p) * a.rx_stride * (a.per_column ? K : 1) + (a.per_column ? k : 0)) * M + m) * M;
#pragma unroll 1
                    for (int i = 0; i <= m; ++i) acc = cadd(acc, cmul(__ldg(l + i), hp[i * K + k]));
                }
                if (u < kInRegs) res[u] = acc;
                else s_stage[(u - kInRegs) * blockDim.x + threadIdx.x] = acc;
            }
            __syncthreads();
#pragma unroll
            for (int u = 0; u < kPerThread; ++u) {
                const int e = threadIdx.x + u * blockDim.x;
                if (e >= n_el) break;
                s_h[e] = u < kInRegs ? res[u] : s_stage[(u - kInRegs) * blockDim.x + threadIdx.x];
            }
            __syncthreads();
        }
        if (a.h_out)
            for (int e = threadIdx.x; e < n_el; e += blockDim.x) a.h_out[e0 + e] = s_h[e];
        if (a.x)
            for (int rr = threadIdx.x; rr < np * M; rr += blockDim.x) {
                const float2* hp = s_h + rr * K;
                const float2* xp = a.x + (p0 + rr / M) * a.x_stride * K;
                float2 acc = make_float2(0.f, 0.f);
                for (int k = 0; k < K; ++k) acc = mac(acc, hp[k], xp[k]);
                store_y(a, p0 * M + rr, acc);
            }
    }
}

// L = chol(R) per n x n matrix, one thread per matrix in interleaved shared-memory scratch (sb_dense::chol_lower);
// the strictly upper triangle of L is written as 0. A non-positive pivot makes that matrix's factor NaN from there on.
__global__ void chol_lower_kernel(const float2* __restrict__ r, float2* __restrict__ l, long long count, int n) {
    extern __shared__ float2 s_chol[];
    const sb_dense::Scratch A{s_chol, (int)blockDim.x, (int)threadIdx.x};
    const int nn = n * n;
    for (long long base = (long long)blockIdx.x * blockDim.x; base < count; base += (long long)gridDim.x * blockDim.x) {
        const long long q = base + threadIdx.x;
        if (q >= count) continue;
        const float2* rq = r + q * nn;
        for (int e = 0; e < nn; ++e) A(e) = rq[e];
        sb_dense::chol_lower(A, n);
        float2* lq = l + q * nn;
        for (int i = 0; i < n; ++i)
            for (int j = 0; j < n; ++j) lq[i * n + j] = j <= i ? A(i * n + j) : make_float2(0.f, 0.f);
    }
}

}  // namespace

extern "C" int sb_flat_fading(const float* d_h_in, int64_t h_in_stride, uint64_t seed_h, uint64_t offset_h,
                              const float* d_l_tx, int64_t l_tx_stride, const float* d_l_rx, int64_t l_rx_stride,
                              int32_t per_column, float* d_h_out, const float* d_x, int64_t x_stride, const float* d_no,
                              int64_t no_inner, uint64_t seed_n, uint64_t offset_n, float* d_y, int64_t num,
                              int32_t num_rx_ant, int32_t num_tx_ant, void* stream) {
    const int M = num_rx_ant, K = num_tx_ant;
    SB_CHECK_ARG(num >= 0 && M >= 1 && K >= 1, "sb_flat_fading: bad sizes (num >= 0, num_rx_ant >= 1, num_tx_ant >= 1)");
    SB_CHECK_ARG((h_in_stride == 0 || h_in_stride == 1) && (l_tx_stride == 0 || l_tx_stride == 1) &&
                     (l_rx_stride == 0 || l_rx_stride == 1) && (x_stride == 0 || x_stride == 1),
                 "sb_flat_fading: strides must be 0 or 1");
    SB_CHECK_ARG(per_column == 0 || (per_column == 1 && d_l_rx && !d_l_tx),
                 "sb_flat_fading: per_column is 0, or 1 with an rx factor set and no tx factor");
    SB_CHECK_ARG(d_h_out || d_x, "sb_flat_fading: nothing to compute (no h output and no x)");
    SB_CHECK_ARG(!d_x || d_y, "sb_flat_fading: x needs y");
    SB_CHECK_ARG(!d_no || (d_x && no_inner >= 1), "sb_flat_fading: noise needs x and no_inner >= 1");
    const bool corr = d_l_tx || d_l_rx;
    if (d_l_rx && M > kMaxCorrDim) {
        sb_set_error("sb_flat_fading: num_rx_ant = %d with an rx factor, the limit is %d", M, kMaxCorrDim);
        return SB_EUNSUPPORTED;
    }
    if (d_l_tx && K > kMaxCorrDim) {
        sb_set_error("sb_flat_fading: num_tx_ant = %d with a tx factor, the limit is %d", K, kMaxCorrDim);
        return SB_EUNSUPPORTED;
    }
    if (corr && (long long)M * K > kMaxTileElems) {
        sb_set_error("sb_flat_fading: %d x %d channel with correlation, the limit is M K <= %d", M, K, kMaxTileElems);
        return SB_EUNSUPPORTED;
    }
    if (num == 0) return SB_OK;                            // empty batch: nothing to do, pointers may be null
    FfArgs a{(const float2*)d_h_in, h_in_stride, seed_h, offset_h, (const float2*)d_l_tx, l_tx_stride,
             (const float2*)d_l_rx, l_rx_stride, per_column, (float2*)d_h_out, (const float2*)d_x, x_stride, d_no,
             no_inner, seed_n, offset_n, (float2*)d_y, num, M, K};
    const cudaStream_t st = (cudaStream_t)stream;
    if (!corr) {
        flat_fading_rows_kernel<<<sb_grid(num * M, 256, 8), 256, 0, st>>>(a);
    } else {
        const int MK = M * K;
        const int tile = std::max(1, kTileElems / MK);
        const int elems = tile * MK;
        const int threads = std::min(1024, std::max(128, ((elems + kPerThread - 1) / kPerThread + 31) / 32 * 32));
        const int staged = std::max(0, (elems + threads - 1) / threads - kInRegs);
        const size_t smem = sizeof(float2) * ((size_t)elems + (size_t)staged * threads);
        if (smem > 48 * 1024)
            SB_CUDA(cudaFuncSetAttribute(flat_fading_tile_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        flat_fading_tile_kernel<<<sb_grid((num + tile - 1) / tile, 1, 8), threads, smem, st>>>(a, tile);
    }
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_chol_lower(const float* d_r, float* d_l, int64_t count, int32_t n, void* stream) {
    SB_CHECK_ARG(count >= 0 && n >= 1, "sb_chol_lower: bad sizes (count >= 0, n >= 1)");
    if (n > kMaxCorrDim) {
        sb_set_error("sb_chol_lower: n = %d, the limit is %d", n, kMaxCorrDim);
        return SB_EUNSUPPORTED;
    }
    if (count == 0) return SB_OK;
    SB_CHECK_ARG(d_r && d_l, "sb_chol_lower: missing input or output");
    size_t smem = 0;
    const int threads = sb_dense::scratch_threads(sizeof(float2) * (size_t)n * n, sb_dense::kScratchSmemCap, &smem);
    if (smem > 48 * 1024)
        SB_CUDA(cudaFuncSetAttribute(chol_lower_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    chol_lower_kernel<<<sb_grid(count, threads, 8), threads, smem, (cudaStream_t)stream>>>((const float2*)d_r,
                                                                                          (float2*)d_l, count, n);
    SB_LAUNCH_CHECK();
    return SB_OK;
}
