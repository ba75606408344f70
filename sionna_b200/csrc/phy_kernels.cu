// phy_kernels.cu -- bytes-bound element-wise kernels of the link-level chain (sm_90a):
//   sb_binary_source   BinarySource.call                 mapping.py:1350-1352
//   sb_qam_map         Mapper.call                       mapping.py:497-519
//   sb_demap           Demapper.call + SymbolLogits2LLRs mapping.py:664-691, 927-967
//   sb_symbol_demap    SymbolDemapper.call               mapping.py:776-792
//   sb_awgn            AWGN.call + complex_normal        channel/awgn.py:63-78, utils/misc.py:19-54
//   sb_count_errors    count_errors / count_block_errors utils/metrics.py:94-144
// (paths relative to /root/reference/src/sionna/phy). All are one pass over HBM with coalesced accesses and
// grids sized as a multiple of the SM count; transcendental functions of the demapper come from sb_math.h so the
// CPU oracle reproduces LLRs bit for bit.
#include "sb_common.h"
#include "sb_math.h"
#include "sb_math2.cuh"
#include "rng.cuh"
#include "demap_qam.cuh"
#include "demap_prior.cuh"

namespace {

// ---------------------------------------------------------------------------------------------------------
__global__ void binary_source_kernel(float* __restrict__ out, long long n, unsigned long long seed,
                                     unsigned long long offset) {
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;   // one Philox block -> 128 bits
    long long stride = (long long)gridDim.x * blockDim.x;
    for (long long blk = i; blk * 128 < n; blk += stride) {
        uint4 r = philox4x32_10(seed, offset, (unsigned long long)blk);
        unsigned w[4] = {r.x, r.y, r.z, r.w};
        long long base = blk * 128;
#pragma unroll
        for (int k = 0; k < 4; ++k)
#pragma unroll 8
            for (int b = 0; b < 32; ++b) {
                long long idx = base + k * 32 + b;
                if (idx < n) out[idx] = (float)((w[k] >> b) & 1u);
            }
    }
}

// ---------------------------------------------------------------------------------------------------------
// bits [n_sym, m] (float 0/1) -> points[index], index = sum bit_k << (m-1-k)   (mapping.py:500-514)
__global__ void qam_map_kernel(const float* __restrict__ bits, const float2* __restrict__ points, int m,
                               float2* __restrict__ out, int* __restrict__ idx_out, long long n_sym) {
    extern __shared__ float2 s_pts[];
    for (int i = threadIdx.x; i < (1 << m); i += blockDim.x) s_pts[i] = points[i];
    __syncthreads();
    long long stride = (long long)gridDim.x * blockDim.x;
    for (long long s = (long long)blockIdx.x * blockDim.x + threadIdx.x; s < n_sym; s += stride) {
        int v = 0;
        for (int k = 0; k < m; ++k) v = (v << 1) | ((int)bits[s * m + k] & 1);
        out[s] = s_pts[v];
        if (idx_out) idx_out[s] = v;
    }
}

// ---------------------------------------------------------------------------------------------------------
// Stores the M LLRs of the symbols base + threadIdx.x (those < n_sym) through the warp's own tile of 32 * M floats of
// shared memory (s_out: 32 * M floats per warp of the CTA), so that a warp's global stores are contiguous; no CTA barrier.
template <int M>
__device__ __forceinline__ void store_llrs_warp(float* s_out, const float* out, long long base, long long n_sym,
                                                float* __restrict__ llr) {
    const int lane = threadIdx.x & 31, wbase = (threadIdx.x >> 5) * 32 * M;
    __syncwarp();                                                   // previous tile's copy-out has finished
    if (base + threadIdx.x < n_sym) {
#pragma unroll
        for (int i = 0; i < M; ++i) s_out[wbase + lane * M + i] = out[i];
    }
    __syncwarp();
    const long long wfirst = base + (threadIdx.x & ~31);
    const long long rem = n_sym - wfirst;
    const int cnt = rem <= 0 ? 0 : (int)((rem < 32 ? rem : 32) * M);
    for (int q = lane; q < cnt; q += 32) llr[wfirst * M + q] = s_out[wbase + q];
}

// One thread per symbol, M = bits per symbol at compile time: demap_symbol (demap_prior.cuh) with the noise variance
// max(no, tiny), the LLRs leave through store_llrs_warp.
template <int METHOD, int M>   // METHOD 0 = app, 1 = maxlog
__global__ void __launch_bounds__(128) demap_kernel(const float2* __restrict__ y, const float* __restrict__ no,
                                                    long long no_inner, const float2* __restrict__ points,
                                                    const float* __restrict__ prior, long long prior_inner,
                                                    float* __restrict__ llr, long long n_sym, int hard_out) {
    extern __shared__ float2 s_pts[];
    constexpr int NPTS = 1 << M;
    float* s_out = reinterpret_cast<float*>(s_pts + NPTS);          // [blockDim.x * M] store_llrs_warp tiles
    for (int i = threadIdx.x; i < NPTS; i += blockDim.x) s_pts[i] = points[i];
    __syncthreads();
    const float tiny = 1.17549435e-38f;   // np.finfo(float32).tiny (mapping.py:653)
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long base = (long long)blockIdx.x * blockDim.x; base < n_sym; base += stride) {
        const long long s = base + threadIdx.x;
        float out[M];
        if (s < n_sym) {
            const float2 yy = y[s];
            const float n0 = fmaxf(no[s / no_inner], tiny);
            float ls1[M], ls0[M];
            const bool with_prior = prior != nullptr;
            if (with_prior) {
#pragma unroll
                for (int k = 0; k < M; ++k) {
                    float pk = prior[(s / prior_inner) * M + k];
                    ls1[k] = log_sigmoidf(pk);                       // label bit 1 -> +prior
                    ls0[k] = log_sigmoidf(__fmul_rn(-1.f, pk));
                }
            }
            demap_symbol<METHOD, M>(yy, n0, s_pts, ls1, ls0, with_prior, out);
#pragma unroll
            for (int i = 0; i < M; ++i) out[i] = hard_out ? (out[i] > 0.f ? 1.f : 0.f) : out[i];   // utils/misc.py:270
        }
        store_llrs_warp<M>(s_out, out, base, n_sym, llr);
    }
}

// Separable constellations (every square QAM of mapping.py:104-117: even label bits select the real PAM level, odd
// label bits the imaginary one): the 2-D sums factor, exp(e_j) = exp(e_re) exp(e_im), and the factor of the other
// dimension cancels in the LLR, so bit i only needs the 2^(M/2) exponents of its own dimension:
//   LLR_(2u+d) = logsumexp_{t: bit u of t = 1} e_d(t) - logsumexp_{t: bit u = 0} e_d(t),  e_d(t) = -(y_d - a_d(t))^2 * (1/no)
// (max instead of logsumexp for maxlog). 2 * 2^(M/2) exponents instead of 2^M and M * 2^(M/2) instead of M * 2^M
// exp() per symbol. Same value as the generic kernel up to fp32 rounding (tests: rtol 1e-4 against the oracle).
template <int METHOD, int H>   // H = M / 2 bits per dimension
__global__ void __launch_bounds__(128) demap_qam_kernel(const float2* __restrict__ y, const float* __restrict__ no,
                                                        long long no_inner, const float* __restrict__ lev_re,
                                                        const float* __restrict__ lev_im, float* __restrict__ llr,
                                                        long long n_sym, int hard_out) {
    constexpr int L = 1 << H, M = 2 * H;
    extern __shared__ float s_out_q[];                              // [blockDim.x * M] store_llrs_warp tiles
    float lr[L], li[L];
#pragma unroll
    for (int t = 0; t < L; ++t) { lr[t] = lev_re[t]; li[t] = lev_im[t]; }
    const float tiny = 1.17549435e-38f;
    const long long stride = (long long)gridDim.x * blockDim.x;
    for (long long base = (long long)blockIdx.x * blockDim.x; base < n_sym; base += stride) {
        const long long s = base + threadIdx.x;
        float out[M];
        if (s < n_sym) {
            const float2 yy = y[s];
            const float inv_n0 = __fdiv_rn(1.0f, fmaxf(no[s / no_inner], tiny));   // one division per symbol
            demap_qam_symbol<METHOD, H>(yy, inv_n0, lr, li, lev_re, lev_im, hard_out, out);
        }
        store_llrs_warp<M>(s_out_q, out, base, n_sym, llr);
    }
}

// ---------------------------------------------------------------------------------------------------------
// SymbolDemapper: e_c = -|y - c|^2 / no + prior_c over the P points, out = log_softmax(e) [n_sym, P] (float) or the
// first argmax [n_sym] (int32). G lanes (a power of two >= min(P, 32), at most a warp) serve one symbol, lane l the
// points l, l + G, ...; a warp's 32 / G symbols are consecutive, so each store instruction of the warp writes 32
// consecutive logits (4 P bytes out per 8 bytes in: the kernel is bound by its stores). The exponents are recomputed
// in each of the three passes (max, sum of exp, store) from the points in shared memory. exp and log are sb_math.h's.
// a / b for a >= 0, b >= 1 with a 32-bit division when both fit (a 64-bit one costs several times more instructions)
__device__ __forceinline__ long long idx_div(long long a, long long b) {
    return ((a | b) >> 32) == 0 ? (long long)((unsigned)a / (unsigned)b) : a / b;
}

template <int G>
__global__ void __launch_bounds__(256) symbol_demap_kernel(const float2* __restrict__ y, const float* __restrict__ no,
                                                           long long no_inner, const float2* __restrict__ points,
                                                           int P, const float* __restrict__ prior,
                                                           long long prior_inner, void* __restrict__ out,
                                                           long long n_sym, int hard_out) {
    extern __shared__ float2 s_pts[];
    for (int i = threadIdx.x; i < P; i += blockDim.x) s_pts[i] = points[i];
    __syncthreads();
    constexpr int SPW = 32 / G;                                     // symbols per warp
    const int lane = threadIdx.x & 31, g = lane % G;
    const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const long long nwarps = ((long long)gridDim.x * blockDim.x) >> 5;
    for (long long w = warp; w * SPW < n_sym; w += nwarps) {       // warp-uniform trip count: shuffles see every lane
        const long long s = w * SPW + lane / G;
        const bool valid = s < n_sym;
        const long long sv = valid ? s : n_sym - 1;
        const float2 yy = y[sv];
        const float inv_n0 = __frcp_rn(no[idx_div(sv, no_inner)]);   // one reciprocal per symbol, as demap_qam_kernel
        const float* pr = prior ? prior + idx_div(sv, prior_inner) * P : nullptr;
        auto expo = [&](int c) {
            const float2 pt = s_pts[c];
            const float dr = yy.x - pt.x, di = yy.y - pt.y;
            float e = -((dr * dr + di * di) * inv_n0);
            if (pr) e += pr[c];
            return e;
        };
        float mx = -INFINITY;
        int arg = P;                                                // P: this lane has no point
        for (int c = g; c < P; c += G) {
            const float e = expo(c);
            if (e > mx || c == g) { mx = e; arg = c; }               // first maximum
        }
#pragma unroll
        for (int o = G / 2; o > 0; o >>= 1) {                       // maximum over the group, ties to the lowest index
            const float om = __shfl_xor_sync(0xffffffffu, mx, o);
            const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
            if (om > mx || (om == mx && oa < arg)) { mx = om; arg = oa; }
        }
        if (hard_out) {
            if (valid && g == 0) reinterpret_cast<int*>(out)[s] = arg;
            continue;
        }
        float sum = 0.f;
        for (int c = g; c < P; c += G) sum += sb_expf(expo(c) - mx);          // sum >= 1: the maximum's term
#pragma unroll
        for (int o = G / 2; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        const float lse = sb_logf(sum);
        float* o_row = reinterpret_cast<float*>(out) + s * P;
        if (valid)
            for (int c = g; c < P; c += G) o_row[c] = (expo(c) - mx) - lse;   // tf.nn.log_softmax: shifted - log sum
    }
}

// ---------------------------------------------------------------------------------------------------------
// y = x + sqrt(no) * n,  n ~ CN(0, 1): re, im ~ N(0, 1/2) (utils/misc.py:46-52, channel/awgn.py:66-78).
// One Philox block (4 uniforms -> 2 Box-Muller pairs) serves two complex samples.
__global__ void awgn_kernel(const float2* x, const float* __restrict__ no, long long no_inner,
                            float2* y, long long n, unsigned long long seed, unsigned long long offset) {
    long long stride = (long long)gridDim.x * blockDim.x;
    const float stddev = 0.70710678118654752f;   // sqrt(var/2), var = 1
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; 2 * p < n; p += stride) {
        uint4 r = philox4x32_10(seed, offset, (unsigned long long)p);
        float2 g0 = box_muller(r.x, r.y), g1 = box_muller(r.z, r.w);
        long long i0 = 2 * p, i1 = 2 * p + 1;
        float s0 = sqrtf(no[i0 / no_inner]);
        float2 a = x[i0];
        y[i0] = make_float2(a.x + (g0.x * stddev) * s0, a.y + (g0.y * stddev) * s0);
        if (i1 < n) {
            float s1 = sqrtf(no[i1 / no_inner]);
            float2 b = x[i1];
            y[i1] = make_float2(b.x + (g1.x * stddev) * s1, b.y + (g1.y * stddev) * s1);
        }
    }
}

// Real-valued Philox draws, four outputs per Philox block. NORMAL: out = a + b * N(0,1) by two Box-Muller pairs
// (GaussianPriorSource); otherwise out = a + (b - a) * u, u in [0, 1) with 24 random bits (TDL Doppler / angle / phase).
template <bool NORMAL>
__global__ void philox_fill_kernel(float* __restrict__ out, long long n, float a, float b, unsigned long long seed,
                                   unsigned long long offset) {
    long long stride = (long long)gridDim.x * blockDim.x;
    const float w = b - a;
    for (long long p = (long long)blockIdx.x * blockDim.x + threadIdx.x; 4 * p < n; p += stride) {
        uint4 r = philox4x32_10(seed, offset, (unsigned long long)p);
        float v[4];
        if (NORMAL) {
            float2 g0 = box_muller(r.x, r.y), g1 = box_muller(r.z, r.w);
            v[0] = g0.x; v[1] = g0.y; v[2] = g1.x; v[3] = g1.y;
        } else {
            unsigned u[4] = {r.x, r.y, r.z, r.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) v[k] = (float)(u[k] >> 8) * 5.9604644775390625e-08f;   // 2^-24
        }
#pragma unroll
        for (int k = 0; k < 4; ++k)
            if (4 * p + k < n) out[4 * p + k] = a + (NORMAL ? b : w) * v[k];
    }
}

// ---------------------------------------------------------------------------------------------------------
// counters[0] += #(b != b_hat), counters[1] += #rows with any difference, counters[2] += B*k, counters[3] += B.
// One warp per row; block-level reduction, one atomic per block and counter.
__global__ void count_errors_kernel(const float* __restrict__ b, const float* __restrict__ bh, long long rows, int k,
                                    unsigned long long* __restrict__ counters) {
    __shared__ unsigned long long s_bit[32], s_blk[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    unsigned long long bit_e = 0, blk_e = 0;
    for (long long r = (long long)blockIdx.x * nwarps + warp; r < rows; r += (long long)gridDim.x * nwarps) {
        const float* pb = b + r * k;
        const float* ph = bh + r * k;
        unsigned cnt = 0;
        for (int i = lane; i < k; i += 32) cnt += (pb[i] != ph[i]);
        cnt = __reduce_add_sync(0xffffffffu, cnt);
        bit_e += cnt;
        blk_e += (cnt != 0);
    }
    if (lane == 0) { s_bit[warp] = bit_e; s_blk[warp] = blk_e; }
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long tb = 0, tk = 0;
        for (int w = 0; w < nwarps; ++w) { tb += s_bit[w]; tk += s_blk[w]; }
        if (tb) atomicAdd(&counters[0], tb);
        if (tk) atomicAdd(&counters[1], tk);
        if (blockIdx.x == 0) {
            atomicAdd(&counters[2], (unsigned long long)rows * (unsigned long long)k);
            atomicAdd(&counters[3], (unsigned long long)rows);
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// CRCEncoder.call (fec/crc.py:175-215) and, CHECK, CRCDecoder.call (fec/crc.py:300-327). The reference multiplies the
// bit row with a dense [n, L] generator matrix and reduces mod 2; the CRC is linear, so the parity word is the XOR of
// the (bit-packed) matrix rows selected by the set bits. One warp per row of n bits: lanes stride over the bits,
// XOR-reduce, then
//   encode: out row = [bits | parity] (n + L values, MSB = first parity bit);
//   check:  the row is a whole word [info | parity], valid = (parity of the word == 0); out (optional) gets the
//           n - L information bits.
template <bool CHECK>
__global__ void crc_kernel(const float* __restrict__ x, const unsigned* __restrict__ gtab, int n, int L,
                           float* __restrict__ out, unsigned char* __restrict__ valid, long long rows) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const int k = CHECK ? n - L : n;                                // bits copied to out
    const long long out_len = CHECK ? k : n + L;
    for (long long r = (long long)blockIdx.x * nwarps + warp; r < rows; r += (long long)gridDim.x * nwarps) {
        const float* b = x + r * (long long)n;
        unsigned acc = 0;
        for (int i = lane; i < n; i += 32) {
            float v = b[i];
            if (!CHECK || (out && i < k)) out[r * out_len + i] = v;
            if (((int)v) & 1) acc ^= gtab[i];
        }
        acc = __reduce_xor_sync(0xffffffffu, acc);
        if (CHECK) {
            if (lane == 0) valid[r] = acc == 0u ? 1 : 0;
        } else if (lane < L) {
            out[r * out_len + k + lane] = (float)((acc >> (L - 1 - lane)) & 1u);
        }
    }
}

// TB5GScrambler.call (fec/scrambling.py:442-468): binary: |x - c|; soft values: x * (1 - 2c). seq has seq_rows rows
// (one per stream) of length n; row r of x uses seq row (r mod seq_rows).
__global__ void scramble_kernel(const float* __restrict__ x, const float* __restrict__ seq, int binary,
                                float* __restrict__ out, long long rows, int n, int seq_rows) {
    const long long total = rows * n;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int j = (int)(i % n);
        long long r = i / n;
        float c = seq[(r % seq_rows) * n + j];
        float v = x[i];
        out[i] = binary ? fabsf(v - c) : v * (-2.f * c + 1.f);
    }
}

}  // namespace

extern "C" int sb_binary_source(float* d_out, int64_t n, uint64_t seed, uint64_t offset, void* stream) {
    if (n == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_out && n >= 0, "sb_binary_source: bad arguments");
    binary_source_kernel<<<sb_grid((n + 127) / 128, 128, 8), 128, 0, (cudaStream_t)stream>>>(d_out, n, seed, offset);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_qam_map(const float* d_bits, const float* d_points, int32_t m, float* d_out, int32_t* d_idx_out,
                          int64_t n_sym, void* stream) {
    if (n_sym == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_bits && d_points && d_out && m >= 1 && m <= 12 && n_sym >= 0, "sb_qam_map: bad arguments");
    size_t smem = sizeof(float2) << m;
    qam_map_kernel<<<sb_grid(n_sym, 256, 8), 256, smem, (cudaStream_t)stream>>>(
        d_bits, (const float2*)d_points, m, (float2*)d_out, d_idx_out, n_sym);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_demap(const float* d_y, const float* d_no, int64_t no_inner, const float* d_points, int32_t m,
                        int32_t method, const float* d_prior, int64_t prior_inner, float* d_llr, int64_t n_sym,
                        int32_t hard_out, void* stream) {
    if (n_sym == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_y && d_no && d_points && d_llr && m >= 1 && m <= 12 && n_sym >= 0 && no_inner >= 1,
                 "sb_demap: bad arguments");
    SB_CHECK_ARG(method == 0 || method == 1, "sb_demap: method must be 0 (app) or 1 (maxlog)");
    SB_CHECK_ARG(!d_prior || prior_inner >= 1, "sb_demap: prior_inner must be >= 1");
    const size_t smem = (sizeof(float2) << m) + sizeof(float) * 128 * m;
    const int grid = sb_grid(n_sym, 128, 8);
    sb_dispatch<0, 1>(method, [&](auto METHOD) {
        return sb_dispatch<1, 12>(m, [&](auto M) {
            demap_kernel<METHOD, M><<<grid, 128, smem, (cudaStream_t)stream>>>(
                (const float2*)d_y, d_no, no_inner, (const float2*)d_points, d_prior, prior_inner, d_llr, n_sym, hard_out);
            return SB_OK;
        });
    });
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_symbol_demap(const float* d_y, const float* d_no, int64_t no_inner, const float* d_points,
                               int32_t num_points, const float* d_prior, int64_t prior_inner, void* d_out, int64_t n_sym,
                               int32_t hard_out, void* stream) {
    SB_CHECK_ARG(num_points >= 2 && num_points <= 1024, "sb_symbol_demap: num_points = %d, supported are 2 ... 1024",
                 num_points);
    SB_CHECK_ARG(n_sym >= 0 && no_inner >= 1 && (!d_prior || prior_inner >= 1) && (hard_out == 0 || hard_out == 1),
                 "sb_symbol_demap: bad arguments");
    if (n_sym == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_y && d_no && d_points && d_out, "sb_symbol_demap: missing input or output");
    int lanes = 1;
    while (lanes < num_points && lanes < 32) lanes *= 2;
    const long long warps = (n_sym + 32 / lanes - 1) / (32 / lanes);
    const int grid = sb_grid(warps, 8, 8);
    const size_t smem = sizeof(float2) * num_points;
    const int rc = sb_dispatch<1, 5>(__builtin_ctz(lanes), [&](auto L) {
        symbol_demap_kernel<(1 << L)><<<grid, 256, smem, (cudaStream_t)stream>>>(
            (const float2*)d_y, d_no, no_inner, (const float2*)d_points, num_points, d_prior, prior_inner, d_out, n_sym,
            hard_out);
        return SB_OK;
    });
    if (rc) return rc;
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_demap_qam(const float* d_y, const float* d_no, int64_t no_inner, const float* d_levels_re,
                            const float* d_levels_im, int32_t m, int32_t method, float* d_llr, int64_t n_sym,
                            int32_t hard_out, void* stream) {
    if (n_sym == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_y && d_no && d_levels_re && d_levels_im && d_llr && m >= 2 && m <= 10 && m % 2 == 0 && no_inner >= 1 &&
                     (method == 0 || method == 1), "sb_demap_qam: bad arguments (m even, 2..10; method 0 | 1)");
    const size_t smem = sizeof(float) * 128 * m;
    const int grid = sb_grid(n_sym, 128, 8);
    sb_dispatch<0, 1>(method, [&](auto METHOD) {
        return sb_dispatch<1, 5>(m / 2, [&](auto H) {
            demap_qam_kernel<METHOD, H><<<grid, 128, smem, (cudaStream_t)stream>>>((const float2*)d_y, d_no, no_inner, d_levels_re,
                                                                                   d_levels_im, d_llr, n_sym, hard_out);
            return SB_OK;
        });
    });
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_awgn(const float* d_x, const float* d_no, int64_t no_inner, float* d_y, int64_t n, uint64_t seed,
                       uint64_t offset, void* stream) {
    if (n == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_x && d_no && d_y && n >= 0 && no_inner >= 1, "sb_awgn: bad arguments");
    awgn_kernel<<<sb_grid((n + 1) / 2, 256, 8), 256, 0, (cudaStream_t)stream>>>((const float2*)d_x, d_no, no_inner,
                                                                              (float2*)d_y, n, seed, offset);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_normal(float* d_out, int64_t n, float mean, float stddev, uint64_t seed, uint64_t offset, void* stream) {
    if (n == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_out && n >= 0, "sb_normal: bad arguments");
    philox_fill_kernel<true><<<sb_grid((n + 3) / 4, 256, 8), 256, 0, (cudaStream_t)stream>>>(d_out, n, mean, stddev, seed, offset);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_uniform(float* d_out, int64_t n, float lo, float hi, uint64_t seed, uint64_t offset, void* stream) {
    if (n == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_out && n >= 0 && hi >= lo, "sb_uniform: bad arguments");
    philox_fill_kernel<false><<<sb_grid((n + 3) / 4, 256, 8), 256, 0, (cudaStream_t)stream>>>(d_out, n, lo, hi, seed, offset);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_count_errors(const float* d_b, const float* d_b_hat, int64_t rows, int32_t k, int64_t* d_counters,
                               void* stream) {
    if (rows == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_b && d_b_hat && d_counters && rows >= 0 && k >= 1, "sb_count_errors: bad arguments");
    count_errors_kernel<<<sb_grid(rows * 32, 256, 8), 256, 0, (cudaStream_t)stream>>>(
        d_b, d_b_hat, rows, k, (unsigned long long*)d_counters);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_crc_encode(const float* d_bits, const uint32_t* d_gen_rows, int32_t k, int32_t crc_length, float* d_out,
                             int64_t rows, void* stream) {
    if (rows == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_bits && d_gen_rows && d_out && k >= 1 && crc_length >= 1 && crc_length <= 32 && rows >= 0,
                 "sb_crc_encode: bad arguments");
    crc_kernel<false><<<sb_grid(rows * 32, 256, 8), 256, 0, (cudaStream_t)stream>>>(d_bits, d_gen_rows, k, crc_length, d_out,
                                                                                   nullptr, rows);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_crc_check(const float* d_x, const uint32_t* d_gen_rows, int32_t n, int32_t crc_length, float* d_info,
                            uint8_t* d_valid, int64_t rows, void* stream) {
    if (rows == 0) return SB_OK;
    SB_CHECK_ARG(d_x && d_gen_rows && d_valid && crc_length >= 1 && crc_length <= 32 && n >= crc_length && rows >= 0,
                 "sb_crc_check: bad arguments");
    crc_kernel<true><<<sb_grid(rows * 32, 256, 8), 256, 0, (cudaStream_t)stream>>>(d_x, d_gen_rows, n, crc_length, d_info,
                                                                                  d_valid, rows);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_scramble(const float* d_x, const float* d_seq, int32_t binary, float* d_out, int64_t rows, int32_t n,
                           int32_t seq_rows, void* stream) {
    if (rows == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_x && d_seq && d_out && rows >= 0 && n >= 1 && seq_rows >= 1, "sb_scramble: bad arguments");
    scramble_kernel<<<sb_grid(rows * n, 256, 8), 256, 0, (cudaStream_t)stream>>>(d_x, d_seq, binary, d_out, rows, n, seq_rows);
    SB_LAUNCH_CHECK();
    return SB_OK;
}
