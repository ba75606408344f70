// ofdm_mimo.cu -- OFDM (de)modulation, resource-grid gathers, LS channel estimation + interpolation and per-RE LMMSE
// equalisation for sm_90a. Replaces (paths under /root/reference/src/sionna/phy/):
//   sb_ofdm_modulate      OFDMModulator.call   ofdm/modulator.py:97-124   + ifft  signal/utils.py:206-249
//   sb_ofdm_demodulate    OFDMDemodulator.call ofdm/demodulator.py:162-203 + fft   signal/utils.py:161-204
//   sb_gather_rows        tf.gather based re-indexing: RemoveNulledSubcarriers ofdm/resource_grid.py:551,
//                         ResourceGridDemapper :466-520, NearestNeighborInterpolator ofdm/channel_estimation.py:409-435
//   sb_rg_map             ResourceGridMapper.call  ofdm/resource_grid.py:394-412
//   sb_ls_at_pilots       BaseChannelEstimator.call pilot gather :138-150 + LSChannelEstimator :257-285
//   sb_interp_lin         LinearInterpolator._interpolate ofdm/channel_estimation.py:657-734
//   sb_pusch_precode      PUSCHPrecoder.call       nr/pusch_precoder.py:75-95
//   sb_pusch_ls_combine   PUSCHLSChannelEstimator.estimate_at_pilot_locations   nr/pusch_channel_estimation.py:117-169
//   sb_lmmse_equalize     lmmse_equalizer mimo/equalization.py:101-233 (+ whiten_channel mimo/utils.py:292-357,
//                         lmmse_matrix :11-99)
//   sb_mimo_linalg        inv_cholesky, whiten_channel, lmmse_matrix, lmmse_equalizer(whiten_interference=False),
//                         zf_equalizer, mf_equalizer, matrix_pinv (mimo/equalization.py:11-466, utils/linalg.py)
//   sb_ofdm_lmmse         OFDMEqualizer.call ofdm/equalization.py:109-275 with the LMMSE equaliser fused in: the
//                         interference-plus-noise covariance S = H_u H_u^H + diag(no) + diag(sum err_var) is
//                         assembled on chip per resource element and never written to HBM (the reference materialises a
//                         [.., M, M] tensor, 2 KB per RE for M = 16).
//   sb_ofdm_equalize      the same with the LMMSE (whitened or not), ZF or MF equaliser fused in (LMMSEEqualizer,
//                         ZFEqualizer, MFEqualizer, ofdm/equalization.py:277-462)
// All kernels are one pass over HBM; FFT twiddles come from sincospif (<= 1 ulp), parity bar 1e-5 (the reference's own
// round-trip test tolerance, test/unit/ofdm/test_ofdm.py:85-96).
#include "sb_common.h"
#include "lmmse_diag.cuh"
#include "dense_mimo.cuh"

namespace {

using sb_dense::Scratch;
using sb_dense::chol_lower;
using sb_dense::chol_solve_col;
using sb_dense::whiten;
using sb_dense::OfdmEqParams;

// ---------------------------------------------------------------------------------------------------------------
// Mixed-radix Stockham FFT in shared memory: one CTA transforms one length-N vector (ping-pong buffers, twiddle table
// W[k] = exp(-2 pi i k / N)). Radices are the prime factors of N (4 is used for pairs of 2); a radix-p butterfly is a
// direct p-point DFT, so any N works (72 = 2*2*2*3*3, 76 = 2*2*19, 2^k, 12*PRB ...).
// ---------------------------------------------------------------------------------------------------------------
struct FftPlan {
    int n, n_radix;
    int radix[24];
    int span_shift[24];      // log2 of the stage's span (product of the previous radices) if it is a power of two, else -1
};

__device__ void fft_inplace_smem(float2* buf0, float2* buf1, const float2* W, const FftPlan& plan, float2** result) {
    const int N = plan.n, tid = threadIdx.x, T = blockDim.x;
    float2* x = buf0;
    float2* y = buf1;
    int n = N, s = 1;
    for (int st = 0; st < plan.n_radix; ++st) {
        const int p = plan.radix[st], m = n / p;
        const int wstep = N / p;                       // exp(-2 pi i r c / p) = W[(r*c mod p) * N/p]
        const int sh = plan.span_shift[st];
        for (int b = tid; b < N / p; b += T) {         // butterfly (q, k): q in [0, s), k in [0, m)
            const int k = sh >= 0 ? (b >> sh) : b / s;
            const int q = b - k * s;
            // twiddle exponents c * k * s stay below N (k < m, c < p, p * m * s = N): no modulo needed
            if (p == 2) {
                float2 a0 = x[q + s * k], a1 = x[q + s * (k + m)];
                y[q + s * (2 * k)] = cadd(a0, a1);
                y[q + s * (2 * k + 1)] = cmul(csub(a0, a1), W[k * s]);
            } else if (p == 4) {
                float2 a0 = x[q + s * k], a1 = x[q + s * (k + m)], a2 = x[q + s * (k + 2 * m)], a3 = x[q + s * (k + 3 * m)];
                float2 t0 = cadd(a0, a2), t1 = csub(a0, a2), t2 = cadd(a1, a3), t3 = csub(a1, a3);
                float2 t3j = make_float2(t3.y, -t3.x);                   // -j * t3
                y[q + s * (4 * k)] = cadd(t0, t2);
                y[q + s * (4 * k + 1)] = cmul(cadd(t1, t3j), W[k * s]);
                y[q + s * (4 * k + 2)] = cmul(csub(t0, t2), W[2 * k * s]);
                y[q + s * (4 * k + 3)] = cmul(csub(t1, t3j), W[3 * k * s]);
            } else {
                for (int c = 0; c < p; ++c) {
                    float2 acc = make_float2(0.f, 0.f);
                    for (int r = 0; r < p; ++r) acc = cadd(acc, cmul(x[q + s * (k + r * m)], W[((r * c) % p) * wstep]));
                    y[q + s * (p * k + c)] = cmul(acc, W[c * k * s]);
                }
            }
        }
        __syncthreads();
        float2* t = x; x = y; y = t;
        n = m;
        s *= p;
    }
    *result = x;
}

// Generic path, one CTA per transform. off / len: offsets of the OFDM symbols in a time-domain row and the row length.
//   DEMOD = 0, OFDMModulator: x [rows, nsym, N] (frequency domain, DC in the centre) -> out [rows, sum_l (N + cp[l])]
//     ifftshift -> ifft * sqrt(N) -> cyclic prefix (modulator.py:100-124, signal/utils.py:240-249).
//   DEMOD = 1, OFDMDemodulator: x [rows, >= sum_l (N + cp[l])] -> out [rows, nsym, N]: strip CP, fft / sqrt(N), phase
//     compensation exp(-j 2 pi k l_min / N) (fp32, demodulator.py:131-134, 196-198), fftshift (:201).
// Shared memory: 3 N float2 (two data buffers and the twiddles), so N = 8192 fits the 227 KB opt-in limit. The phase
// compensation is evaluated per output bin rather than tabulated: a fourth N-entry table would cap N at 7264.
template <int DEMOD>
__global__ void ofdm_fft_kernel(const float2* __restrict__ x, float2* __restrict__ out, FftPlan plan, int nsym,
                                const int* __restrict__ cp, const int* __restrict__ off, int len, int l_min,
                                long long rows, int shift) {
    extern __shared__ float2 sm[];
    const int N = plan.n, tid = threadIdx.x, T = blockDim.x;
    float2* b0 = sm; float2* b1 = sm + N; float2* W = sm + 2 * N;
    for (int k = tid; k < N; k += T) {
        float sn, cs;
        sincospif(-2.0f * (float)k / (float)N, &sn, &cs);
        W[k] = make_float2(cs, sn);
    }
    const float scale = 1.0f / sqrtf((float)N);     // modulator: ifft = conj(fft(conj))/N, then * sqrt(N)
    for (long long job = blockIdx.x; job < rows * nsym; job += gridDim.x) {
        const int l = (int)(job % nsym);
        const float2* src = DEMOD ? x + (job / nsym) * len + off[l] + cp[l] : x + job * N;
        __syncthreads();
        if (DEMOD) {
            for (int k = tid; k < N; k += T) b0[k] = src[k];
        } else {
            for (int k = tid; k < N; k += T) {
                float2 v = src[shift ? (k + N / 2) % N : k];   // ifftshift: out[k] = in[(k + floor(N/2)) mod N]
                b0[k] = make_float2(v.x, -v.y);
            }
        }
        __syncthreads();
        float2* res;
        fft_inplace_smem(b0, b1, W, plan, &res);
        if (DEMOD) {
            float2* dst = out + job * N;
            for (int k = tid; k < N; k += T) {
                int ks = shift ? (k + N / 2) % N : k;   // fftshift: out[k'] with k' = (k + floor(N/2)) mod N takes bin k
                // tmp = -2 pi l_min / N * k in fp32 as the reference computes it, then exp(j tmp). The complex product
                // is spelled out (a.y * pc rounded, a.x * pc fused) so that its rounding does not depend on how the
                // compiler contracts cmul.
                const float tmp = -2.0f * 3.14159265358979323846f * (float)l_min / (float)N * (float)k;
                const float2 a = cscale(res[k], scale), pc = make_float2(cosf(tmp), sinf(tmp));
                dst[ks] = make_float2(fmaf(a.x, pc.x, -__fmul_rn(a.y, pc.y)), fmaf(a.x, pc.y, __fmul_rn(a.y, pc.x)));
            }
        } else {
            const int c = cp[l];
            float2* dst = out + (job / nsym) * len + off[l];
            for (int i = tid; i < N + c; i += T) {
                float2 v = res[(i - c + N) % N];
                dst[i] = make_float2(v.x * scale, -v.y * scale);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// FFT sizes up to 1024 (every OFDM grid up to 85 PRB, e.g. 72, 76, 128, 180, 600): one WARP per FPW transforms, several
// warps per CTA, no CTA-wide barrier in the loop. Stockham stages; a lane owns a whole radix-p BUTTERFLY (inputs in
// registers), the FPW * N/p butterflies of a stage are dealt over the lanes:
//   p = 2, 4      the usual add / subtract networks;
//   odd p <= 19   (3, 5, 7, 11, 13, 17, 19: the 76-point grid is 4 * 19) real-symmetric form of the p-point DFT: with
//                 a_r = x_r + x_(p-r), b_r = x_r - x_(p-r) the outputs c and p - c are E_c +- O_c,
//                 E_c = x_0 + sum_r a_r cos(2 pi r c / p), O_c = -j sum_r b_r sin(2 pi r c / p): (p-1)^2 real FMAs per
//                 butterfly instead of 4 p (p-1), the roots are warp-uniform (broadcast) shared-memory loads;
//   other p       direct p-term sums.
// The largest prime comes last in the plan, where the Stockham twiddles are all 1 (k = 0) and are skipped.
// ---------------------------------------------------------------------------------------------------------------
struct SmallFftPlan {
    int n, n_stages;
    int p[12];
    unsigned mg_nb[12], mg_span[12];   // ceil(2^32 / (n / p)), ceil(2^32 / span): exact quotients for indices < 4096
    float2 roots[75];                  // exp(-2 pi i j / P), j < P, for P = 3, 5, 7, 11, 13, 17, 19 (root_offset(P))
};

__host__ __device__ constexpr int root_offset(int P) {
    return P == 3 ? 0 : P == 5 ? 3 : P == 7 ? 8 : P == 11 ? 15 : P == 13 ? 26 : P == 17 ? 39 : 56;
}

// one butterfly of odd prime radix P: inputs xi[r * rs], outputs yo[c * os] * W[c * tws]. The P-th roots are kernel
// parameters, and every index (r * c mod P) is a compile-time constant: the FMAs take them straight from the constant
// bank (no loads, no index arithmetic).
template <int P>
__device__ __forceinline__ void fft_butterfly_odd(const float2* xi, int rs, float2* yo, int os, const SmallFftPlan& plan,
                                                  const float2* __restrict__ W, int tws) {
    constexpr int HP = (P - 1) / 2, RO = root_offset(P);
    const float2 x0 = xi[0];
    float2 a[HP], b[HP];
    float2 s0 = x0;
#pragma unroll
    for (int r = 0; r < HP; ++r) {
        const float2 u = xi[(r + 1) * rs], v = xi[(P - 1 - r) * rs];
        a[r] = cadd(u, v);
        b[r] = csub(u, v);
        s0 = cadd(s0, a[r]);
    }
    yo[0] = s0;
#pragma unroll
    for (int c = 1; c <= HP; ++c) {
        float2 E = x0, O = make_float2(0.f, 0.f);
#pragma unroll
        for (int r = 0; r < HP; ++r) {
            const float2 w = plan.roots[RO + ((r + 1) * c) % P];   // (cos t, -sin t), t = 2 pi (r + 1) c / P
            E.x = fmaf(a[r].x, w.x, E.x);
            E.y = fmaf(a[r].y, w.x, E.y);
            O.x = fmaf(-b[r].y, w.y, O.x);                          // -j b sin t
            O.y = fmaf(b[r].x, w.y, O.y);
        }
        float2 xc = cadd(E, O), xpc = csub(E, O);
        if (tws) {
            xc = cmul(xc, W[c * tws]);
            xpc = cmul(xpc, W[(P - c) * tws]);
        }
        yo[c * os] = xc;
        yo[(P - c) * os] = xpc;
    }
}

// FPW transforms per warp at a time. Buffers: x / y [FPW][N].
template <int FPW>
__device__ __forceinline__ float2* fft_small_warp(float2* x, float2* y, const float2* __restrict__ W,
                                                  const SmallFftPlan& plan, int lane) {
    const int N = plan.n;
    int span = 1, cur = N;
    for (int st = 0; st < plan.n_stages; ++st) {
        const int p = plan.p[st], m = cur / p, rs = span * m;
        const int nb = N / p;                                      // butterflies per transform: b = q + span * k
        const unsigned mg_nb = plan.mg_nb[st], mg_span = plan.mg_span[st];
        for (int i = lane; i < FPW * nb; i += 32) {
            const int f = nb == 1 ? i : (int)__umulhi((unsigned)i, mg_nb), bb = i - f * nb;
            const int k = span == 1 ? bb : (int)__umulhi((unsigned)bb, mg_span), q = bb - k * span;
            const float2* xi = x + f * N + q + span * k;
            float2* yo = y + f * N + q + span * p * k;
            const int tws = k * span;                              // root index step of the Stockham twiddle (c * tws < N)
            switch (p) {
                case 2: {
                    const float2 a0 = xi[0], a1 = xi[rs];
                    yo[0] = cadd(a0, a1);
                    yo[span] = cmul(csub(a0, a1), W[tws]);
                    break;
                }
                case 4: {
                    const float2 a0 = xi[0], a1 = xi[rs], a2 = xi[2 * rs], a3 = xi[3 * rs];
                    const float2 t0 = cadd(a0, a2), t1 = csub(a0, a2), t2 = cadd(a1, a3), t3 = csub(a1, a3);
                    const float2 t3j = make_float2(t3.y, -t3.x);   // -j * t3
                    yo[0] = cadd(t0, t2);
                    yo[span] = cmul(cadd(t1, t3j), W[tws]);
                    yo[2 * span] = cmul(csub(t0, t2), W[2 * tws]);
                    yo[3 * span] = cmul(csub(t1, t3j), W[3 * tws]);
                    break;
                }
                case 3: fft_butterfly_odd<3>(xi, rs, yo, span, plan, W, tws); break;
                case 5: fft_butterfly_odd<5>(xi, rs, yo, span, plan, W, tws); break;
                case 7: fft_butterfly_odd<7>(xi, rs, yo, span, plan, W, tws); break;
                case 11: fft_butterfly_odd<11>(xi, rs, yo, span, plan, W, tws); break;
                case 13: fft_butterfly_odd<13>(xi, rs, yo, span, plan, W, tws); break;
                case 17: fft_butterfly_odd<17>(xi, rs, yo, span, plan, W, tws); break;
                case 19: fft_butterfly_odd<19>(xi, rs, yo, span, plan, W, tws); break;
                default: {                                         // larger primes: direct p-term sums
                    const int wstep = N / p;
                    for (int c = 0; c < p; ++c) {
                        float2 acc = xi[0];
                        int widx = 0;
                        for (int r = 1; r < p; ++r) {
                            widx += c * wstep;
                            widx -= widx >= N ? N : 0;
                            acc = cadd(acc, cmul(xi[r * rs], W[widx]));
                        }
                        yo[c * span] = cmul(acc, W[c * tws]);
                    }
                }
            }
        }
        __syncwarp();
        float2* t = x; x = y; y = t;
        cur = m;
        span *= p;
    }
    return x;
}

__device__ __forceinline__ void cp_async8(float2* smem_dst, const float2* gmem_src) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"((unsigned)__cvta_generic_to_shared(smem_dst)), "l"(gmem_src));
}

// A warp works on batches of FPW consecutive (row, symbol) jobs. Three shared-memory buffers per warp rotate: while the
// FFT stages ping-pong between two of them, cp.async fills the third with the next batch's samples (no registers, the
// global-load latency hides behind the butterflies).
template <int DEMOD, int FPW>
__global__ void __launch_bounds__(256, 2) ofdm_fft_small_kernel(const float2* __restrict__ x, float2* __restrict__ out,
                                                             const __grid_constant__ SmallFftPlan plan, int nsym,
                                                             const int* __restrict__ cp,
                                                             const int* __restrict__ off, int len, int l_min,
                                                             long long rows, int shift) {
    extern __shared__ float2 sm[];
    const int N = plan.n, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
    float2* W = sm;
    float2* PC = sm + N;                                           // phase compensation (demodulator only)
    float2* bufs = sm + (DEMOD ? 2 : 1) * N;
    for (int k = tid; k < N; k += blockDim.x) {
        float sn, cs;
        sincospif(-2.0f * (float)k / (float)N, &sn, &cs);
        W[k] = make_float2(cs, sn);
        if (DEMOD) {
            float tmp = -2.0f * 3.14159265358979323846f * (float)l_min / (float)N * (float)k;
            PC[k] = make_float2(cosf(tmp), sinf(tmp));
        }
    }
    __syncthreads();
    float2* bin = bufs + (size_t)3 * FPW * N * warp;               // receives the next batch
    float2* bx = bin + (size_t)FPW * N;
    float2* by = bx + (size_t)FPW * N;
    const float scale = 1.0f / sqrtf((float)N);
    const long long jobs = rows * nsym;
    const int h = N / 2;
    const long long jstep = (long long)gridDim.x * nwarps * FPW;

    // asynchronous copy of batch jb into dst: the demodulator copies the samples behind the cyclic prefix, the modulator
    // applies the ifftshift to the source index (the conjugation of ifft = conj(fft(conj(.))) / N happens on arrival)
    auto prefetch = [&](long long jb, float2* dst) {
        if (jb < jobs) {
            long long row = jb / nsym;
            int l = (int)(jb - row * nsym);
#pragma unroll
            for (int f = 0; f < FPW; ++f) {
                if (jb + f < jobs) {                               // tail: stale buffer contents are transformed, never stored
                    if (DEMOD) {
                        const float2* src = x + row * len + off[l] + cp[l];
                        for (int k = lane; k < N; k += 32) cp_async8(dst + f * N + k, src + k);
                    } else {
                        const float2* src = x + (jb + f) * N;
                        for (int k = lane; k < N; k += 32) {
                            int ks = k;
                            if (shift) { ks = k + h; ks -= ks >= N ? N : 0; }   // ifftshift
                            cp_async8(dst + f * N + k, src + ks);
                        }
                    }
                }
                if (++l == nsym) { l = 0; ++row; }
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };

    long long jb = ((long long)blockIdx.x * nwarps + warp) * FPW;
    prefetch(jb, bin);
    for (; jb < jobs; jb += jstep) {
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncwarp();
        { float2* t = bin; bin = bx; bx = t; }                     // bx: this batch; bin: free again (stored last round)
        prefetch(jb + jstep, bin);
        if (!DEMOD) {
            for (int k = lane; k < FPW * N; k += 32) bx[k].y = -bx[k].y;
            __syncwarp();
        }
        const float2* res = fft_small_warp<FPW>(bx, by, W, plan, lane);
        long long row = jb / nsym;
        int l = (int)(jb - row * nsym);
#pragma unroll
        for (int f = 0; f < FPW; ++f) {
            if (jb + f < jobs) {
                const float2* rf = res + f * N;
                if (DEMOD) {
                    float2* dst = out + (jb + f) * N;
                    for (int k = lane; k < N; k += 32) {
                        int ks = k;
                        if (shift) { ks = k + h; ks -= ks >= N ? N : 0; }   // fftshift
                        dst[ks] = cmul(cscale(rf[k], scale), PC[k]);
                    }
                } else {
                    const int c = cp[l];
                    float2* dst = out + row * len + off[l];
                    for (int i = lane; i < N + c; i += 32) {
                        int k = i - c;
                        k += k < 0 ? N : 0;
                        const float2 v = rf[k];
                        dst[i] = make_float2(v.x * scale, -v.y * scale);
                    }
                }
            }
            if (++l == nsym) { l = 0; ++row; }
        }
        __syncwarp();
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
}

// ---------------------------------------------------------------------------------------------------------------
// N = 4096 and 2048 (the 100 / 50 MHz NR grids), N = R0 * 256 with R0 = 16 / 8: three in-place passes (decimation in
// frequency) - radix R0, radix 16, radix 16 - instead of six radix-4 Stockham passes. A thread owns one butterfly per
// pass (up to 16 points in registers, two levels of radix-4 / radix-2 with the constant roots between them), so a pass is
// one shared-memory round trip and 256 threads cover the transform. In place means ONE data buffer per transform: a
// second one receives the next transform by cp.async while this one is computed, and two CTAs fit on an SM. The result
// sits in digit-reversed order (X[j0 + R0 (j1 + 16 j2)] at position 256 j0 + 16 j1 + j2); the copy-out loop undoes that.
// The buffer is padded (i + i/16 + i/256) so that the pass patterns and the digit-reversed copy-out are (nearly) bank-
// conflict free, and the inter-pass twiddles are stored the way the passes read them. The demodulator's phase-
// compensation factors of the R0 bins a thread copies out live in registers for the lifetime of the (persistent) CTA.
// ---------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ int pad16(int i) { return i + (i >> 4) + (i >> 8); }

__device__ __forceinline__ void radix4(float2& a0, float2& a1, float2& a2, float2& a3) {   // b_c = sum_r a_r (-j)^(r c)
    const float2 s02 = cadd(a0, a2), d02 = csub(a0, a2), s13 = cadd(a1, a3), d13 = csub(a1, a3);
    const float2 d13j = make_float2(d13.y, -d13.x);                   // -j (a1 - a3)
    a0 = cadd(s02, s13);
    a1 = cadd(d02, d13j);
    a2 = csub(s02, s13);
    a3 = csub(d02, d13j);
}

// 16-point DFT in place; on return output j' = j1' + 4 j0' is v[4 j1' + j0']
__device__ __forceinline__ void radix16(float2* v) {
    // level 1: radix-4 over j1 for each j0 (elements j0 + 4 j1), then the 16th roots W16^(j0 j1')
#pragma unroll
    for (int j0 = 0; j0 < 4; ++j0) radix4(v[j0], v[j0 + 4], v[j0 + 8], v[j0 + 12]);   // v[j0 + 4 j1'] = a[j0][j1']
    const float c1 = 0.92387953251128674f, s1 = 0.38268343236508977f, h = 0.70710678118654752f;
    // W16^q = (cos(2 pi q / 16), -sin(2 pi q / 16)), q = j0 * j1'
    v[5] = cmul(v[5], make_float2(c1, -s1));          // j0 = 1, j1' = 1: q = 1
    v[9] = cmul(v[9], make_float2(h, -h));            // j0 = 1, j1' = 2: q = 2
    v[13] = cmul(v[13], make_float2(s1, -c1));        // j0 = 1, j1' = 3: q = 3
    v[6] = cmul(v[6], make_float2(h, -h));            // j0 = 2, j1' = 1: q = 2
    v[10] = make_float2(v[10].y, -v[10].x);           // j0 = 2, j1' = 2: q = 4: -j
    v[14] = cmul(v[14], make_float2(-h, -h));         // j0 = 2, j1' = 3: q = 6
    v[7] = cmul(v[7], make_float2(s1, -c1));          // j0 = 3, j1' = 1: q = 3
    v[11] = cmul(v[11], make_float2(-h, -h));         // j0 = 3, j1' = 2: q = 6
    v[15] = cmul(v[15], make_float2(-c1, s1));        // j0 = 3, j1' = 3: q = 9
    // level 2: radix-4 over j0 for each j1' (elements 4 j1' + j0): output j0' lands at v[4 j1' + j0'] = u[j1' + 4 j0']
#pragma unroll
    for (int j1 = 0; j1 < 4; ++j1) radix4(v[4 * j1], v[4 * j1 + 1], v[4 * j1 + 2], v[4 * j1 + 3]);
}

// 8-point DFT in place (j = j0 + 2 j1: radix-4 over j1, the 8th roots, radix-2 over j0); on return output
// j' = j1' + 4 j0' is v[2 j1' + j0']
__device__ __forceinline__ void radix8(float2* v) {
    radix4(v[0], v[2], v[4], v[6]);                   // a[0][j1'] at v[2 j1']
    radix4(v[1], v[3], v[5], v[7]);                   // a[1][j1'] at v[1 + 2 j1']
    const float h = 0.70710678118654752f;
    v[3] = cmul(v[3], make_float2(h, -h));            // W8^1
    v[5] = make_float2(v[5].y, -v[5].x);              // W8^2 = -j
    v[7] = cmul(v[7], make_float2(-h, -h));           // W8^3
#pragma unroll
    for (int j1 = 0; j1 < 4; ++j1) {
        const float2 s = cadd(v[2 * j1], v[2 * j1 + 1]), d = csub(v[2 * j1], v[2 * j1 + 1]);
        v[2 * j1] = s;
        v[2 * j1 + 1] = d;
    }
}

// register index of output j' of the first pass
template <int R0>
__device__ __forceinline__ constexpr int first_pass_slot(int jp) { return R0 == 16 ? 4 * (jp & 3) + (jp >> 2) : 2 * (jp & 3) + (jp >> 2); }

template <int DEMOD, int R0>
__global__ void __launch_bounds__(256, 2) ofdm_fft_r16_kernel(const float2* __restrict__ x, float2* __restrict__ out, int nsym,
                                                           const int* __restrict__ cp, const int* __restrict__ off,
                                                           int len, int l_min, long long rows, int shift) {
    constexpr int N = 256 * R0, PAD = N + N / 16 + N / 256, LOG_R0 = R0 == 16 ? 4 : 3;
    extern __shared__ float2 sm[];
    // twiddles laid out the way the passes read them (lanes along the fastest index: conflict-free):
    //   T0[j' * 256 + m] = W_N^(m j') for pass 0,  T1[j' * 16 + m'] = W_256^(m' j') for pass 1
    float2* T0 = sm;
    float2* T1 = sm + N;
    float2* buf0 = T1 + 256;
    float2* buf1 = buf0 + PAD;
    const int tid = threadIdx.x;
    for (int e = tid; e < N + 256; e += 256) {
        const int k = e < N ? (e & 255) * (e >> 8) : R0 * ((e - N) & 15) * ((e - N) >> 4);   // exponent of W_N, < N
        float sn, cs;
        sincospif(-2.0f * (float)k / (float)N, &sn, &cs);
        sm[e] = make_float2(cs, sn);
    }
    float2 pc[R0];                                                   // demodulator: phase compensation of bins tid + 256 i
    if (DEMOD) {
#pragma unroll
        for (int i = 0; i < R0; ++i) {
            // tmp = -2 pi l_min / N * k in fp32 as the reference computes it, then exp(j tmp)
            const float tmp = -2.0f * 3.14159265358979323846f * (float)l_min / (float)N * (float)(tid + 256 * i);
            pc[i] = make_float2(cosf(tmp), sinf(tmp));
        }
    }
    const float scale = 1.0f / sqrtf((float)N);
    const long long jobs = rows * nsym;
    auto prefetch = [&](long long job, float2* dst) {
        if (job < jobs) {
            if (DEMOD) {
                const long long row = job / nsym;
                const int l = (int)(job - row * nsym);
                const float2* src = x + row * len + off[l] + cp[l];
                for (int k = tid; k < N; k += 256) cp_async8(dst + pad16(k), src + k);
            } else {
                const float2* src = x + job * N;
                for (int k = tid; k < N; k += 256) cp_async8(dst + pad16(k), src + (shift ? ((k + N / 2) & (N - 1)) : k));
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    // position of bin k = j0 + R0 (j1 + 16 j2) in the buffer
    auto bin_pos = [](int k) { return ((k & (R0 - 1)) << 8) | (((k >> LOG_R0) & 15) << 4) | (k >> (LOG_R0 + 4)); };
    float2* cur = buf0;
    float2* nxt = buf1;
    long long job = blockIdx.x;
    prefetch(job, cur);
    for (; job < jobs; job += gridDim.x) {
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();                                             // data of `job` visible; `nxt` no longer read by anyone
        prefetch(job + gridDim.x, nxt);
        float2 v[16];
        // pass 0 (radix R0): n = m + 256 j, m = tid; twiddle W_N^(m j')
        {
            const int m = tid;
#pragma unroll
            for (int j = 0; j < R0; ++j) {
                v[j] = cur[pad16(m + 256 * j)];
                if (!DEMOD) v[j].y = -v[j].y;                        // ifft = conj(fft(conj(.))) / N
            }
            if (R0 == 16) radix16(v); else radix8(v);
#pragma unroll
            for (int jp = 0; jp < R0; ++jp) {
                float2 u = v[first_pass_slot<R0>(jp)];
                if (jp) u = cmul(u, T0[jp * 256 + m]);
                cur[pad16(m + 256 * jp)] = u;
            }
        }
        __syncthreads();
        // pass 1 (radix 16) inside block b of 256 points: m' + 16 j; twiddle W_256^(m' j'); 16 R0 butterflies
        if (tid < 16 * R0) {
            const int b = tid >> 4, mp = tid & 15, base = 256 * b + mp;
#pragma unroll
            for (int j = 0; j < 16; ++j) v[j] = cur[pad16(base + 16 * j)];
            radix16(v);
#pragma unroll
            for (int jp = 0; jp < 16; ++jp) {
                float2 u = v[4 * (jp & 3) + (jp >> 2)];
                if (jp) u = cmul(u, T1[jp * 16 + mp]);
                cur[pad16(base + 16 * jp)] = u;
            }
        }
        __syncthreads();
        // pass 2 (radix 16): 16 contiguous points, no twiddle
        if (tid < 16 * R0) {
            const int base = 16 * tid;
#pragma unroll
            for (int j = 0; j < 16; ++j) v[j] = cur[pad16(base + j)];
            radix16(v);
#pragma unroll
            for (int jp = 0; jp < 16; ++jp) cur[pad16(base + jp)] = v[4 * (jp & 3) + (jp >> 2)];
        }
        __syncthreads();
        // copy-out in natural bin order
        const long long row = job / nsym;
        const int l = (int)(job - row * nsym);
        if (DEMOD) {
            float2* dst = out + job * N;
#pragma unroll
            for (int i = 0; i < R0; ++i) {
                const int k = tid + 256 * i;
                const int ks = shift ? ((k + N / 2) & (N - 1)) : k;  // fftshift
                dst[ks] = cmul(cscale(cur[pad16(bin_pos(k))], scale), pc[i]);
            }
        } else {
            const int c = cp[l];
            float2* dst = out + row * len + off[l];
            for (int i = tid; i < N + c; i += 256) {
                const int k = (i - c) & (N - 1);
                const float2 v0 = cur[pad16(bin_pos(k))];
                dst[i] = make_float2(v0.x * scale, -v0.y * scale);
            }
        }
        { float2* t = cur; cur = nxt; nxt = t; }
    }
    asm volatile("cp.async.wait_group 0;" ::: "memory");
}

template <int DEMOD, int R0>
int launch_fft_r16(const float2* x, float2* out, int nsym, const int* cp, const int* off, int len, int l_min, long long rows,
                   int shift, cudaStream_t stream) {
    constexpr int N = 256 * R0, PAD = N + N / 16 + N / 256;
    const size_t smem = sizeof(float2) * ((size_t)N + 256 + 2 * PAD);
    auto kern = ofdm_fft_r16_kernel<DEMOD, R0>;
    SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<sb_grid(rows * nsym, 1, R0 == 16 ? 2 : 4), 256, smem, stream>>>(x, out, nsym, cp, off, len, l_min, rows, shift);
    return SB_OK;
}

template <int DEMOD>
int launch_fft_pow2(int n, const float2* x, float2* out, int nsym, const int* cp, const int* off, int len, int l_min,
                    long long rows, int shift, cudaStream_t stream) {
    return n == 4096 ? launch_fft_r16<DEMOD, 16>(x, out, nsym, cp, off, len, l_min, rows, shift, stream)
                     : launch_fft_r16<DEMOD, 8>(x, out, nsym, cp, off, len, l_min, rows, shift, stream);
}

// ---------------------------------------------------------------------------------------------------------------
// out[b, r, j] = in[b, (in_rows == 1 ? 0 : r), idx[r, j]]  (idx < 0 -> 0).  WORDS = 32-bit words per element: 1 (float),
// 2 (complex64 / float64) or 4 (complex128) -- a bit copy, so the wider types need no arithmetic variant.
template <int WORDS>
__global__ void gather_rows_kernel(const float* __restrict__ in, const int* __restrict__ idx, float* __restrict__ out,
                                   long long B, int R, int J, int in_rows, int L) {
    const long long rows = B * R;
    for (long long row = (long long)blockIdx.x * blockDim.y + threadIdx.y; row < rows; row += (long long)gridDim.x * blockDim.y) {
        const int r = (int)(row % R);
        const long long b = row / R;
        const int* ip = idx + (size_t)r * J;
        const float* src = in + (b * in_rows + (in_rows == 1 ? 0 : r)) * (long long)L * WORDS;
        float* dst = out + row * (long long)J * WORDS;
        for (int j = threadIdx.x; j < J; j += blockDim.x) {
            const int sidx = ip[j];
            if (WORDS == 4) {
                reinterpret_cast<float4*>(dst)[j] = sidx < 0 ? make_float4(0.f, 0.f, 0.f, 0.f) : reinterpret_cast<const float4*>(src)[sidx];
            } else if (WORDS == 2) {
                reinterpret_cast<float2*>(dst)[j] = sidx < 0 ? make_float2(0.f, 0.f) : reinterpret_cast<const float2*>(src)[sidx];
            } else {
                dst[j] = sidx < 0 ? 0.f : src[sidx];
            }
        }
    }
}

// ResourceGridMapper: map[ts, g] >= 0: data symbol index; -1: zero; <= -2: pilot index -(v + 2)
__global__ void rg_map_kernel(const float2* __restrict__ x, const float2* __restrict__ pilots, const int* __restrict__ map,
                              float2* __restrict__ out, long long B, int TS, int G, int D, int P) {
    const long long rows = B * TS;
    for (long long row = (long long)blockIdx.x * blockDim.y + threadIdx.y; row < rows; row += (long long)gridDim.x * blockDim.y) {
        const int ts = (int)(row % TS);
        const int* mp = map + (size_t)ts * G;
        const float2* xp = x + row * (long long)D;
        const float2* pp = pilots + (size_t)ts * P;
        float2* op = out + row * (long long)G;
        for (int g = threadIdx.x; g < G; g += blockDim.x) {
            const int v = mp[g];
            float2 o = make_float2(0.f, 0.f);
            if (v >= 0) o = xp[v];
            else if (v <= -2) o = pp[-(v + 2)];
            op[g] = o;
        }
    }
}

// LS estimate at the pilot positions: h[b, ts, p] = y[b, pilot_ind[ts, p]] / pilots[ts, p] (0 where the pilot is 0),
// err[b, ts, p] = no[b / no_inner] / |pilots|^2 (0 where the pilot is 0)   (channel_estimation.py:138-150, 257-285)
__global__ void ls_at_pilots_kernel(const float2* __restrict__ y, const int* __restrict__ pilot_ind,
                                    const float2* __restrict__ pilots, const float* __restrict__ no, long long no_inner,
                                    float2* __restrict__ h, float* __restrict__ err, long long B, int TS, int P, int L) {
    const long long rows = B * TS;
    for (long long row = (long long)blockIdx.x * blockDim.y + threadIdx.y; row < rows; row += (long long)gridDim.x * blockDim.y) {
        const int ts = (int)(row % TS);
        const long long b = row / TS;
        const float2* yp = y + b * (long long)L;
        const float nb = no[b / no_inner];
        for (int q = threadIdx.x; q < P; q += blockDim.x) {
            const float2 pl = pilots[(size_t)ts * P + q];
            const float2 yy = yp[pilot_ind[(size_t)ts * P + q]];
            const float a2 = pl.x * pl.x + pl.y * pl.y;
            const bool z = (pl.x == 0.f && pl.y == 0.f);
            h[row * P + q] = z ? make_float2(0.f, 0.f) : cdiv(yy, pl);
            const float ab = sqrtf(a2);                 // tf.abs(pilots)**2
            err[row * P + q] = z ? 0.f : nb / (ab * ab);
        }
    }
}

// LinearInterpolator (channel_estimation.py:657-734): frequency interpolation on the pilot-carrying OFDM symbols, optional
// time averaging, then time interpolation. Tables per stream row ts (host, channel_estimation.py:522-655):
//   fx0/fx1 [TS, S, F] pilot subcarrier positions (-1 if the symbol has no pilot), fy0/fy1 [TS, S, F] pilot indices + 1
//   (0 = the zero pad), ty0/ty1 [TS, S] OFDM symbol indices used for the time interpolation, npil [TS] number of
//   pilot-carrying symbols. in: h [B, TS, P] -> out [B, TS, S, F].
__device__ __forceinline__ float2 lerp_c(float x, float x0, float x1, float2 y0, float2 y1) {
    float dx = x1 - x0;
    float2 slope = dx == 0.f ? make_float2(0.f, 0.f) : make_float2((y1.x - y0.x) / dx, (y1.y - y0.y) / dx);   // divide_no_nan
    float t = x - x0;
    return make_float2(t * slope.x + y0.x, t * slope.y + y0.y);
}
__device__ __forceinline__ float lerp_c(float x, float x0, float x1, float y0, float y1) {
    float dx = x1 - x0;
    float slope = dx == 0.f ? 0.f : (y1 - y0) / dx;
    return (x - x0) * slope + y0;
}
__device__ __forceinline__ float2 vzero(float2) { return make_float2(0.f, 0.f); }
__device__ __forceinline__ float vzero(float) { return 0.f; }
__device__ __forceinline__ float2 vfloor0(float2 a) { return a; }            // only real error variances are floored
__device__ __forceinline__ float vfloor0(float a) { return fmaxf(a, 0.f); }
__device__ __forceinline__ float2 vadd(float2 a, float2 b) { return cadd(a, b); }
__device__ __forceinline__ float vadd(float a, float b) { return a + b; }
__device__ __forceinline__ float2 vdiv(float2 a, float n) { return make_float2(a.x / n, a.y / n); }
__device__ __forceinline__ float vdiv(float a, float n) { return a / n; }

template <typename T>
__device__ __forceinline__ T freq_interp(const T* hp, const int* fx0, const int* fx1, const int* fy0, const int* fy1, int idx,
                                         int f) {
    int i0 = fy0[idx], i1 = fy1[idx];
    T y0 = i0 > 0 ? hp[i0 - 1] : vzero(T());
    T y1 = i1 > 0 ? hp[i1 - 1] : vzero(T());
    return lerp_c((float)f, (float)fx0[idx], (float)fx1[idx], y0, y1);
}
// T = float2 (channel estimates) or float (error variances). A CTA owns (batch', stream) rows; a thread owns one
// subcarrier column f of the row and walks the OFDM symbols: the two frequency-interpolated values y(s0, f), y(s1, f) a
// symbol interpolates between are re-evaluated only when (s0, s1) changes (once or twice per slot), so an output costs
// two table words + one lerp; stores are contiguous over f.
template <typename T>
__global__ void interp_lin_kernel(const T* __restrict__ h, const int* __restrict__ fx0, const int* __restrict__ fx1,
                                  const int* __restrict__ fy0, const int* __restrict__ fy1, const int* __restrict__ ty0,
                                  const int* __restrict__ ty1, const int* __restrict__ npil, int flags,
                                  T* __restrict__ out, long long B, int TS, int S, int F, int P) {
    const int time_avg = flags & 1;
    const bool floor0 = (flags & 2) != 0;                       // error variances: max(., 0) after interpolation (:171)
    const int SF = S * F;
    const long long rows = B * TS;
    for (long long row = blockIdx.x; row < rows; row += gridDim.x) {
        const int ts = (int)(row % TS);
        const T* hp = h + row * (long long)P;
        T* op = out + row * (long long)SF;
        const int base = ts * SF;
        for (int f = threadIdx.x; f < F; f += blockDim.x) {
            if (time_avg) {
                T acc = vzero(T());
                for (int s2 = 0; s2 < S; ++s2) acc = vadd(acc, freq_interp<T>(hp, fx0, fx1, fy0, fy1, base + s2 * F + f, f));
                T v = vdiv(acc, (float)npil[ts]);              // every symbol carries the average: time interpolation is flat
                if (floor0) v = vfloor0(v);
                for (int s = 0; s < S; ++s) op[s * F + f] = v;
            } else {
                int last0 = -1, last1 = -1;
                T y0 = vzero(T()), y1 = vzero(T());
                for (int s = 0; s < S; ++s) {
                    const int s0 = ty0[ts * S + s], s1 = ty1[ts * S + s];
                    if (s0 != last0) { y0 = freq_interp<T>(hp, fx0, fx1, fy0, fy1, base + s0 * F + f, f); last0 = s0; }
                    if (s1 != last1) { y1 = freq_interp<T>(hp, fx0, fx1, fy0, fy1, base + s1 * F + f, f); last1 = s1; }
                    T v = lerp_c((float)s, (float)s0, (float)s1, y0, y1);
                    if (floor0) v = vfloor0(v);
                    op[s * F + f] = v;
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Dense per-vector linear algebra, complex64, one thread per received vector; matrices live in shared memory interleaved
// by thread (Scratch, dense_mimo.cuh). The LMMSE kernels and the mimo_linalg modes are compositions of these steps:
//   chol_lower, whiten                                                        (dense_mimo.cuh)
//   tx_lmmse_matrix  G = (H^H H + r I)^-1 H^H via chol + cholesky_solve      (mimo/equalization.py:95-97; r = 0:
//                    matrix_pinv, utils/linalg.py)
//   lmmse_epilogue   x_hat = G y / diag(G H), no_eff = Re(1 / diag(G H) - 1)  (mimo/equalization.py:217-231)
//   herm_quad        Re g S g^H of a row vector g from S's lower triangle      (diag(G S G^H), :335-342, :459-464)
// ---------------------------------------------------------------------------------------------------------------
// G = (H^H H + ridge I)^-1 H^H (K x M) for H (M x K): A = H^H H + ridge I = C C^H (K x K, A is overwritten by C), then
// C C^H G = H^H column by column. ridge 1: LMMSE (the diagonal starts at 1, as before the argument existed); 0: the
// pseudo-inverse.
__device__ void tx_lmmse_matrix(const Scratch& H, const Scratch& A, const Scratch& G, int M, int K, float ridge) {
    for (int a = 0; a < K; ++a)
        for (int b = 0; b <= a; ++b) {
            float2 acc = make_float2(a == b ? ridge : 0.f, 0.f);
            for (int m = 0; m < M; ++m) acc = cadd(acc, cmulc(H(m * K + b), H(m * K + a)));   // conj(H[m,a]) * H[m,b]
            A(a * K + b) = acc;
        }
    chol_lower(A, K);
    for (int m = 0; m < M; ++m)
        chol_solve_col(A, K, [&](int k) { float2 v = H(m * K + k); v.y = -v.y; return v; }, G, M, m);
}

// xh[k] = (G y)_k / (G H)_kk, ne[k] = Re(1 / (G H)_kk - 1) for k < K, with G[k, m] = g(k, m), y[m] = y(m), H (M x K)
template <typename GF, typename YF>
__device__ __forceinline__ void lmmse_epilogue(const GF& g, const YF& y, const Scratch& H, int M, int K, float2* xh, float* ne) {
    for (int k = 0; k < K; ++k) {
        float2 gy = make_float2(0.f, 0.f), dd = make_float2(0.f, 0.f);
        for (int m = 0; m < M; ++m) {
            const float2 gkm = g(k, m);
            gy = cadd(gy, cmul(gkm, y(m)));
            dd = cadd(dd, cmul(gkm, H(m * K + k)));
        }
        xh[k] = cdiv(gy, dd);
        float2 inv = cdiv(make_float2(1.f, 0.f), dd);
        ne[k] = inv.x - 1.f;
    }
}

// Re(g S g^H) = sum_a S_aa |g_a|^2 + 2 Re sum_{a > b} g_a S_ab conj(g_b) for Hermitian S, of which only the lower
// triangle s(a, b), a >= b, is read; g(a) = g_a, a < n
template <typename SF, typename GF>
__device__ __forceinline__ float herm_quad(const SF& s, const GF& g, int n) {
    float diag = 0.f, off = 0.f;
    for (int a = 0; a < n; ++a) {
        const float2 ga = g(a);
        diag += s(a, a).x * (ga.x * ga.x + ga.y * ga.y);
        float2 t = make_float2(0.f, 0.f);
        for (int b = 0; b < a; ++b) t = cadd(t, cmulc(s(a, b), g(b)));                // sum_b S_ab conj(g_b)
        off += ga.x * t.x - ga.y * t.y;                                                   // Re(g_a t)
    }
    return diag + 2.f * off;
}

// ZF / MF per vector from H (M x K) in scratch, y(m) and the noise covariance's lower triangle s(a, b):
//   ZF (mimo/equalization.py:316-342): G = matrix_pinv(H) = (H^H H)^-1 H^H in G (K x M, A = chol(H^H H) scratch),
//      x_hat = G y, no_eff = Re diag(G S G^H)
//   MF (:437-464): B = H^H H, x_hat_k = (H^H y)_k / B_kk and, with G = diag(B)^-1 H^H, whose (I - G H) row k is
//      -B_kj / B_kk off the diagonal and 0 on it,  no_eff_k = (sum_{j != k} |B_kj|^2 + h_k^H S h_k) / B_kk^2
template <typename YF, typename SF>
__device__ void zf_core(const Scratch& H, const YF& y, const Scratch& A, const Scratch& G, const SF& s, int M, int K,
                        float2* xh, float* ne) {
    tx_lmmse_matrix(H, A, G, M, K, 0.f);
    for (int k = 0; k < K; ++k) {
        float2 gy = make_float2(0.f, 0.f);
        for (int m = 0; m < M; ++m) gy = cadd(gy, cmul(G(k * M + m), y(m)));
        xh[k] = gy;
        ne[k] = herm_quad(s, [&](int m) { return G(k * M + m); }, M);
    }
}
template <typename YF, typename SF>
__device__ void mf_core(const Scratch& H, const YF& y, const SF& s, int M, int K, float2* xh, float* ne) {
    for (int k = 0; k < K; ++k) {
        float bkk = 0.f, off = 0.f;
        float2 z = make_float2(0.f, 0.f);
        for (int m = 0; m < M; ++m) {
            const float2 h = H(m * K + k);
            bkk += h.x * h.x + h.y * h.y;
            z = cadd(z, cmulc(y(m), h));                                                  // conj(H_mk) y_m
        }
        for (int j = 0; j < K; ++j) {
            if (j == k) continue;
            float2 b = make_float2(0.f, 0.f);
            for (int m = 0; m < M; ++m) b = cadd(b, cmulc(H(m * K + j), H(m * K + k)));   // B_kj
            off += b.x * b.x + b.y * b.y;
        }
        const float q = herm_quad(s, [&](int m) { float2 h = H(m * K + k); h.y = -h.y; return h; }, M);
        const float inv = 1.f / bkk;
        xh[k] = cscale(z, inv);
        ne[k] = fabsf((off + q) * inv * inv);
    }
}

// LMMSE equalisation of one received vector with noise covariance S (mimo/equalization.py:101-233, whitening
// mimo/utils.py:292-357). Per-thread scratch: S [M, M], H [M, K], y [M], A [K, K], G [K, M].
struct LmmseScratch {
    Scratch S, H, Y, A, G;
    __device__ __forceinline__ LmmseScratch(float2* smem, int T, int t, int M, int K)
        : S{smem, T, t}, H{smem + (size_t)M * M * T, T, t}, Y{smem + (size_t)(M * M + M * K) * T, T, t},
          A{smem + (size_t)(M * M + M * K + M) * T, T, t}, G{smem + (size_t)(M * M + M * K + M + K * K) * T, T, t} {}
    static size_t elems(int M, int K) {                                                     // per thread
        const size_t m = (size_t)M, k = (size_t)K;
        return m * m + m * k + m + k * k + k * m;
    }
};

// in: S (M x M, row-major, lower triangle read), H (M x K), y (M). out: xh[K], ne[K].
__device__ void lmmse_core(const LmmseScratch& w, int M, int K, float2* xh, float* ne) {
    chol_lower(w.S, M);
    whiten(w.S, w.Y, w.H, M, K);
    tx_lmmse_matrix(w.H, w.A, w.G, M, K, 1.f);
    lmmse_epilogue([&](int k, int m) { return w.G(k * M + m); }, w.Y, w.H, M, K, xh, ne);
}

// lmmse_equalizer(y [R, M], h [R, M, K], s [R, M, M]) -> x_hat [R, K], no_eff [R, K]
__global__ void lmmse_kernel(const float2* __restrict__ y, const float2* __restrict__ h, const float2* __restrict__ s,
                             float2* __restrict__ xh, float* __restrict__ ne, long long R, int M, int K) {
    extern __shared__ float2 smem[];
    const int T = blockDim.x, t = threadIdx.x;
    const LmmseScratch w(smem, T, t, M, K);
    float2 xo[16];
    float no[16];
    for (long long r = (long long)blockIdx.x * T + t; r < R; r += (long long)gridDim.x * T) {
        for (int e = 0; e < M * M; ++e) w.S(e) = s[r * M * M + e];
        for (int e = 0; e < M * K; ++e) w.H(e) = h[r * M * K + e];
        for (int e = 0; e < M; ++e) w.Y(e) = y[r * M + e];
        lmmse_core(w, M, K, xo, no);
        for (int k = 0; k < K; ++k) { xh[r * K + k] = xo[k]; ne[r * K + k] = no[k]; }
    }
}

// ---- the reference's small dense helpers as callable kernels (thread per matrix, scratch interleaved in shared memory) ---
//   mode 0  inv_cholesky(s)            utils/linalg.py:8-32          out0 = L^-1 [R, M, M] (lower triangular)
//   mode 1  whiten_channel(y, h, s)    mimo/utils.py:292-357         out0 = L^-1 y [R, M], out1 = L^-1 H [R, M, K]
//   mode 2  lmmse_matrix(h, s)         mimo/equalization.py:11-99    out0 = G = H^H (H H^H + S)^-1 [R, K, M]; s == nullptr:
//                                                                    G = (H^H H + I)^-1 H^H
//   mode 3  lmmse_equalizer(whiten_interference=False)  :183-233     out0 = x_hat [R, K], out1 = no_eff [R, K] (float)
//   mode 4  zf_equalizer(y, h, s)      mimo/equalization.py:235-343  out0 = x_hat [R, K], out1 = no_eff [R, K] (float)
//   mode 5  mf_equalizer(y, h, s)      mimo/equalization.py:345-466  out0 = x_hat [R, K], out1 = no_eff [R, K] (float)
//   mode 6  matrix_pinv(h)             utils/linalg.py               out0 = (H^H H)^-1 H^H [R, K, M]
__global__ void mimo_linalg_kernel(int mode, const float2* __restrict__ y, const float2* __restrict__ h,
                                   const float2* __restrict__ s, float2* __restrict__ out0, void* __restrict__ out1v,
                                   long long R, int M, int K) {
    extern __shared__ float2 smem[];
    const int T = blockDim.x, t = threadIdx.x;
    const bool rx_side = !(mode == 2 && s == nullptr);             // factorise the M x M receive-side matrix (else K x K)
    Scratch A{smem, T, t}, H{smem + (size_t)M * M * T, T, t}, X{smem + (size_t)(M * M + M * K) * T, T, t};
    for (long long r = (long long)blockIdx.x * T + t; r < R; r += (long long)gridDim.x * T) {
        if (h) for (int e = 0; e < M * K; ++e) H(e) = h[r * M * K + e];
        if (mode <= 1) {                                            // L = chol(S), then L^-1 by forward substitution
            for (int e = 0; e < M * M; ++e) A(e) = s[r * M * M + e];
            chol_lower(A, M);
            if (mode == 0) {
                for (int c = 0; c < M; ++c)
                    for (int i = 0; i < M; ++i) {
                        float2 v = make_float2(i == c ? 1.f : 0.f, 0.f);
                        for (int k = c; k < i; ++k) v = csub(v, cmul(A(i * M + k), X(k * M + c)));
                        float d = A(i * M + i).x;
                        X(i * M + c) = i < c ? make_float2(0.f, 0.f) : make_float2(v.x / d, v.y / d);
                    }
                for (int e = 0; e < M * M; ++e) out0[r * M * M + e] = X(e);
            } else {
                float2* hw = reinterpret_cast<float2*>(out1v);
                for (int i = 0; i < M; ++i) X(i) = y[r * M + i];
                whiten(A, X, H, M, K);
                for (int i = 0; i < M; ++i) out0[r * M + i] = X(i);
                for (int e = 0; e < M * K; ++e) hw[r * M * K + e] = H(e);
            }
            continue;
        }
        if (mode >= 4) {                                            // ZF, MF, pinv: K x K Gram matrix in A, G in X
            const long long rs = r * M * M;
            const auto sf = [&](int a, int b) { return s[rs + a * M + b]; };
            const auto yf = [&](int m) { return y[r * M + m]; };
            if (mode == 4) {
                zf_core(H, yf, A, X, sf, M, K, out0 + r * K, reinterpret_cast<float*>(out1v) + r * K);
            } else if (mode == 5) {
                mf_core(H, yf, sf, M, K, out0 + r * K, reinterpret_cast<float*>(out1v) + r * K);
            } else {
                tx_lmmse_matrix(H, A, X, M, K, 0.f);
                for (int e = 0; e < K * M; ++e) out0[r * K * M + e] = X(e);
            }
            continue;
        }
        // modes 2, 3: G
        if (rx_side) {                                              // G^H = (H H^H + S)^-1 H, column by column
            for (int a = 0; a < M; ++a)
                for (int b = 0; b <= a; ++b) {
                    float2 acc = s[r * M * M + a * M + b];
                    for (int k = 0; k < K; ++k) acc = cadd(acc, cmulc(H(a * K + k), H(b * K + k)));
                    A(a * M + b) = acc;
                }
            chol_lower(A, M);
            for (int c = 0; c < K; ++c) chol_solve_col(A, M, [&](int i) { return H(i * K + c); }, X, K, c);   // X = G^H [M, K]
        } else {
            tx_lmmse_matrix(H, A, X, M, K, 1.f);                           // X = G [K, M]
        }
        if (mode == 2) {
            for (int k = 0; k < K; ++k)
                for (int m = 0; m < M; ++m) {
                    float2 g = X(k * M + m);
                    if (rx_side) { g = X(m * K + k); g.y = -g.y; }                 // G = (G^H)^H
                    out0[(r * K + k) * M + m] = g;
                }
        } else {                                                    // mode 3 has s: X = G^H
            float* ne = reinterpret_cast<float*>(out1v);
            lmmse_epilogue([&](int k, int m) { float2 g = X(m * K + k); g.y = -g.y; return g; },
                           [&](int m) { return y[r * M + m]; }, H, M, K, out0 + r * K, ne + r * K);
        }
    }
}

// Equalisers of sb_ofdm_equalize
enum { EQ_LMMSE = 0, EQ_LMMSE_NO_WHITEN = 1, EQ_ZF = 2, EQ_MF = 3 };

// One resource element of ofdm_linear_kernel: S (lower triangle, ofdm_load_re), H, y in w -> xh[K], ne[K]
template <int EQ>
__device__ __forceinline__ void linear_core(const LmmseScratch& w, int M, int K, float2* xh, float* ne) {
    const auto sf = [&](int a, int b) { return w.S(a * M + b); };
    const auto yf = [&](int m) { return w.Y(m); };
    if constexpr (EQ == EQ_LMMSE) {
        lmmse_core(w, M, K, xh, ne);
    } else if constexpr (EQ == EQ_LMMSE_NO_WHITEN) {              // as sb_mimo_linalg mode 3: (H H^H + S) G^H = H
        for (int a = 0; a < M; ++a)
            for (int b = 0; b <= a; ++b) {
                float2 acc = w.S(a * M + b);
                for (int k = 0; k < K; ++k) acc = cadd(acc, cmulc(w.H(a * K + k), w.H(b * K + k)));
                w.S(a * M + b) = acc;
            }
        chol_lower(w.S, M);
        for (int c = 0; c < K; ++c) chol_solve_col(w.S, M, [&](int i) { return w.H(i * K + c); }, w.G, K, c);
        lmmse_epilogue([&](int k, int m) { float2 g = w.G(m * K + k); g.y = -g.y; return g; }, yf, w.H, M, K, xh, ne);
    } else if constexpr (EQ == EQ_ZF) {
        zf_core(w.H, yf, w.A, w.G, sf, M, K, xh, ne);
    } else {
        mf_core(w.H, yf, sf, M, K, xh, ne);
    }
}

// OFDMEqualizer + a linear equaliser fused (inputs and tables: OfdmEqParams, dense_mimo.cuh) -> x_hat / no_eff
// [B, TXS, num_data]
template <int EQ>
__global__ void ofdm_linear_kernel(const OfdmEqParams p) {
    extern __shared__ float2 smem[];
    const int T = blockDim.x, t = threadIdx.x, M = p.ANT, K = p.K;
    const LmmseScratch w(smem, T, t, M, K);
    float2 xo[16];
    float no_e[16];
    const long long total = p.B * p.RX * (long long)p.S * p.F;
    for (long long i = (long long)blockIdx.x * T + t; i < total; i += (long long)gridDim.x * T) {
        const sb_dense::OfdmRe e = sb_dense::ofdm_re(p, i);
        // skip resource elements that carry data for none of this receiver's streams
        if (!sb_dense::ofdm_re_has_data(p, e)) continue;
        sb_dense::ofdm_load_re(p, e, w.Y, w.H, w.S);
        linear_core<EQ>(w, M, K, xo, no_e);
        for (int k = 0; k < K; ++k) {
            const long long o = sb_dense::ofdm_out_index(p, e, k);
            if (o >= 0) {
                p.xh[o] = xo[k];
                p.ne[o] = no_e[k];
            }
        }
    }
}

// Fast path of ofdm_linear_kernel for receivers without interfering streams (KU == 0): S = D = diag(no + sum err_var)
// is diagonal and everything fits in registers. One thread per resource element streams once over the antennas (reads
// coalesced over the subcarrier index) and accumulates
//   LMMSE:   B = H_w^H H_w (K x K Hermitian, lower triangle) and z = H_w^H y_w,  H_w = H / sqrt(d), y_w = y / sqrt(d)
//            then A = B + I = C C^H, A^-1 = C^-H C^-1 and, without forming G = A^-1 H_w^H (K x M),
//            G y_w = A^-1 z,   diag(G H_w)_k = sum_j (A^-1)_kj B_jk          (same quantities as lmmse_core)
//   ZF, MF:  B = H^H H, z = H^H y and C = H^H D H (ZF: lower triangle, MF: diagonal) of the unwhitened channel
//            (lmmse_diag.cuh: zf_diag_solve, mf_diag_solve)
// LMMSE without whitening runs the LMMSE instantiation when M >= K + 2: with a diagonal S both forms are the same
// estimate. On (nearly) square systems the whitened register solve's single-precision error exceeds the unwhitened
// evaluation's (10x at M = K = 3), so M <= K + 1 runs the shared-memory kernel, which keeps the unwhitened steps.
// ZF holds the full C
// besides B and the chunk's loads; it runs 3 CTAs per SM (2 at K = 4), which leaves it the registers to do so without
// spilling.
template <int EQ, int K>
__global__ void __launch_bounds__(128, EQ == EQ_ZF ? (K == 4 ? 2 : 3) : 4) ofdm_linear_diag_kernel(const OfdmEqParams p) {
    const long long SF = (long long)p.S * p.F;
    const long long total = p.B * p.RX * SF;
    const int M = p.ANT;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        long long re = i % SF;
        int rx = (int)((i / SF) % p.RX);
        long long b = i / (SF * p.RX);
        int s = (int)(re / p.F), f = (int)(re % p.F);
        int ts[K], dp[K];
        bool any = false;
#pragma unroll
        for (int k = 0; k < K; ++k) {
            ts[k] = p.out_ts[rx * K + k];
            dp[k] = p.data_pos[(size_t)ts[k] * SF + re];
            any = any || dp[k] >= 0;
        }
        if (!any) continue;
        int des[K];
#pragma unroll
        for (int k = 0; k < K; ++k) des[k] = p.des[rx * K + k];
        float2 Bm[K * (K + 1) / 2], z[K];
        sb_lmmse::lmmse_diag_clear<K>(Bm, z);
        constexpr int NC = EQ == EQ_ZF ? K * (K + 1) / 2 : K;
        float2 Cm[NC];                                                              // C = H^H D H (ZF, MF)
#pragma unroll
        for (int e = 0; e < NC; ++e) Cm[e] = make_float2(0.f, 0.f);
        // antennas in chunks of 4: all loads of a chunk (y, K channel columns, the error variances, no) are issued before
        // any of them is used, so 4 * (K + 1) 8-byte loads per thread are in flight instead of one dependent load at a
        // time (the one-antenna-per-trip version was latency bound: long_scoreboard 3.4 warps per issue, 27 % of HBM peak).
        // Running pointers (one 64-bit add per array and antenna) instead of a 64-bit product per load.
        constexpr int CH = 4;
        const long long row0 = (b * p.RX + rx) * M;
        const float2* yp = p.y + row0 * SF + re;                                    // antenna stride SF
        const float2* hp[K];
#pragma unroll
        for (int k = 0; k < K; ++k) hp[k] = p.hhat + (row0 * p.TXS + des[k]) * SF + re;   // antenna stride TXS * SF
        const long long hstep = (long long)p.TXS * SF;
        const float* evp = p.ev + b * p.ev_stride[0] + rx * p.ev_stride[1] + s * p.ev_stride[4] + f * p.ev_stride[5];
        const float* nop = p.no + b * p.no_stride[0] + rx * p.no_stride[1];
        const long long ev_m = p.ev_stride[2], ev_q = p.ev_stride[3], no_m = p.no_stride[2];
        auto accumulate = [&](float2 yv, const float2* hv, float d) {
            if constexpr (EQ == EQ_LMMSE) {
                // whitening by 1 / sqrt(d): one division per antenna, multiplications for the K + 1 scalings
                const float w = rsqrtf(d);                                    // MUFU.RSQ, <= 2 ulp
                const float2 yw = make_float2(yv.x * w, yv.y * w);
                float2 hw[K];
#pragma unroll
                for (int k = 0; k < K; ++k) hw[k] = make_float2(hv[k].x * w, hv[k].y * w);
#pragma unroll
                for (int a = 0; a < K; ++a) {
                    z[a] = cadd(z[a], cmulc(yw, hw[a]));                       // conj(H_w[m, a]) * y_w[m]
#pragma unroll
                    for (int q = 0; q <= a; ++q) Bm[a * (a + 1) / 2 + q] = cadd(Bm[a * (a + 1) / 2 + q], cmulc(hw[q], hw[a]));
                }
            } else {
#pragma unroll
                for (int a = 0; a < K; ++a) {
                    z[a] = cadd(z[a], cmulc(yv, hv[a]));                       // conj(H[m, a]) * y[m]
#pragma unroll
                    for (int q = 0; q <= a; ++q) {
                        const float2 b = cmulc(hv[q], hv[a]);                  // conj(H[m, a]) * H[m, q]
                        Bm[a * (a + 1) / 2 + q] = cadd(Bm[a * (a + 1) / 2 + q], b);
                        if constexpr (EQ == EQ_ZF) Cm[a * (a + 1) / 2 + q] = cadd(Cm[a * (a + 1) / 2 + q], cscale(b, d));
                        else if (q == a) Cm[a].x += d * b.x;
                    }
                }
            }
        };
        int m0 = 0;
#pragma unroll 1
        for (; m0 + CH <= M; m0 += CH) {
            float2 yv[CH], hv[CH][K];
            float dv[CH];
#pragma unroll
            for (int c = 0; c < CH; ++c) {
                yv[c] = yp[c * SF];
#pragma unroll
                for (int k = 0; k < K; ++k) hv[c][k] = hp[k][c * hstep];
                float evs = 0.f;
                for (int q = 0; q < p.TXS; ++q) evs += evp[(m0 + c) * ev_m + q * ev_q];
                dv[c] = nop[(m0 + c) * no_m] + evs;
            }
            yp += CH * SF;
#pragma unroll
            for (int k = 0; k < K; ++k) hp[k] += CH * hstep;
#pragma unroll
            for (int c = 0; c < CH; ++c) accumulate(yv[c], hv[c], dv[c]);
        }
#pragma unroll 1
        for (; m0 < M; ++m0) {                                                      // M not a multiple of 4
            float2 hv[K];
#pragma unroll
            for (int k = 0; k < K; ++k) { hv[k] = *hp[k]; hp[k] += hstep; }
            float evs = 0.f;
            for (int q = 0; q < p.TXS; ++q) evs += evp[m0 * ev_m + q * ev_q];
            accumulate(*yp, hv, nop[m0 * no_m] + evs);
            yp += SF;
        }
        float2 xo[K];
        float no_e[K];
        if constexpr (EQ == EQ_LMMSE) sb_lmmse::lmmse_diag_solve<K>(Bm, z, xo, no_e);
        else if constexpr (EQ == EQ_ZF) sb_lmmse::zf_diag_solve<K>(Bm, Cm, z, xo, no_e);
        else sb_lmmse::mf_diag_solve<K>(Bm, Cm, z, xo, no_e);
#pragma unroll
        for (int k = 0; k < K; ++k) {
            if (dp[k] >= 0) {
                p.xh[(b * p.TXS + ts[k]) * (long long)p.ND + dp[k]] = xo[k];
                p.ne[(b * p.TXS + ts[k]) * (long long)p.ND + dp[k]] = no_e[k];
            }
        }
    }
}

int make_plan(int n, FftPlan* plan) {
    plan->n = n;
    plan->n_radix = 0;
    int m = n;
    auto push = [&](int p) { if (plan->n_radix >= 24) return -1; plan->radix[plan->n_radix++] = p; return 0; };
    while (m % 4 == 0) { if (push(4)) return -1; m /= 4; }
    for (int p = 2; m > 1; ++p) {
        if ((long long)p * p > m) p = m;             // remaining m is prime
        while (m % p == 0) { if (push(p)) return -1; m /= p; }
    }
    int span = 1;
    for (int st = 0; st < plan->n_radix; ++st) {
        int lg = -1;
        if ((span & (span - 1)) == 0) { lg = 0; while ((1 << lg) < span) ++lg; }
        plan->span_shift[st] = lg;
        span *= plan->radix[st];
    }
    return 0;
}

// Host side of the small-FFT path: the stage radices (the plan travels as a kernel parameter).
int get_small_plan(int n, SmallFftPlan* out) {
    FftPlan fp;
    if (make_plan(n, &fp) != 0 || fp.n_radix > 12) { sb_set_error("fft size %d has too many factors", n); return SB_EUNSUPPORTED; }
    SmallFftPlan sp{};
    sp.n = n;
    sp.n_stages = fp.n_radix;
    int span = 1;
    for (int st = 0; st < fp.n_radix; ++st) {
        sp.p[st] = fp.radix[st];
        const unsigned nb = (unsigned)(n / sp.p[st]);                  // divisor 1 is special-cased in the kernel
        sp.mg_nb[st] = nb == 1 ? 0u : (unsigned)(((1ull << 32) + nb - 1) / nb);
        sp.mg_span[st] = span == 1 ? 0u : (unsigned)(((1ull << 32) + (unsigned)span - 1) / (unsigned)span);
        span *= sp.p[st];
    }
    const int primes[7] = {3, 5, 7, 11, 13, 17, 19};
    for (int P : primes)
        for (int j = 0; j < P; ++j) {
            const double t = -2.0 * 3.14159265358979323846 * (double)j / (double)P;
            sp.roots[root_offset(P) + j] = make_float2((float)cos(t), (float)sin(t));
        }
    *out = sp;
    return SB_OK;
}

constexpr int kSmallFftMax = 1024;

template <int DEMOD, int FPW>
int launch_fft_small_fpw(const SmallFftPlan& sp, const float2* x, float2* out, int nsym, const int* cp, const int* off,
                         int len, int l_min, long long rows, int shift, cudaStream_t stream) {
    const int warps = 8, n = sp.n;
    size_t smem = sizeof(float2) * (size_t)n * ((DEMOD ? 2 : 1) + 3 * FPW * warps);
    auto kern = ofdm_fft_small_kernel<DEMOD, FPW>;
    SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ = 1;
    SB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, warps * 32, smem));
    const int grid = sb_grid(rows * nsym, warps * FPW, std::max(1, occ));
    kern<<<grid, warps * 32, smem, stream>>>(x, out, sp, nsym, cp, off, len, l_min, rows, shift);
    return SB_OK;
}

template <int DEMOD>
int launch_fft_small(const float2* x, float2* out, int n, int nsym, const int* cp, const int* off, int len, int l_min,
                     long long rows, int shift, cudaStream_t stream) {
    SmallFftPlan sp;
    int rc = get_small_plan(n, &sp);
    if (rc) return rc;
    // transforms per warp. Measured at N = 76, modulator / demodulator ms per 458 k transforms: 2 -> 0.39 / 0.37,
    // 4 -> 0.277 / 0.254, 8 -> 0.34 / 0.29 (8 halves the resident warps per SM).
    const int fpw = n <= 128 ? 4 : (n <= 256 ? 2 : 1);         // three buffers of fpw transforms per warp, 2 CTAs per SM
    if (fpw == 4) return launch_fft_small_fpw<DEMOD, 4>(sp, x, out, nsym, cp, off, len, l_min, rows, shift, stream);
    if (fpw == 2) return launch_fft_small_fpw<DEMOD, 2>(sp, x, out, nsym, cp, off, len, l_min, rows, shift, stream);
    return launch_fft_small_fpw<DEMOD, 1>(sp, x, out, nsym, cp, off, len, l_min, rows, shift, stream);
}

// Body of sb_ofdm_modulate (DEMOD = 0) and sb_ofdm_demodulate (DEMOD = 1), `name` is the entry point named in errors.
// N <= 1024: warp-per-transform kernel; N = 2048, 4096: radix-16 kernel; any other N <= 8192: one CTA per transform.
template <int DEMOD>
int ofdm_fft(const char* name, const float* d_x, float* d_out, int64_t rows, int32_t nsym, int32_t n, const int32_t* d_cp,
             const int32_t* d_off, int32_t len, int32_t l_min, int32_t shift, cudaStream_t stream) {
    if (rows == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_x && d_out && d_cp && d_off && rows >= 0 && nsym > 0 && n > 0 && n <= 8192,
                 "%s: bad arguments (need 1 <= fft_size <= 8192, num_symbols >= 1)", name);
    const float2* x = (const float2*)d_x;
    float2* out = (float2*)d_out;
    int rc = SB_OK;
    if (n <= kSmallFftMax) {
        rc = launch_fft_small<DEMOD>(x, out, n, nsym, d_cp, d_off, len, l_min, rows, shift, stream);
    } else if (n == 4096 || n == 2048) {
        rc = launch_fft_pow2<DEMOD>(n, x, out, nsym, d_cp, d_off, len, l_min, rows, shift, stream);
    } else {
        FftPlan plan;
        SB_CHECK_ARG(make_plan(n, &plan) == 0, "%s: fft_size has too many factors", name);
        const int threads = std::min(256, std::max(32, (n / 2 + 31) / 32 * 32));
        const size_t smem = sizeof(float2) * 3 * (size_t)n;
        int dev = 0, optin = 0;
        SB_CUDA(cudaGetDevice(&dev));
        SB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
        if (smem > (size_t)optin) {
            sb_set_error("%s: fft_size %d needs %zu bytes of shared memory per CTA, the device offers %d", name, n, smem, optin);
            return SB_EUNSUPPORTED;
        }
        auto kern = ofdm_fft_kernel<DEMOD>;
        SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<sb_grid(rows * nsym, 1, 8), threads, smem, stream>>>(x, out, plan, nsym, d_cp, d_off, len, l_min, rows, shift);
    }
    if (rc) return rc;
    SB_LAUNCH_CHECK();
    return SB_OK;
}

}  // namespace

extern "C" int sb_ofdm_modulate(const float* d_x, float* d_out, int64_t rows, int32_t num_symbols, int32_t fft_size,
                                const int32_t* d_cp, const int32_t* d_out_off, int32_t out_len, int32_t shift, void* stream) {
    return ofdm_fft<0>("sb_ofdm_modulate", d_x, d_out, rows, num_symbols, fft_size, d_cp, d_out_off, out_len, 0, shift,
                       (cudaStream_t)stream);
}

extern "C" int sb_ofdm_demodulate(const float* d_x, float* d_out, int64_t rows, int32_t num_symbols, int32_t fft_size,
                                  const int32_t* d_cp, const int32_t* d_in_off, int32_t in_len, int32_t l_min,
                                  int32_t shift, void* stream) {
    return ofdm_fft<1>("sb_ofdm_demodulate", d_x, d_out, rows, num_symbols, fft_size, d_cp, d_in_off, in_len, l_min, shift,
                       (cudaStream_t)stream);
}

extern "C" int sb_gather_rows(const float* d_in, const int32_t* d_idx, float* d_out, int64_t batch, int32_t rows,
                              int32_t cols_out, int32_t in_rows, int32_t cols_in, int32_t words, void* stream) {
    // empty batch, or no columns to gather (the data REs of an all-pilot grid): nothing to do, pointers may be null
    if (batch == 0 || cols_out == 0) return SB_OK;
    SB_CHECK_ARG(d_in && d_idx && d_out && batch >= 0 && rows > 0 && cols_out > 0 && cols_in > 0 &&
                     (in_rows == 1 || in_rows == rows) && (words == 1 || words == 2 || words == 4),
                 "sb_gather_rows: bad arguments");
    long long total = batch * rows * (long long)cols_out;
    if (total == 0) return SB_OK;
    const RowLaunch rl = row_launch(batch * rows, cols_out);
    if (words == 1)
        gather_rows_kernel<1><<<rl.grid, rl.block, 0, (cudaStream_t)stream>>>(d_in, d_idx, d_out, batch, rows, cols_out, in_rows, cols_in);
    else if (words == 4)
        gather_rows_kernel<4><<<rl.grid, rl.block, 0, (cudaStream_t)stream>>>(d_in, d_idx, d_out, batch, rows, cols_out, in_rows, cols_in);
    else
        gather_rows_kernel<2><<<rl.grid, rl.block, 0, (cudaStream_t)stream>>>(d_in, d_idx, d_out, batch, rows, cols_out, in_rows, cols_in);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_rg_map(const float* d_x, const float* d_pilots, const int32_t* d_map, float* d_out, int64_t batch,
                         int32_t num_streams, int32_t grid_size, int32_t num_data, int32_t num_pilots, void* stream) {
    if (batch == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    // d_x is never read without data REs (an all-pilot grid), nor d_pilots without pilots: either may then be null
    SB_CHECK_ARG((d_x || num_data == 0) && (d_pilots || num_pilots == 0) && d_map && d_out && batch >= 0 &&
                     num_streams > 0 && grid_size > 0 && num_data >= 0 && num_pilots >= 0, "sb_rg_map: bad arguments");
    long long total = batch * num_streams * (long long)grid_size;
    if (total == 0) return SB_OK;
    const RowLaunch rl = row_launch(batch * num_streams, grid_size);
    rg_map_kernel<<<rl.grid, rl.block, 0, (cudaStream_t)stream>>>((const float2*)d_x, (const float2*)d_pilots, d_map,
                                                                         (float2*)d_out, batch, num_streams, grid_size,
                                                                         num_data, num_pilots);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_ls_at_pilots(const float* d_y, const int32_t* d_pilot_ind, const float* d_pilots, const float* d_no,
                               int64_t no_inner, float* d_h, float* d_err, int64_t batch, int32_t num_streams,
                               int32_t num_pilots, int32_t grid_size, void* stream) {
    if (batch == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_y && d_pilot_ind && d_pilots && d_no && d_h && d_err && batch >= 0 && num_streams > 0 &&
                     num_pilots > 0 && grid_size > 0 && no_inner >= 1, "sb_ls_at_pilots: bad arguments");
    long long total = batch * num_streams * (long long)num_pilots;
    if (total == 0) return SB_OK;
    const RowLaunch rl = row_launch(batch * num_streams, num_pilots);
    ls_at_pilots_kernel<<<rl.grid, rl.block, 0, (cudaStream_t)stream>>>(
        (const float2*)d_y, d_pilot_ind, (const float2*)d_pilots, d_no, no_inner, (float2*)d_h, d_err, batch, num_streams,
        num_pilots, grid_size);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_interp_lin(const float* d_h, const int32_t* d_fx0, const int32_t* d_fx1, const int32_t* d_fy0,
                             const int32_t* d_fy1, const int32_t* d_ty0, const int32_t* d_ty1, const int32_t* d_npil,
                             int32_t time_avg, float* d_out, int64_t batch, int32_t num_streams, int32_t num_symbols,
                             int32_t num_subcarriers, int32_t num_pilots, int32_t words, void* stream) {
    if (batch == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_h && d_fx0 && d_fx1 && d_fy0 && d_fy1 && d_ty0 && d_ty1 && d_npil && d_out && batch >= 0 &&
                     (words == 1 || words == 2), "sb_interp_lin: bad arguments (words: 1 = real, 2 = complex)");
    const long long rows = batch * num_streams;
    if (rows == 0 || num_symbols * num_subcarriers == 0) return SB_OK;
    const int grid = sb_grid(rows, 1, 16);
    const int threads = std::min(256, std::max(32, (num_subcarriers + 31) / 32 * 32));
    if (words == 2)
        interp_lin_kernel<float2><<<grid, threads, 0, (cudaStream_t)stream>>>(
            (const float2*)d_h, d_fx0, d_fx1, d_fy0, d_fy1, d_ty0, d_ty1, d_npil, time_avg, (float2*)d_out, batch,
            num_streams, num_symbols, num_subcarriers, num_pilots);
    else
        interp_lin_kernel<float><<<grid, threads, 0, (cudaStream_t)stream>>>(
            d_h, d_fx0, d_fx1, d_fy0, d_fy1, d_ty0, d_ty1, d_npil, time_avg, d_out, batch, num_streams, num_symbols,
            num_subcarriers, num_pilots);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

// ---- PUSCH (nr/pusch_precoder.py, nr/pusch_channel_estimation.py) ---------------------------------------------------
namespace {
// y[b, t, p, re] = sum_l W[t, p, l] x[b, t, l, re]: codebook precoding of the layer grids onto the antenna ports
__global__ void pusch_precode_kernel(const float2* __restrict__ x, const float2* __restrict__ w, float2* __restrict__ y,
                                     long long total, int num_tx, int L, int P, long long re) {
    // grid-stride: sb_grid() caps the grid at 16 CTAs per SM
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        long long r = i % re;
        long long bp = i / re;
        int p = (int)(bp % P);
        long long bt = bp / P;
        int t = (int)(bt % num_tx);
        const float2* wp = w + ((size_t)t * P + p) * L;
        const float2* xp = x + (size_t)bt * L * re + r;
        float2 acc = make_float2(0.f, 0.f);
        for (int l = 0; l < L; ++l) {
            float2 a = wp[l], b = __ldg(xp + (size_t)l * re);
            acc.x += a.x * b.x - a.y * b.y;
            acc.y += a.x * b.y + a.y * b.x;
        }
        y[i] = acc;
    }
}

// CDM de-spreading of LS estimates at the DMRS REs, in place. Row = one (batch', tx stream): P = num_dmrs_syms * pps
// pilots ordered symbol-major. One thread owns one frequency group of n = 2 * num_cdm_groups_without_data consecutive
// pilots on one DMRS symbol (single-symbol DMRS) or on a pair of adjacent DMRS symbols (double-symbol DMRS):
//   time:  v_k = (h[s0][k] + h[s1][k]) / 2                    (dmrs_length == 2, pusch_channel_estimation.py:138-149)
//   freq:  avg = (sum_k v_k) / 2;  h[k] = |v_k| > 0 ? avg : 0 (:153-165)
__global__ void pusch_ls_combine_kernel(float2* __restrict__ h, long long rows, int P, int pps, int dmrs_length, int n) {
    const int groups = pps / n;
    const int units = (P / pps) / dmrs_length;              // symbol pairs (or single symbols) per row
    const long long total = rows * units * groups;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        int g = (int)(i % groups);
        long long ru = i / groups;
        int u = (int)(ru % units);
        long long row = ru / units;
        float2* p0 = h + (size_t)row * P + (size_t)u * dmrs_length * pps + (size_t)g * n;
        float2* p1 = p0 + pps;
        float2 sum = make_float2(0.f, 0.f);
        for (int k = 0; k < n; ++k) {
            float2 v = p0[k];
            if (dmrs_length == 2) {
                float2 b = p1[k];
                v = make_float2((v.x + b.x) * 0.5f, (v.y + b.y) * 0.5f);
                p0[k] = v;
            }
            sum.x += v.x;
            sum.y += v.y;
        }
        float2 avg = make_float2(sum.x * 0.5f, sum.y * 0.5f);
        for (int k = 0; k < n; ++k) {
            float2 v = p0[k];
            float2 o = (v.x != 0.f || v.y != 0.f) ? avg : make_float2(0.f, 0.f);
            p0[k] = o;
            if (dmrs_length == 2) p1[k] = o;
        }
    }
}

__global__ void scale_real_kernel(float* __restrict__ x, long long n, float s) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        x[i] *= s;
}
}  // namespace

extern "C" int sb_pusch_precode(const float* d_x, const float* d_w, float* d_y, int64_t batch, int32_t num_tx,
                                int32_t num_layers, int32_t num_ports, int64_t num_re, void* stream) {
    if (batch == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_x && d_w && d_y && batch >= 0 && num_tx > 0 && num_layers > 0 && num_ports > 0 && num_re > 0,
                 "sb_pusch_precode: bad arguments");
    long long total = batch * num_tx * (long long)num_ports * num_re;
    if (total == 0) return SB_OK;
    pusch_precode_kernel<<<sb_grid(total, 256, 16), 256, 0, (cudaStream_t)stream>>>(
        (const float2*)d_x, (const float2*)d_w, (float2*)d_y, total, num_tx, num_layers, num_ports, num_re);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_pusch_ls_combine(float* d_h, float* d_err_var, int64_t rows, int32_t num_pilots,
                                   int32_t pilots_per_dmrs_symbol, int32_t dmrs_length, int32_t group_size, void* stream) {
    if (rows == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_h && d_err_var && rows >= 0 && num_pilots > 0 && pilots_per_dmrs_symbol > 0 &&
                     num_pilots % pilots_per_dmrs_symbol == 0 && (dmrs_length == 1 || dmrs_length == 2) &&
                     (num_pilots / pilots_per_dmrs_symbol) % dmrs_length == 0 && group_size > 0 &&
                     pilots_per_dmrs_symbol % group_size == 0, "sb_pusch_ls_combine: bad arguments");
    if (rows == 0) return SB_OK;
    long long units = (long long)rows * (num_pilots / pilots_per_dmrs_symbol / dmrs_length) *
                      (pilots_per_dmrs_symbol / group_size);
    pusch_ls_combine_kernel<<<sb_grid(units, 256, 16), 256, 0, (cudaStream_t)stream>>>(
        (float2*)d_h, rows, num_pilots, pilots_per_dmrs_symbol, dmrs_length, group_size);
    SB_LAUNCH_CHECK();
    long long n = (long long)rows * num_pilots;
    scale_real_kernel<<<sb_grid(n, 256, 16), 256, 0, (cudaStream_t)stream>>>(d_err_var, n, dmrs_length == 2 ? 0.25f : 0.5f);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

using sb_dense::scratch_threads;
using sb_dense::kScratchSmemCap;

extern "C" int sb_lmmse_equalize(const float* d_y, const float* d_h, const float* d_s, float* d_x_hat, float* d_no_eff,
                                 int64_t num, int32_t M, int32_t K, void* stream) {
    if (num == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_y && d_h && d_s && d_x_hat && d_no_eff && num >= 0 && M >= 1 && K >= 1 && K <= 16 && K <= M,
                 "sb_lmmse_equalize: bad arguments (need 1 <= K <= 16, K <= M)");
    size_t smem = 0;
    const size_t per_thread = sizeof(float2) * LmmseScratch::elems(M, K);
    int threads = scratch_threads(per_thread, kScratchSmemCap, &smem);
    if (!threads) {
        sb_set_error("sb_lmmse_equalize: M = %d, K = %d needs %zu bytes of shared-memory scratch per vector, the limit is %zu",
                     M, K, per_thread, kScratchSmemCap);
        return SB_EUNSUPPORTED;
    }
    SB_CUDA(cudaFuncSetAttribute(lmmse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    lmmse_kernel<<<sb_grid(num, threads, 16), threads, smem, (cudaStream_t)stream>>>(
        (const float2*)d_y, (const float2*)d_h, (const float2*)d_s, (float2*)d_x_hat, d_no_eff, num, M, K);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_mimo_linalg(int32_t mode, const float* d_y, const float* d_h, const float* d_s, float* d_out0, void* d_out1,
                              int64_t num, int32_t M, int32_t K, void* stream) {
    if (num == 0) return SB_OK;
    SB_CHECK_ARG(mode >= 0 && mode <= 6 && num > 0 && M >= 1 && d_out0, "sb_mimo_linalg: bad arguments");
    SB_CHECK_ARG(mode == 0 ? (d_s != nullptr) : (d_h && K >= 1 && K <= M), "sb_mimo_linalg: missing input / need 1 <= K <= M");
    SB_CHECK_ARG(mode != 1 || (d_y && d_s && d_out1), "sb_mimo_linalg: whiten_channel needs y, h, s and two outputs");
    SB_CHECK_ARG((mode != 3 && mode != 4 && mode != 5) || (d_y && d_s && d_out1),
                 "sb_mimo_linalg: the equaliser needs y, h, s and two outputs");
    if (mode == 0) K = M;
    int dev = 0, optin = 0;
    SB_CUDA(cudaGetDevice(&dev));
    SB_CUDA(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
    size_t smem = 0;
    const size_t per_thread = sizeof(float2) * ((size_t)M * M + 2 * (size_t)M * K);
    int threads = scratch_threads(per_thread, (size_t)optin, &smem);
    if (!threads) {
        sb_set_error("sb_mimo_linalg: M = %d, K = %d needs %zu bytes of shared-memory scratch per matrix, the device offers %d",
                     M, K, per_thread, optin);
        return SB_EUNSUPPORTED;
    }
    SB_CUDA(cudaFuncSetAttribute(mimo_linalg_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    mimo_linalg_kernel<<<sb_grid(num, threads, 16), threads, smem, (cudaStream_t)stream>>>(
        mode, (const float2*)d_y, (const float2*)d_h, (const float2*)d_s, (float2*)d_out0, d_out1, num, M, K);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

// Launches the equaliser eq (EQ_*) over the OFDM problem p after the caller's argument checks (who names the caller in
// the scratch-limit message)
static int ofdm_linear(const char* who, int eq, const OfdmEqParams& p, long long total_re, cudaStream_t stream) {
    const int M = p.ANT, K = p.K;
    if (p.KU == 0 && K <= 4 && (eq != EQ_LMMSE_NO_WHITEN || M >= K + 2)) {   // diagonal S: register kernel
        const int rc = sb_dispatch<1, 4>(K, [&](auto KC) {
            const int grid = sb_grid(total_re, 128, 16);
            if (eq == EQ_ZF) ofdm_linear_diag_kernel<EQ_ZF, KC><<<grid, 128, 0, stream>>>(p);
            else if (eq == EQ_MF) ofdm_linear_diag_kernel<EQ_MF, KC><<<grid, 128, 0, stream>>>(p);
            else ofdm_linear_diag_kernel<EQ_LMMSE, KC><<<grid, 128, 0, stream>>>(p);
            return SB_OK;
        });
        if (rc) return rc;
        SB_LAUNCH_CHECK();
        return SB_OK;
    }
    size_t smem = 0;
    const size_t per_thread = sizeof(float2) * LmmseScratch::elems(M, K);
    int threads = scratch_threads(per_thread, kScratchSmemCap, &smem);
    if (!threads) {
        sb_set_error("%s: %d receive antennas, %d streams need %zu bytes of shared-memory scratch per resource "
                     "element, the limit is %zu", who, M, K, per_thread, kScratchSmemCap);
        return SB_EUNSUPPORTED;
    }
    const int rc = sb_dispatch<0, 3>(eq, [&](auto E) {
        SB_CUDA(cudaFuncSetAttribute(ofdm_linear_kernel<E>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        ofdm_linear_kernel<E><<<sb_grid(total_re, threads, 16), threads, smem, stream>>>(p);
        return SB_OK;
    });
    if (rc) return rc;
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_ofdm_lmmse(const float* d_y, const float* d_h_hat, const float* d_err_var, const int64_t* h_ev_stride,
                             const float* d_no, const int64_t* h_no_stride, const int32_t* d_desired,
                             const int32_t* d_undesired, const int32_t* d_out_stream, const int32_t* d_data_pos,
                             float* d_x_hat, float* d_no_eff, int64_t batch, int32_t num_rx, int32_t num_rx_ant,
                             int32_t num_tx_streams, int32_t num_symbols, int32_t num_subcarriers,
                             int32_t streams_per_rx, int32_t interferers_per_rx, int32_t num_data, void* stream) {
    if (batch == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_y && d_h_hat && d_err_var && h_ev_stride && d_no && h_no_stride && d_desired && d_out_stream &&
                     d_data_pos && d_x_hat && d_no_eff && batch >= 0 && streams_per_rx >= 1 && streams_per_rx <= 16 &&
                     streams_per_rx <= num_rx_ant && (interferers_per_rx == 0 || d_undesired),
                 "sb_ofdm_lmmse: bad arguments (need 1 <= streams_per_rx <= min(16, num_rx_ant))");
    const sb_dense::MimoProblem pb = sb_dense::ofdm_problem(d_y, d_h_hat, d_err_var, h_ev_stride, d_no, h_no_stride,
                                                            d_desired, d_undesired, d_out_stream, d_data_pos, batch,
                                                            num_rx, num_rx_ant, num_tx_streams, num_symbols,
                                                            num_subcarriers, streams_per_rx, interferers_per_rx,
                                                            num_data);
    OfdmEqParams p = pb.ofdm;
    p.xh = (float2*)d_x_hat; p.ne = d_no_eff;
    return ofdm_linear("sb_ofdm_lmmse", EQ_LMMSE, p, pb.P, (cudaStream_t)stream);
}

extern "C" int sb_ofdm_equalize(int32_t equalizer, const float* d_y, const float* d_h_hat, const float* d_err_var,
                                const int64_t* h_ev_stride, const float* d_no, const int64_t* h_no_stride,
                                const int32_t* d_desired, const int32_t* d_undesired, const int32_t* d_out_stream,
                                const int32_t* d_data_pos, float* d_x_hat, float* d_no_eff, int64_t batch,
                                int32_t num_rx, int32_t num_rx_ant, int32_t num_tx_streams, int32_t num_symbols,
                                int32_t num_subcarriers, int32_t streams_per_rx, int32_t interferers_per_rx,
                                int32_t num_data, void* stream) {
    SB_CHECK_ARG(equalizer >= EQ_LMMSE && equalizer <= EQ_MF, "sb_ofdm_equalize: equalizer must be 0 (lmmse), "
                 "1 (lmmse without whitening), 2 (zf) or 3 (mf)");
    SB_CHECK_ARG(batch >= 0 && num_rx >= 1 && num_rx_ant >= 1 && num_tx_streams >= 1 && num_symbols >= 1 &&
                     num_subcarriers >= 1 && interferers_per_rx >= 0 && num_data >= 0,
                 "sb_ofdm_equalize: bad sizes");
    if (streams_per_rx < 1 || streams_per_rx > 16 || streams_per_rx > num_rx_ant) {
        sb_set_error("sb_ofdm_equalize: %d streams per receiver with %d receive antennas; supported are "
                     "1 <= streams_per_rx <= min(16, num_rx_ant)", streams_per_rx, num_rx_ant);
        return SB_EUNSUPPORTED;
    }
    if (batch == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_y && d_h_hat && d_err_var && h_ev_stride && d_no && h_no_stride && d_desired && d_out_stream &&
                     d_data_pos && d_x_hat && d_no_eff && (interferers_per_rx == 0 || d_undesired),
                 "sb_ofdm_equalize: bad pointers");
    const sb_dense::MimoProblem pb = sb_dense::ofdm_problem(d_y, d_h_hat, d_err_var, h_ev_stride, d_no, h_no_stride,
                                                            d_desired, d_undesired, d_out_stream, d_data_pos, batch,
                                                            num_rx, num_rx_ant, num_tx_streams, num_symbols,
                                                            num_subcarriers, streams_per_rx, interferers_per_rx,
                                                            num_data);
    OfdmEqParams p = pb.ofdm;
    p.xh = (float2*)d_x_hat; p.ne = d_no_eff;
    return ofdm_linear("sb_ofdm_equalize", equalizer, p, pb.P, (cudaStream_t)stream);
}
