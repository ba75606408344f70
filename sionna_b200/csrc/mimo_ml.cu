// mimo_ml.cu -- maximum-likelihood MIMO detection for sm_90a. Replaces (paths under /root/reference/src/sionna/phy/):
//   sb_mimo_ml    MaximumLikelihoodDetector.call   mimo/detection.py:473-537 (+ whiten_channel mimo/utils.py:292-357,
//                 SymbolLogits2LLRs.call mapping.py:927-967)
//   sb_ofdm_ml    OFDM MaximumLikelihoodDetector(WithPrior)  ofdm/detection.py:448-738: OFDMEqualizer's per-resource-element
//                 covariance S = H_u H_u^H + diag(no) + diag(sum err_var) (dense_mimo.cuh) instead of the [.., M, M] tensor
// The reference enumerates all |C|^K candidate vectors and materialises H x for each ([.., |C|^K, M] complex per problem);
// here nothing per candidate leaves the chip.
//
// Two launches per call:
//   1. ml_prologue_kernel, one thread per problem (scratch in shared memory, as the LMMSE kernels): the detectors'
//      shared loader (load_whitened, dense_mimo.cuh) gives y_w and H_w, then modified Gram-Schmidt on [H_w | y_w]:
//        H_w = Q R (R upper trapezoidal K x K, rows >= min(M, K) zero),  yq = Q^H y_w,  c0 = ||y_w - Q yq||^2,
//      so that ||y_w - H_w x||^2 = c0 + ||yq - R x||^2 for every x. The record (R, yq, c0: 8 (K^2 + K + 1) bytes) and the
//      K output positions go to the caller's workspace in HBM (sb_ml_workspace_bytes): the prologue needs
//      8 (M^2 + M K + M) bytes of scratch per problem (2.7 KB for M = 16, K = 4), which would cap the enumeration's
//      occupancy if both ran in one kernel.
//   2. ml_enum_kernel: candidates enumerated with stream 0 varying fastest. Row r of yq - R x depends on x_r..x_{K-1}
//      only, so the rows >= 1 and the stream-0 row's offset b0 = yq_0 - sum_{j>0} R_0j x_j are recomputed once per inner
//      loop over x_0 (O(K) per |C| candidates), and a candidate costs 2 FMAs for yq_0 - R_00 x_0, 2 for |.|^2 and the
//      accumulator updates. Metric d(x) = c0 + ||yq - R x||^2 - sum_k prior[k, x_k].
//      Accumulators per (stream k, point c): pass 1 m_kc = min d (maxlog: logit = -m_kc). app adds pass 2, which sums
//      exp(m_kc - d) with each accumulator's own offset (every term <= 1, the minimiser contributes exactly 1, so no
//      accumulator the reference keeps finite underflows): stream 0 gets one exp per candidate; for streams k >= 1 the
//      inner loop is summed once against its own minimum l, T = sum_c exp(l - d_c), and added as exp(m_kc - l) T.
//      logit = -m_kc + log(sum).
//      Work split, chosen at launch from |C|^(K-1) and K |C|:
//        G = 32  a warp per problem, lanes take contiguous ranges of the outer index (x_1..x_{K-1}), lane-private
//                accumulators in shared memory combined at the end (large candidate sets: 4 x 16-QAM, 8 x QPSK);
//        G = 1   a thread per problem (small candidate sets: 2 x 16-QAM, 2 x QPSK, and large constellations whose
//                K |C| accumulators would not fit a warp's lane-private copies).
//      The finish step writes symbol logits, argmax indices (first on ties) or bit LLRs / hard bits (SymbolLogits2LLRs:
//      logsumexp or max over each label set, mapping.py:927-967) straight into the caller's output layout.
#include "sb_common.h"
#include "dense_mimo.cuh"

namespace {

using sb_dense::Scratch;
using sb_dense::MimoProblem;
using sb_dense::qr_record_size;
using sb_dense::kScratchSmemCap;

constexpr int kMlMaxK = 8;
constexpr long long kMlMaxCandidates = 65536;
constexpr int kMlMaxPoints = 1024;
// One thread per problem (load_whitened, then qr_record in the identity order); output positions to oidx [P, K]
__global__ void ml_prologue_kernel(const MimoProblem pb, float2* __restrict__ recs, long long* __restrict__ oidx) {
    extern __shared__ float2 smem[];
    const int T = blockDim.x, t = threadIdx.x, M = pb.M, K = pb.K;
    const Scratch S{smem, T, t}, H{smem + (size_t)M * M * T, T, t}, Y{smem + (size_t)(M * M + M * K) * T, T, t};
    for (long long i = (long long)blockIdx.x * T + t; i < pb.P; i += (long long)gridDim.x * T) {
        if (!sb_dense::load_whitened(pb, i, S, H, Y, oidx + i * K)) continue;
        sb_dense::qr_record(Y, H, M, K, [](int j) { return j; }, recs + i * qr_record_size(K));
    }
}

struct MlParams {
    const float2* rec; const long long* oidx; const float2* points; const float* prior;
    void* out;
    long long P;
    int NP, bits, maxlog, symbol, hard;
};

// accumulator a = k * NP + c of one problem: p[a * stride + idx]
struct Acc {
    float* p;
    int stride, idx;
    __device__ __forceinline__ float& operator()(int a) const { return p[a * stride + idx]; }
};

// d = P1 + |b0 - R00 p|^2 - pr (every metric of the problem goes through this one expression, so both app passes see
// bit-identical values)
__device__ __forceinline__ float ml_leaf(float2 b0, float r00, float2 pt, float p1, float pr) {
    const float tx = fmaf(-r00, pt.x, b0.x), ty = fmaf(-r00, pt.y, b0.y);
    return fmaf(tx, tx, fmaf(ty, ty, p1)) - pr;
}

// One pass over the outer indices [o0, o1) of one problem. PASS 1: priv = min d; PASS 2: priv += exp(mins - d).
template <int K, int PASS>
__device__ __forceinline__ void ml_pass(const float2 (&R)[K][K], const float2 (&yq)[K], const float2* __restrict__ spts,
                                        int NP, int lg, const Acc& sprior, bool has_prior, const Acc& priv,
                                        const Acc& mins, long long o0, long long o1) {
    if (o0 >= o1) return;
    int x[K];
    x[0] = 0;
#pragma unroll
    for (int j = 1; j < K; ++j) x[j] = (int)((o0 >> (lg * (j - 1))) & (NP - 1));
    float P[K + 1];
    P[K] = 0.f;
    float2 b0 = yq[0];
    int h = K - 1;
    for (long long o = o0; o < o1; ++o) {
        // rows h .. 1 and the stream-0 offset b0 for the current outer digits
#pragma unroll
        for (int r = K - 1; r >= 1; --r) {
            if (r <= h) {
                float2 b = yq[r];
#pragma unroll
                for (int j = r; j < K; ++j) {
                    const float2 pj = spts[x[j]];
                    b.x = fmaf(-R[r][j].x, pj.x, fmaf(R[r][j].y, pj.y, b.x));
                    b.y = fmaf(-R[r][j].x, pj.y, fmaf(-R[r][j].y, pj.x, b.y));
                }
                float pr = has_prior ? sprior(r * NP + x[r]) : 0.f;
                P[r] = fmaf(b.x, b.x, fmaf(b.y, b.y, P[r + 1])) - pr;
            }
        }
        b0 = yq[0];
#pragma unroll
        for (int j = 1; j < K; ++j) {
            const float2 pj = spts[x[j]];
            b0.x = fmaf(-R[0][j].x, pj.x, fmaf(R[0][j].y, pj.y, b0.x));
            b0.y = fmaf(-R[0][j].x, pj.y, fmaf(-R[0][j].y, pj.x, b0.y));
        }
        const float p1 = P[1], r00 = R[0][0].x;
        float lmin = INFINITY;
        if (PASS == 1) {
            for (int c = 0; c < NP; ++c) {
                const float d = ml_leaf(b0, r00, spts[c], p1, has_prior ? sprior(c) : 0.f);
                priv(c) = fminf(priv(c), d);
                lmin = fminf(lmin, d);
            }
#pragma unroll
            for (int k = 1; k < K; ++k) priv(k * NP + x[k]) = fminf(priv(k * NP + x[k]), lmin);
        } else {
            for (int c = 0; c < NP; ++c) lmin = fminf(lmin, ml_leaf(b0, r00, spts[c], p1, has_prior ? sprior(c) : 0.f));
            if (lmin < INFINITY) {
                float tsum = 0.f;
                for (int c = 0; c < NP; ++c) {
                    const float d = ml_leaf(b0, r00, spts[c], p1, has_prior ? sprior(c) : 0.f);
                    if (d < INFINITY) {
                        priv(c) += expf(mins(c) - d);
                        tsum += expf(lmin - d);
                    }
                }
#pragma unroll
                for (int k = 1; k < K; ++k) priv(k * NP + x[k]) += expf(mins(k * NP + x[k]) - lmin) * tsum;
            }
        }
        // next outer index: digit 1 is the least significant; h = highest digit that changed
        h = 1;
        if constexpr (K > 1) {
            ++x[1];
#pragma unroll
            for (int j = 1; j + 1 < K; ++j)
                if (x[j] == NP) { x[j] = 0; ++x[j + 1]; h = j + 1; }
        }
    }
}

// G lanes per problem (1 or 32). Shared memory: points [NP] float2, then per group
//   G = 1:  per thread (interleaved over the CTA's threads) A [K NP] (pass 1, then the mins / logits), B [K NP]
//           (pass-2 sums), prior [K NP] if given
//   G = 32: per warp lane-private [K NP][32], mins / logits [K NP], prior [K NP] if given
template <int K, int G>
__global__ void __launch_bounds__(256) ml_enum_kernel(const MlParams q) {
    extern __shared__ float2 smem[];
    const int NP = q.NP, AK = K * NP, T = blockDim.x, t = threadIdx.x;
    const int lane = G == 1 ? 0 : (t & 31);
    const bool has_prior = q.prior != nullptr;
    float2* spts = smem;
    for (int i = t; i < NP; i += T) spts[i] = q.points[i];
    __syncthreads();
    float* base = reinterpret_cast<float*>(smem + NP);
    const int lg = 31 - __clz(NP);
    Acc priv1, priv2, mins, sprior;
    long long gid, gstride;
    if (G == 1) {
        priv1 = Acc{base, T, t};
        mins = priv1;
        priv2 = Acc{base + (size_t)AK * T, T, t};
        sprior = Acc{base + (size_t)2 * AK * T, T, t};
        gid = (long long)blockIdx.x * T + t;
        gstride = (long long)gridDim.x * T;
    } else {
        const int w = t >> 5, per_warp = AK * (33 + (has_prior ? 1 : 0));
        float* wb = base + (size_t)w * per_warp;
        priv1 = Acc{wb, 32, lane};
        priv2 = priv1;
        mins = Acc{wb + 32 * AK, 1, 0};
        sprior = Acc{wb + 33 * AK, 1, 0};
        gid = (long long)blockIdx.x * (T >> 5) + w;
        gstride = (long long)gridDim.x * (T >> 5);
    }
    long long NO = 1;
    for (int k = 1; k < K; ++k) NO *= NP;
    for (long long p = gid; p < q.P; p += gstride) {            // uniform over the group
        const long long* oi = q.oidx + p * K;
        bool any = false;
#pragma unroll
        for (int k = 0; k < K; ++k) any = any || oi[k] >= 0;
        if (!any) continue;
        const float2* rec = q.rec + p * qr_record_size(K);
        float2 R[K][K], yq[K];
#pragma unroll
        for (int r = 0; r < K; ++r) {
#pragma unroll
            for (int j = 0; j < K; ++j) R[r][j] = j >= r ? rec[r * K + j] : make_float2(0.f, 0.f);
            yq[r] = rec[K * K + r];
        }
        const float c0 = rec[K * K + K].x;
        if (G == 32) __syncwarp();                              // previous problem's finish step has read mins
        for (int a = lane; a < AK; a += G) {
            if (has_prior) {
                const long long o = oi[a / NP];
                sprior(a) = o >= 0 ? q.prior[o * NP + a % NP] : 0.f;
            }
        }
        for (int a = 0; a < AK; ++a) priv1(a) = INFINITY;
        if (G == 32) __syncwarp();
        const long long o0 = G == 1 ? 0 : NO / G * lane, o1 = G == 1 ? NO : NO / G * (lane + 1);
        ml_pass<K, 1>(R, yq, spts, NP, lg, sprior, has_prior, priv1, mins, o0, o1);
        if (G == 32) {                                          // mins over the lanes (rotated: conflict-free)
            __syncwarp();
            for (int a = lane; a < AK; a += 32) {
                float m = INFINITY;
                for (int l = 0; l < 32; ++l) m = fminf(m, priv1.p[a * 32 + ((l + lane) & 31)]);
                mins(a) = m;
            }
            __syncwarp();
        }
        if (!q.maxlog) {
            for (int a = 0; a < AK; ++a) priv2(a) = 0.f;
            ml_pass<K, 2>(R, yq, spts, NP, lg, sprior, has_prior, priv2, mins, o0, o1);
            if (G == 32) __syncwarp();
            for (int a = lane; a < AK; a += G) {
                float sum;
                if (G == 1) {
                    sum = priv2(a);
                } else {
                    sum = 0.f;
                    for (int l = 0; l < 32; ++l) sum += priv2.p[a * 32 + ((l + lane) & 31)];
                }
                const float m = mins(a);
                mins(a) = m < INFINITY ? -(m + c0) + logf(sum) : -INFINITY;
            }
        } else {
            for (int a = lane; a < AK; a += G) {
                const float m = mins(a);
                mins(a) = m < INFINITY ? -(m + c0) : -INFINITY;
            }
        }
        if (G == 32) __syncwarp();
        // finish: mins now holds the logits [K, NP]
        if (q.symbol && q.hard) {
            for (int k = lane; k < K; k += G) {
                if (oi[k] < 0) continue;
                int best = 0;
                float bv = mins(k * NP);
                for (int c = 1; c < NP; ++c) {
                    const float v = mins(k * NP + c);
                    if (v > bv) { bv = v; best = c; }
                }
                reinterpret_cast<int*>(q.out)[oi[k]] = best;
            }
        } else if (q.symbol) {
            for (int a = lane; a < AK; a += G) {
                const long long o = oi[a / NP];
                if (o >= 0) reinterpret_cast<float*>(q.out)[o * NP + a % NP] = mins(a);
            }
        } else {
            const int m = q.bits;
            for (int it = lane; it < K * m; it += G) {
                const int k = it / m, i = it % m;
                const long long o = oi[k];
                if (o < 0) continue;
                float mx0 = -INFINITY, mx1 = -INFINITY;
                for (int c = 0; c < NP; ++c) {
                    const float v = mins(k * NP + c);
                    if ((c >> (m - 1 - i)) & 1) mx1 = fmaxf(mx1, v); else mx0 = fmaxf(mx0, v);
                }
                float llr;
                if (q.maxlog) {
                    llr = mx1 - mx0;
                } else {                                        // tf.reduce_logsumexp: max replaced by 0 if not finite
                    const float s0 = isfinite(mx0) ? mx0 : 0.f, s1 = isfinite(mx1) ? mx1 : 0.f;
                    float e0 = 0.f, e1 = 0.f;
                    for (int c = 0; c < NP; ++c) {
                        const float v = mins(k * NP + c);
                        if ((c >> (m - 1 - i)) & 1) e1 += expf(v - s1); else e0 += expf(v - s0);
                    }
                    llr = (logf(e1) + s1) - (logf(e0) + s0);
                }
                reinterpret_cast<float*>(q.out)[o * m + i] = q.hard ? (llr > 0.f ? 1.f : 0.f) : llr;
            }
        }
    }
}

// Malformed arguments (no streams, a constellation size that is not a power of two >= 2, flags outside {0, 1}) are
// SB_EINVAL; well-formed configurations beyond the kernels' limits are SB_EUNSUPPORTED.
int ml_check(const char* who, int K, int num_points, int method, int output, int hard_out) {
    if (K < 1 || num_points < 2 || (num_points & (num_points - 1)) || method < 0 || method > 1 || output < 0 ||
        output > 1 || hard_out < 0 || hard_out > 1) {
        sb_set_error("%s: bad arguments (need K >= 1 streams, a power-of-two constellation of >= 2 points, "
                     "method / output / hard_out in {0, 1})", who);
        return SB_EINVAL;
    }
    if (K > kMlMaxK) {
        sb_set_error("%s: %d streams, the limit is %d", who, K, kMlMaxK);
        return SB_EUNSUPPORTED;
    }
    if (num_points > kMlMaxPoints) {
        sb_set_error("%s: a constellation of %d points, the limit is %d", who, num_points, kMlMaxPoints);
        return SB_EUNSUPPORTED;
    }
    long long n = 1;
    for (int k = 0; k < K; ++k) n *= num_points;
    if (n > kMlMaxCandidates) {
        sb_set_error("%s: %d streams of %d points are %lld candidate vectors, the limit is %lld", who, K, num_points, n,
                     kMlMaxCandidates);
        return SB_EUNSUPPORTED;
    }
    return SB_OK;
}

// workspace: P records of qr_record_size(K) float2, then P x K output positions (int64)
size_t ml_workspace_bytes(long long P, int K) {
    return (sizeof(float2) * qr_record_size(K) + sizeof(long long) * K) * (size_t)P;
}

// Both launches on the caller's workspace of P records.
int ml_run(const char* who, const MimoProblem& pb, const float* prior, const float* points, int NP, int method,
           int output, int hard_out, void* out, void* ws, size_t ws_bytes, cudaStream_t stream) {
    const long long P = pb.P;
    const int M = pb.M, K = pb.K;
    if (!ws || ws_bytes < ml_workspace_bytes(P, K)) {
        sb_set_error("%s: the workspace needs %zu bytes (sb_ml_workspace_bytes), %zu given", who, ml_workspace_bytes(P, K),
                     ws ? ws_bytes : (size_t)0);
        return SB_ENOMEM;
    }
    size_t psmem = 0;
    const size_t p_thread = sizeof(float2) * ((size_t)M * M + (size_t)M * K + M);
    const int pthreads = sb_dense::detector_threads(who, 0, p_thread, M, K, &psmem);
    if (!pthreads) return SB_EUNSUPPORTED;
    const int AK = K * NP, bits = 31 - __builtin_clz((unsigned)NP);
    long long NO = 1;
    for (int k = 1; k < K; ++k) NO *= NP;
    const bool warp = NO >= 128 && AK <= 256;                  // enough outer indices for 32 lanes, accumulators fit
    const size_t hp = prior ? 1 : 0;
    size_t esmem = 0;
    int ethreads = 0;
    if (warp) {
        const size_t per_warp = sizeof(float) * AK * (33 + hp);
        const int warps = (int)std::min<size_t>(8, (kScratchSmemCap - NP * sizeof(float2)) / per_warp);
        ethreads = 32 * warps;
        esmem = NP * sizeof(float2) + per_warp * warps;
    } else {
        const size_t per_thread = sizeof(float) * AK * (2 + hp);
        ethreads = sb_dense::scratch_threads(per_thread, kScratchSmemCap - NP * sizeof(float2), &esmem);
        esmem += NP * sizeof(float2);
    }
    if (!ethreads || esmem > kScratchSmemCap) {
        sb_set_error("%s: %d streams of %d points need more shared memory per problem than %zu bytes", who, K, NP,
                     kScratchSmemCap);
        return SB_EUNSUPPORTED;
    }
    float2* recs = (float2*)ws;
    long long* oidx = (long long*)((char*)ws + sizeof(float2) * qr_record_size(K) * (size_t)P);
    SB_CUDA(cudaFuncSetAttribute(ml_prologue_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)psmem));
    ml_prologue_kernel<<<sb_grid(P, pthreads, 16), pthreads, psmem, stream>>>(pb, recs, oidx);
    SB_LAUNCH_CHECK();
    MlParams q{recs, oidx, (const float2*)points, prior, out, P, NP, bits, method, output, hard_out};
    return sb_dispatch<1, kMlMaxK>(K, [&](auto KC) -> int {
        constexpr int KK = decltype(KC)::value;
        if (warp) {
            SB_CUDA(cudaFuncSetAttribute(ml_enum_kernel<KK, 32>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)esmem));
            ml_enum_kernel<KK, 32><<<sb_grid(P, ethreads / 32, 64), ethreads, esmem, stream>>>(q);
        } else {
            SB_CUDA(cudaFuncSetAttribute(ml_enum_kernel<KK, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)esmem));
            ml_enum_kernel<KK, 1><<<sb_grid(P, ethreads, 16), ethreads, esmem, stream>>>(q);
        }
        SB_LAUNCH_CHECK();
        return SB_OK;
    });
}

}  // namespace

extern "C" size_t sb_ml_workspace_bytes(int64_t num_problems, int32_t K) {
    return num_problems > 0 && K >= 1 && K <= kMlMaxK ? ml_workspace_bytes(num_problems, K) : 0;
}

extern "C" int sb_mimo_ml(const float* d_y, const float* d_h, const float* d_s, const float* d_prior,
                          const float* d_points, void* d_out, void* d_workspace, size_t workspace_bytes, int64_t num,
                          int32_t M, int32_t K, int32_t num_points, int32_t method, int32_t output, int32_t hard_out,
                          void* stream) {
    const int rc = ml_check("sb_mimo_ml", K, num_points, method, output, hard_out);
    if (rc != SB_OK) return rc;
    if (num == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_y && d_h && d_s && d_points && d_out && num > 0 && M >= 1, "sb_mimo_ml: bad arguments");
    return ml_run("sb_mimo_ml", sb_dense::dense_problem(d_y, d_h, d_s, num, M, K), d_prior, d_points, num_points,
                  method, output, hard_out, d_out, d_workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int sb_ofdm_ml(const float* d_y, const float* d_h_hat, const float* d_err_var, const int64_t* h_ev_stride,
                          const float* d_no, const int64_t* h_no_stride, const int32_t* d_desired,
                          const int32_t* d_undesired, const int32_t* d_out_stream, const int32_t* d_data_pos,
                          const float* d_prior, const float* d_points, void* d_out, void* d_workspace,
                          size_t workspace_bytes, int64_t batch, int32_t num_rx,
                          int32_t num_rx_ant, int32_t num_tx_streams, int32_t num_symbols, int32_t num_subcarriers,
                          int32_t streams_per_rx, int32_t interferers_per_rx, int32_t num_data, int32_t num_points,
                          int32_t method, int32_t output, int32_t hard_out, void* stream) {
    const int rc = ml_check("sb_ofdm_ml", streams_per_rx, num_points, method, output, hard_out);
    if (rc != SB_OK) return rc;
    if (batch == 0) return SB_OK;                       // empty batch: nothing to do, pointers may be null
    const int ac = sb_dense::ofdm_check("sb_ofdm_ml", d_y, d_h_hat, d_err_var, h_ev_stride, d_no, h_no_stride, d_desired,
                                        d_undesired, d_out_stream, d_data_pos, d_points, d_out, batch, num_rx_ant,
                                        interferers_per_rx);
    if (ac != SB_OK) return ac;
    const MimoProblem pb = sb_dense::ofdm_problem(d_y, d_h_hat, d_err_var, h_ev_stride, d_no, h_no_stride, d_desired,
                                                  d_undesired, d_out_stream, d_data_pos, batch, num_rx, num_rx_ant,
                                                  num_tx_streams, num_symbols, num_subcarriers, streams_per_rx,
                                                  interferers_per_rx, num_data);
    return ml_run("sb_ofdm_ml", pb, d_prior, d_points, num_points, method, output, hard_out, d_out, d_workspace,
                  workspace_bytes, (cudaStream_t)stream);
}
