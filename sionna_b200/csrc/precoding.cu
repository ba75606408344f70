// precoding.cu -- transmit precoding for sm_90a. Replaces (paths under the reference's src/sionna/phy/):
//   sb_mimo_precode   rzf_precoding_matrix, cbf_precoding_matrix, rzf_precoder      mimo/precoding.py:12-245
//   sb_ofdm_precode   RZFPrecoder.call ofdm/precoding.py:118-177 and PrecodedChannel with its RZF / CBF / Eye
//                     subclasses :179-566: desired-channel gather, precoding matrix, transmit power, x_precoded and
//                     the effective channel toward every receiver, nulled subcarriers removed
// One group of W lanes per problem (W = the power of two >= max(M, K), at most a warp), so that the 8 x 4 downlink of
// the tutorial packs four problems into a warp and M = 64 spreads over a whole one. Per group, in shared memory:
//   X [K, M + 1]  the desired channel H (K x M), overwritten column by column by (H H^H + alpha I)^-1 H (lane m owns
//                 columns m, m + W, ...: each solves its own right-hand sides), then by G^T with unit-norm columns and
//                 the power scale. The row pad keeps lanes that read the same column of different rows on distinct
//                 banks.
//   C [K, K]      H H^H + alpha I, its lower triangle computed by all lanes, then factorised by one lane (chol_lower)
//   xs [K], sc [K] the symbols of the element and per stream (norm, sqrt(tx_power))
// The arithmetic is the LMMSE kernels' (chol_lower, chol_solve_col, dense_mimo.cuh).
#include "sb_common.h"
#include "dense_mimo.cuh"

namespace {

using sb_dense::Scratch;
using sb_dense::chol_lower;
using sb_dense::chol_solve_col;
using sb_dense::kScratchSmemCap;

constexpr int kMaxStreams = 16;
constexpr int kMaxTxAnt = 1024;
constexpr int kCtaThreads = 128;

enum PrecoderKind { kRzf = 0, kCbf = 1, kIdentity = 2 };

// float2 of shared memory per problem
__host__ __device__ constexpr int group_elems(int M, int K) { return K * (M + 1) + K * K + 2 * K; }

// is_ofdm: problem i = element (b, tx, s, f) of the flattened [B, TX, S, F] grid; the desired channel of stream k is
// hhat[b, pind[tx, k / RA], k % RA, tx, :, s, f]. Dense: problem i has h [K, M] at hhat + i K M.
struct PrecodeParams {
    const float2* hhat;        // OFDM h_hat [B, RX, RA, TX, M, S, F]; dense h [P, K, M]
    const float2* h;           // OFDM channel of h_eff [B, RX, RA, TX, M, S, F]
    const float2* x;           // OFDM [B, TX, K, S, F]; dense [P, K]
    const float* alpha;        // strides (b, tx, s, f); dense: alpha_st[0] per problem
    const float* pw;           // tx_power, strides (b, tx, k, s, f)
    long long alpha_st[4], pw_st[5];
    const int* pind;           // [TX, RPT]
    const int* sc_pos;         // [F]: column of subcarrier f in h_eff, -1 if nulled
    float2* xp;                // OFDM [B, TX, M, S, F]; dense [P, M]
    float2* heff;              // [B, RX, RA, TX, K, S, NE]
    float2* g;                 // dense [P, M, K]
    long long P;
    int is_ofdm, kind, lanes;
    int RX, RA, TX, M, K, S, F, NE, RPT;
};

__global__ void __launch_bounds__(kCtaThreads) precode_kernel(const PrecodeParams p) {
    extern __shared__ float2 smem[];
    const int W = p.lanes, grp = threadIdx.x / W, lane = threadIdx.x % W, groups = blockDim.x / W;
    const int M = p.M, K = p.K, ld = M + 1;
    float2* base = smem + (size_t)grp * group_elems(M, K);
    const Scratch X{base, 1, 0};
    const Scratch C{base + K * ld, 1, 0};
    float2* xs = base + K * ld + K * K;
    float2* sc = xs + K;
    const long long SF = (long long)p.S * p.F;
    // problem i = bt SF + sf (OFDM: bt = b TX + j, sf = s F + f), advanced by the grid stride without 64-bit divisions
    const int stride = gridDim.x * groups, isf = (int)SF;
    const int st_bt = stride / isf, st_sf = stride % isf;
    long long i = (long long)blockIdx.x * groups + grp;
    int bt = (int)(i / SF), sfi = (int)(i % SF);
    // every thread of the CTA runs the same number of rounds, so the __syncwarp()s below are reached by whole warps
    for (long long r0 = (long long)blockIdx.x * groups; r0 < p.P; r0 += stride, i += stride) {
        const bool act = i < p.P;
        const int s = sfi / p.F, f = sfi % p.F, j = bt % p.TX;
        const long long b = bt / p.TX, sf = sfi;
        if (act) {
            if (p.kind != kIdentity)
                for (int e = lane; e < K * M; e += W) {
                    const int k = e / M, m = e % M;
                    long long src;
                    if (p.is_ofdm) {
                        const int rx = p.pind[j * p.RPT + k / p.RA], a = k % p.RA;
                        src = ((((b * p.RX + rx) * p.RA + a) * p.TX + j) * M + m) * SF + sf;
                    } else {
                        src = (i * K + k) * M + m;
                    }
                    X(k * ld + m) = p.hhat[src];
                }
            if (p.x)
                for (int k = lane; k < K; k += W)
                    xs[k] = p.x[p.is_ofdm ? ((b * p.TX + j) * K + k) * SF + sf : i * K + k];
        }
        __syncwarp();
        if (p.kind == kRzf) {                                   // X = (H H^H + alpha I)^-1 H   (precoding.py:77-82)
            if (act) {
                float al = 0.f;
                if (p.alpha)
                    al = p.alpha[p.is_ofdm ? b * p.alpha_st[0] + j * p.alpha_st[1] + s * p.alpha_st[2] + f * p.alpha_st[3]
                                           : i * p.alpha_st[0]];
                for (int e = lane; e < K * (K + 1) / 2; e += W) {          // lower triangle, row by row
                    int a = (int)((sqrtf(8.f * e + 1.f) - 1.f) * 0.5f);
                    while (a * (a + 1) / 2 > e) --a;
                    while ((a + 1) * (a + 2) / 2 <= e) ++a;
                    const int c = e - a * (a + 1) / 2;
                    float2 acc = make_float2(a == c ? al : 0.f, 0.f);
                    for (int m = 0; m < M; ++m) acc = cadd(acc, cmulc(X(a * ld + m), X(c * ld + m)));
                    C(a * K + c) = acc;
                }
            }
            __syncwarp();
            if (act && lane == 0) chol_lower(C, K);
            __syncwarp();
            if (act)
                for (int m = lane; m < M; m += W) chol_solve_col(C, K, [&](int r) { return X(r * ld + m); }, X, ld, m);
            __syncwarp();
        }
        if (act)                                                // per stream: column norm of G and sqrt(tx_power)
            for (int k = lane; k < K; k += W) {
                float n2 = 1.f;
                if (p.kind != kIdentity) {
                    n2 = 0.f;
                    for (int m = 0; m < M; ++m) { const float2 v = X(k * ld + m); n2 += v.x * v.x + v.y * v.y; }
                }
                float sp = 1.f;
                if (p.pw)
                    sp = sqrtf(p.pw[b * p.pw_st[0] + j * p.pw_st[1] + k * p.pw_st[2] + s * p.pw_st[3] + f * p.pw_st[4]]);
                sc[k] = make_float2(sqrtf(n2), sp);
            }
        __syncwarp();
        if (act)                                                // X <- G^T: G = divide_no_nan(X^H, norm) * sqrt(p)
            for (int e = lane; e < K * M; e += W) {
                const int k = e / M, m = e % M;
                const float2 ns = sc[k];
                float2 v;
                if (p.kind == kIdentity) {
                    v = make_float2(k == m ? 1.f : 0.f, 0.f);
                } else {
                    // a reciprocal, not a division: the division's slow-path call made ptxas spill the loop state
                    const float r = ns.x > 0.f ? __frcp_rn(ns.x) : 0.f;
                    v = X(k * ld + m);
                    v = make_float2(v.x * r, -v.y * r);
                }
                X(k * ld + m) = cscale(v, ns.y);
            }
        __syncwarp();
        if (act) {
            if (p.xp)                                           // x_precoded = G x
                for (int m = lane; m < M; m += W) {
                    float2 acc = make_float2(0.f, 0.f);
                    for (int k = 0; k < K; ++k) acc = cadd(acc, cmul(X(k * ld + m), xs[k]));
                    p.xp[p.is_ofdm ? ((b * p.TX + j) * M + m) * SF + sf : i * M + m] = acc;
                }
            if (p.g)
                for (int e = lane; e < M * K; e += W) {
                    const int m = e / K, k = e % K;
                    p.g[i * M * K + e] = X(k * ld + m);
                }
            const int pos = p.heff ? p.sc_pos[f] : -1;
            if (pos >= 0)                                       // h_eff[b, rx, a, j, k] = (H_{rx, j} G_j)[a, k]
                for (int e = lane; e < p.RX * p.RA * K; e += W) {
                    const int ra = e / K, k = e % K;
                    const long long row = ((b * p.RX + ra / p.RA) * p.RA + ra % p.RA) * p.TX + j;
                    const float2* hr = p.h + row * M * SF + sf;
                    float2 acc = make_float2(0.f, 0.f);
                    for (int m = 0; m < M; ++m) acc = cadd(acc, cmul(hr[m * SF], X(k * ld + m)));
                    p.heff[((row * K + k) * p.S + s) * (long long)p.NE + pos] = acc;
                }
        }
        __syncwarp();
        bt += st_bt;
        sfi += st_sf;
        if (sfi >= isf) { sfi -= isf; ++bt; }
    }
}

// Shape checks shared by both entry points: SB_EINVAL for malformed, SB_EUNSUPPORTED beyond the limits
int shape_check(const char* who, int K, int M, int kind) {
    SB_CHECK_ARG(K >= 1 && M >= 1 && kind >= kRzf && kind <= kIdentity,
                 "%s: bad arguments (need K >= 1, M >= 1, kind in {0, 1, 2})", who);
    SB_CHECK_ARG(kind != kIdentity || K == M, "%s: the identity precoder needs num_streams_per_tx = num_tx_ant", who);
    if (K > kMaxStreams) {
        sb_set_error("%s: %d streams, the limit is %d", who, K, kMaxStreams);
        return SB_EUNSUPPORTED;
    }
    if (M > kMaxTxAnt) {
        sb_set_error("%s: %d transmit antennas, the limit is %d", who, M, kMaxTxAnt);
        return SB_EUNSUPPORTED;
    }
    return SB_OK;
}

int precode_run(const char* who, PrecodeParams p, cudaStream_t stream) {
    if (p.P / ((long long)p.S * p.F) > INT32_MAX || (long long)p.S * p.F > INT32_MAX) {
        sb_set_error("%s: %lld problems, the limit is 2^31 per OFDM symbol and subcarrier", who, (long long)p.P);
        return SB_EUNSUPPORTED;
    }
    int lanes = 1;
    while (lanes < std::max(p.M, p.K) && lanes < 32) lanes *= 2;
    const size_t per = sizeof(float2) * group_elems(p.M, p.K);   // K <= 16, M <= 1024: at most 133 KB
    const int groups = (int)std::min<size_t>(kCtaThreads / lanes, kScratchSmemCap / per);   // lanes < 32: all fit
    const size_t smem = per * groups;
    p.lanes = lanes;
    SB_CUDA(cudaFuncSetAttribute(precode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    precode_kernel<<<sb_grid(p.P, groups, 16), groups * lanes, smem, stream>>>(p);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

}  // namespace

extern "C" int sb_mimo_precode(const float* d_h, const float* d_alpha, int64_t alpha_stride, const float* d_x,
                               float* d_g, float* d_gx, int64_t num, int32_t K, int32_t M, int32_t kind, void* stream) {
    const int rc = shape_check("sb_mimo_precode", K, M, kind);
    if (rc != SB_OK) return rc;
    SB_CHECK_ARG(kind != kIdentity && num >= 0 && (alpha_stride == 0 || alpha_stride == 1) && (!d_gx || d_x) &&
                     (!d_alpha || kind == kRzf),
                 "sb_mimo_precode: bad arguments (kind in {0, 1}, alpha_stride in {0, 1}, Gx needs x, alpha needs rzf)");
    if (num == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_h && (d_g || d_gx), "sb_mimo_precode: bad arguments (need h and an output)");
    PrecodeParams p{};
    p.hhat = (const float2*)d_h; p.x = (const float2*)d_x; p.alpha = d_alpha; p.alpha_st[0] = alpha_stride;
    p.g = (float2*)d_g; p.xp = (float2*)d_gx;
    p.P = num; p.is_ofdm = 0; p.kind = kind; p.M = M; p.K = K; p.S = p.F = p.TX = 1;
    return precode_run("sb_mimo_precode", p, (cudaStream_t)stream);
}

extern "C" int sb_ofdm_precode(const float* d_h_hat, const float* d_h, const int32_t* d_precoding_ind, const float* d_x,
                               const float* d_alpha, const int64_t* h_alpha_stride, const float* d_tx_power,
                               const int64_t* h_tx_power_stride, const int32_t* d_sc_pos, float* d_x_precoded,
                               float* d_h_eff, int64_t batch, int32_t num_rx, int32_t num_rx_ant, int32_t num_tx,
                               int32_t num_tx_ant, int32_t num_streams_per_tx, int32_t num_symbols, int32_t fft_size,
                               int32_t num_effective_subcarriers, int32_t kind, void* stream) {
    const int rc = shape_check("sb_ofdm_precode", num_streams_per_tx, num_tx_ant, kind);
    if (rc != SB_OK) return rc;
    SB_CHECK_ARG(batch >= 0 && num_rx >= 1 && num_rx_ant >= 1 && num_tx >= 1 && num_symbols >= 1 && fft_size >= 1 &&
                     num_effective_subcarriers >= 1 && num_effective_subcarriers <= fft_size,
                 "sb_ofdm_precode: bad arguments (sizes)");
    SB_CHECK_ARG(kind == kIdentity || (num_streams_per_tx % num_rx_ant == 0 && num_streams_per_tx / num_rx_ant <= num_rx),
                 "sb_ofdm_precode: The required number of streams per transmitter does not match the channel dimensions");
    if (batch == 0) return SB_OK;                       // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG((kind == kIdentity || (d_h_hat && d_precoding_ind)) && (d_x_precoded || d_h_eff) &&
                     (!d_x_precoded || d_x) && (!d_h_eff || (d_h && d_sc_pos)) && (!d_alpha || h_alpha_stride) &&
                     (!d_tx_power || h_tx_power_stride),
                 "sb_ofdm_precode: bad arguments (pointers)");
    PrecodeParams p{};
    p.hhat = (const float2*)d_h_hat; p.h = (const float2*)d_h; p.x = (const float2*)d_x;
    p.alpha = kind == kRzf ? d_alpha : nullptr; p.pw = d_tx_power;
    for (int d = 0; d < 4; ++d) p.alpha_st[d] = p.alpha ? h_alpha_stride[d] : 0;
    for (int d = 0; d < 5; ++d) p.pw_st[d] = d_tx_power ? h_tx_power_stride[d] : 0;
    p.pind = d_precoding_ind; p.sc_pos = d_sc_pos;
    p.xp = (float2*)d_x_precoded; p.heff = (float2*)d_h_eff;
    p.is_ofdm = 1; p.kind = kind;
    p.RX = num_rx; p.RA = num_rx_ant; p.TX = num_tx; p.M = num_tx_ant; p.K = num_streams_per_tx;
    p.S = num_symbols; p.F = fft_size; p.NE = num_effective_subcarriers;
    p.RPT = kind == kIdentity ? 1 : num_streams_per_tx / num_rx_ant;
    p.P = batch * num_tx * (long long)num_symbols * fft_size;
    return precode_run("sb_ofdm_precode", p, (cudaStream_t)stream);
}
