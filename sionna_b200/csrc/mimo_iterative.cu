// mimo_iterative.cu -- EP and MMSE-PIC MIMO detection for sm_90a. Replaces (paths under /root/reference/src/sionna/phy/):
//   sb_mimo_ep         EPDetector.call        mimo/detection.py:1039-1312 (+ complex2real_channel mimo/utils.py:194-242,
//                      SymbolLogits2LLRs mapping.py:927-967, PAM2QAM mapping.py:1234-1316)
//   sb_mimo_mmse_pic   MMSEPICDetector.call   mimo/detection.py:1314-1643 (+ LLRs2SymbolLogits mapping.py:1045-1059,
//                      SymbolLogits2Moments mapping.py:1061-1139, Demapper with_prior mapping.py:664-691)
//   sb_ofdm_ep / sb_ofdm_mmse_pic   the same detectors per OFDM resource element, with OFDMEqualizer's covariance
//                      S = H_u H_u^H + diag(no) + diag(sum err_var) assembled on chip (dense_mimo.cuh)
// The reference runs both as chains of batched TF ops that materialise [..., 2K, 2K] inverses, a [..., K, K] PIC matrix
// and [..., 2K, |C|] logits per iteration; here one thread keeps a whole problem in shared-memory scratch (one launch
// per call, no workspace).
//
// Shared prologue (it_prologue): y_w and H_w from the detectors' shared loader (load_whitened, dense_mimo.cuh), then
// G = H_w^H H_w and y_mf = H_w^H y_w, K x K complex. Both detectors work on (G, y_mf) only.
//
// EP (ep_kernel): realify(G) and [Re y_mf; Im y_mf] are exactly the reference's H^T H and H^T y of the whitened real
// channel, whose noise variance is 1/2. Per iteration, A = realify(G) + diag(lam) / 2 is symmetric positive definite
// (lam >= 0): a real Cholesky A = L L^T of size n = 2K, L inverted in place, gives
//   Sigma_ii = 1/2 ||L^-1 e_i||^2 (squared column norms of L^-1),  mu = L^-T L^-1 (H^T y + gam / 2)
// without a general inverse. v_obs, x_obs, the PAM softmax over <= 16 levels and the damped (lam, gam) update of
// eqs. (31)-(38) follow the reference operation by operation, with its single-precision clamp 1e-6. The final
// iteration's PAM logits give maxlog LLRs per PAM (real part on the even bit positions), QAM logits through PAM2QAM's
// gather, or the argmax of each PAM.
//
// MMSE-PIC (pic_kernel<METHOD, MB>): per self-iteration, the a-priori LLRs give point logits (demap_prior_logit), whose
// softmax gives x_bar and v; A = G diag(v) + I is inverted in place by complex Gauss-Jordan without pivoting (its
// leading principal minors are those of D^1/2 G D^1/2 + I >= I, so every pivot is real and >= 1 in exact arithmetic);
// mu_i = Re (A^-1 G)_ii, x~_i = (A^-1 (y_mf - sum_{j != i} g_j x_bar_j))_i / mu_i, no_eff = max(1 - v mu, 1e-4) / mu,
// then demapping with the prior (demap_symbol, the arithmetic of sb_demap). The output is llr_d - llr_a.
// The reference's real 2K x 2K inverse is realify of this complex one, so both compute the same quantities.
#include "sb_common.h"
#include "dense_mimo.cuh"
#include "demap_prior.cuh"

namespace {

using sb_dense::Scratch;
using sb_dense::MimoProblem;
using sb_dense::ScratchOf;

constexpr int kItMaxStreams = 16;
constexpr int kEpMaxPoints = 256;                      // 16 PAM levels per real dimension
constexpr int kPicMaxPoints = 1024;

// Scratch of the prologue, in float2 per thread: S [M, M], H [M, K], Y [M], G [K, K], y_mf [K]
__host__ __device__ constexpr size_t it_base_size(int M, int K) {
    return (size_t)M * M + (size_t)M * K + M + (size_t)K * K + K;
}

// load_whitened, then G and y_mf in scratch. False for an OFDM element that carries no data.
__device__ bool it_prologue(const MimoProblem& q, long long i, const Scratch& Sc, const Scratch& H, const Scratch& Y,
                            const Scratch& G, const Scratch& YM, long long* oi) {
    const int M = q.M, K = q.K;
    if (!sb_dense::load_whitened(q, i, Sc, H, Y, oi)) return false;
    for (int a = 0; a < K; ++a) {
        for (int b = 0; b < K; ++b) {
            float2 g = make_float2(0.f, 0.f);
            for (int m = 0; m < M; ++m) g = cadd(g, cmulc(H(m * K + b), H(m * K + a)));   // conj(h_ma) h_mb
            G(a * K + b) = g;
        }
        float2 v = make_float2(0.f, 0.f);
        for (int m = 0; m < M; ++m) v = cadd(v, cmulc(Y(m), H(m * K + a)));
        YM(a) = v;
    }
    return true;
}

// ---------------------------------------------------------------------------------------------------------------------
// EP
struct EpParams {
    MimoProblem pb;
    const float* levels;                                // [L] PAM levels by label, energy 1/2
    void* out;
    int L, hb, l, output, hard;                         // hb = bits per PAM
    float beta;
};

// Scratch after the prologue, floats per thread with n = 2 K: A [n, n], lam, gam, sig, mu, z, xo, vo [n] each
__host__ __device__ constexpr size_t ep_real_size(int K) { return 4 * (size_t)K * K + 14 * (size_t)K; }

// PAM logits -(x_obs - p)^2 / (2 v_obs) (detection.py:1197)
__device__ __forceinline__ float ep_logit(float xo, float vo, float p) {
    const float d = xo - p;
    return -(d * d) / (2.f * vo);
}

// maxlog LLR of bit u (MSB first) of a PAM from its logits
__device__ __forceinline__ float ep_pam_llr(const float* lev, int L, int hb, int u, float xo, float vo) {
    float l0 = -INFINITY, l1 = -INFINITY;
    for (int t = 0; t < L; ++t) {
        const float z = ep_logit(xo, vo, lev[t]);
        if ((t >> (hb - 1 - u)) & 1) l1 = fmaxf(l1, z); else l0 = fmaxf(l0, z);
    }
    return l1 - l0;
}

__device__ __forceinline__ int ep_pam_argmax(const float* lev, int L, float xo, float vo) {
    int best = 0;
    float bz = -INFINITY;
    for (int t = 0; t < L; ++t) {
        const float z = ep_logit(xo, vo, lev[t]);
        if (z > bz) { bz = z; best = t; }                // first maximum (tf.argmax)
    }
    return best;
}

// One thread per problem. Shared memory: levels [L] float, then the prologue's float2 scratch and EP's float scratch.
__global__ void ep_kernel(const EpParams q) {
    extern __shared__ float2 smem[];
    const int T = blockDim.x, t = threadIdx.x;
    const int M = q.pb.M, K = q.pb.K, n = 2 * K, L = q.L, hb = q.hb;
    float* lev = reinterpret_cast<float*>(smem);
    for (int i = t; i < L; i += T) lev[i] = q.levels[i];
    __syncthreads();
    float es;                                           // np.var of the levels
    {
        float mean = 0.f, e2 = 0.f;
        for (int i = 0; i < L; ++i) mean += lev[i];
        mean /= (float)L;
        for (int i = 0; i < L; ++i) e2 += (lev[i] - mean) * (lev[i] - mean);
        es = e2 / (float)L;
    }
    float2* base = smem + 8;                            // 16 floats of levels
    const size_t o_h = (size_t)M * M, o_y = o_h + (size_t)M * K, o_g = o_y + M, o_ym = o_g + (size_t)K * K;
    const Scratch Sc{base, T, t}, H{base + o_h * T, T, t}, Y{base + o_y * T, T, t};
    const Scratch G{base + o_g * T, T, t}, YM{base + o_ym * T, T, t};
    float* rb = reinterpret_cast<float*>(base + it_base_size(M, K) * T);
    const ScratchOf<float> A{rb, T, t};
    const size_t nn = (size_t)n * n;
    const ScratchOf<float> lam{rb + nn * T, T, t}, gam{rb + (nn + n) * T, T, t}, sig{rb + (nn + 2 * n) * T, T, t},
        mu{rb + (nn + 3 * n) * T, T, t}, z{rb + (nn + 4 * n) * T, T, t}, xo{rb + (nn + 5 * n) * T, T, t},
        vo{rb + (nn + 6 * n) * T, T, t};
    const float prec = 1e-6f, beta = q.beta;
    long long oi[kItMaxStreams];
    for (long long i = (long long)blockIdx.x * T + t; i < q.pb.P; i += (long long)gridDim.x * T) {
        if (!it_prologue(q.pb, i, Sc, H, Y, G, YM, oi)) continue;
        for (int r = 0; r < n; ++r) { lam(r) = 1.f / es; gam(r) = 0.f; }
        for (int it = 0; it < q.l; ++it) {
            // A = realify(G) + lam / 2 (lower triangle), A = L L^T in place, then L^-1 in place
            for (int r = 0; r < n; ++r) {
                for (int c = 0; c <= r; ++c) {
                    const float2 g = G((r % K) * K + (c % K));
                    float a = (r < K) == (c < K) ? g.x : (r >= K ? g.y : -g.y);
                    if (r == c) a += 0.5f * lam(r);
                    A(r * n + c) = a;
                }
            }
            for (int j = 0; j < n; ++j) {
                float d = A(j * n + j);
                for (int k = 0; k < j; ++k) d -= A(j * n + k) * A(j * n + k);
                d = sqrtf(d);
                A(j * n + j) = d;
                for (int r = j + 1; r < n; ++r) {
                    float v = A(r * n + j);
                    for (int k = 0; k < j; ++k) v -= A(r * n + k) * A(j * n + k);
                    A(r * n + j) = v / d;
                }
            }
            for (int j = 0; j < n; ++j) {               // column j of L^-1 over column j of L (later columns unread)
                const float dj = 1.f / A(j * n + j);
                A(j * n + j) = dj;
                for (int r = j + 1; r < n; ++r) {
                    float v = A(r * n + j) * dj;
                    for (int k = j + 1; k < r; ++k) v += A(r * n + k) * A(k * n + j);
                    A(r * n + j) = -v / A(r * n + r);
                }
            }
            // Sigma_ii = 1/2 ||L^-1 e_i||^2; mu = L^-T L^-1 (H^T y + gam / 2)
            for (int r = 0; r < n; ++r) {
                float v = 0.f;
                for (int c = 0; c <= r; ++c) {
                    const float2 ym = YM(c % K);
                    v += A(r * n + c) * ((c < K ? ym.x : ym.y) + 0.5f * gam(c));
                }
                z(r) = v;
            }
            for (int c = 0; c < n; ++c) {
                float s2 = 0.f, m2 = 0.f;
                for (int r = c; r < n; ++r) { const float a = A(r * n + c); s2 += a * a; m2 += a * z(r); }
                sig(c) = 0.5f * s2;
                mu(c) = m2;
            }
            const bool last = it == q.l - 1;
            for (int r = 0; r < n; ++r) {
                const float s = sig(r), lm = lam(r), gm = gam(r);
                const float v_obs = fmaxf(1.f / (1.f / s - lm), prec);
                const float x_obs = v_obs * (mu(r) / s - gm);
                xo(r) = x_obs;
                vo(r) = v_obs;
                if (last) continue;                     // the last update does not reach the output
                float mx = -INFINITY;
                for (int u = 0; u < L; ++u) mx = fmaxf(mx, ep_logit(x_obs, v_obs, lev[u]));
                float se = 0.f, sx = 0.f;
                for (int u = 0; u < L; ++u) {
                    const float e = expf(ep_logit(x_obs, v_obs, lev[u]) - mx);
                    se += e;
                    sx += lev[u] * e;
                }
                const float x = sx / se;
                float sv = 0.f;
                for (int u = 0; u < L; ++u) {
                    const float d = lev[u] - x;
                    sv += d * d * expf(ep_logit(x_obs, v_obs, lev[u]) - mx);
                }
                const float v = fmaxf(sv / se, prec);
                const float ln = 1.f / v - 1.f / v_obs, gn = x / v - x_obs / v_obs;
                const bool keep = ln < 0.f;
                lam(r) = (1.f - beta) * (keep ? lm : ln) + beta * lm;
                gam(r) = (1.f - beta) * (keep ? gm : gn) + beta * gm;
            }
        }
        // outputs from the final iteration's PAM logits
        for (int k = 0; k < K; ++k) {
            const long long o = oi[k];
            if (o < 0) continue;
            const float xr = xo(k), vr = vo(k), xi = xo(K + k), vi = vo(K + k);
            if (q.output == 0) {
                float* out = static_cast<float*>(q.out) + o * 2 * hb;
                for (int u = 0; u < hb; ++u) {
                    const float l1 = ep_pam_llr(lev, L, hb, u, xr, vr), l2 = ep_pam_llr(lev, L, hb, u, xi, vi);
                    out[2 * u] = q.hard ? (l1 > 0.f ? 1.f : 0.f) : l1;
                    out[2 * u + 1] = q.hard ? (l2 > 0.f ? 1.f : 0.f) : l2;
                }
            } else if (q.hard) {
                static_cast<int*>(q.out)[o] =
                    sb_dense::pam2qam_index(ep_pam_argmax(lev, L, xr, vr), ep_pam_argmax(lev, L, xi, vi), 2 * hb);
            } else {
                // PAM2QAM's gather (mapping.py:1307-1314): output c takes the flattened (re, im) pair at the QAM index
                // of the pair (c / L, c % L)
                float* out = static_cast<float*>(q.out) + o * L * L;
                for (int c = 0; c < L * L; ++c) {
                    const int g = sb_dense::pam2qam_index(c / L, c % L, 2 * hb);
                    out[c] = ep_logit(xr, vr, lev[g / L]) + ep_logit(xi, vi, lev[g % L]);
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// MMSE-PIC
struct PicParams {
    MimoProblem pb;
    const float2* points;                               // [2^MB]
    const float* prior;                                 // bit LLRs in the output layout, or null (zero prior)
    float* out;
    int num_iter, hard;
};

// Scratch after the prologue, float2 per thread: A [K, K], x_bar, v, G x_bar, x~, no_eff [K] each (v and no_eff in .x);
// then floats: llr_a [K, MB]
__host__ __device__ constexpr size_t pic_size(int K) { return (size_t)K * K + 5 * (size_t)K; }

// One thread per problem. Shared memory: points [2^MB] float2, then the float2 scratch and llr_a.
template <int METHOD, int MB>
__global__ void pic_kernel(const PicParams q) {
    constexpr int NP = 1 << MB;
    extern __shared__ float2 smem[];
    const int T = blockDim.x, t = threadIdx.x;
    const int M = q.pb.M, K = q.pb.K;
    float2* pts = smem;
    for (int i = t; i < NP; i += T) pts[i] = q.points[i];
    __syncthreads();
    float2* base = smem + NP;
    const size_t o_h = (size_t)M * M, o_y = o_h + (size_t)M * K, o_g = o_y + M, o_ym = o_g + (size_t)K * K;
    const Scratch Sc{base, T, t}, H{base + o_h * T, T, t}, Y{base + o_y * T, T, t};
    const Scratch G{base + o_g * T, T, t}, YM{base + o_ym * T, T, t};
    float2* pb = base + it_base_size(M, K) * T;
    const size_t kk = (size_t)K * K;
    const Scratch A{pb, T, t}, XB{pb + kk * T, T, t}, V{pb + (kk + K) * T, T, t}, TG{pb + (kk + 2 * K) * T, T, t},
        XT{pb + (kk + 3 * K) * T, T, t}, NE{pb + (kk + 4 * K) * T, T, t};
    const ScratchOf<float> LA{reinterpret_cast<float*>(pb + pic_size(K) * T), T, t};
    const float tiny = 1.17549435e-38f;                 // np.finfo(float32).tiny, as sb_demap
    long long oi[kItMaxStreams];
    for (long long i = (long long)blockIdx.x * T + t; i < q.pb.P; i += (long long)gridDim.x * T) {
        if (!it_prologue(q.pb, i, Sc, H, Y, G, YM, oi)) continue;
        for (int k = 0; k < K; ++k)
            for (int b = 0; b < MB; ++b) LA(k * MB + b) = q.prior && oi[k] >= 0 ? q.prior[oi[k] * MB + b] : 0.f;
        for (int it = 0; it < q.num_iter; ++it) {
            // soft symbols and variances from the a-priori LLRs (LLRs2SymbolLogits -> SymbolLogits2Moments)
            for (int k = 0; k < K; ++k) {
                float ls1[MB], ls0[MB];
#pragma unroll
                for (int b = 0; b < MB; ++b) {
                    const float pk = LA(k * MB + b);
                    ls1[b] = log_sigmoidf(pk);
                    ls0[b] = log_sigmoidf(__fmul_rn(-1.f, pk));
                }
                float mx = -INFINITY;
                for (int c = 0; c < NP; ++c) mx = fmaxf(mx, demap_prior_logit<MB>(ls1, ls0, c));
                float se = 0.f;
                float2 sx = make_float2(0.f, 0.f);
                for (int c = 0; c < NP; ++c) {
                    const float e = expf(demap_prior_logit<MB>(ls1, ls0, c) - mx);
                    se += e;
                    sx = cadd(sx, cscale(pts[c], e));
                }
                const float2 xb = cscale(sx, 1.f / se);
                float sv = 0.f;
                for (int c = 0; c < NP; ++c) {
                    const float2 d = csub(pts[c], xb);
                    sv += (d.x * d.x + d.y * d.y) * expf(demap_prior_logit<MB>(ls1, ls0, c) - mx);
                }
                XB(k) = xb;
                V(k) = make_float2(sv / se, 0.f);
            }
            // G x_bar, then A = G diag(v) + I and A^-1 in place (Gauss-Jordan, pivots real >= 1)
            for (int r = 0; r < K; ++r) {
                float2 s = make_float2(0.f, 0.f);
                for (int c = 0; c < K; ++c) {
                    const float2 g = G(r * K + c);
                    s = cadd(s, cmul(g, XB(c)));
                    A(r * K + c) = make_float2(g.x * V(c).x + (r == c ? 1.f : 0.f), g.y * V(c).x);
                }
                TG(r) = s;
            }
            for (int p = 0; p < K; ++p) {
                const float2 inv = cdiv(make_float2(1.f, 0.f), A(p * K + p));
                A(p * K + p) = make_float2(1.f, 0.f);
                for (int c = 0; c < K; ++c) A(p * K + c) = cmul(A(p * K + c), inv);
                for (int r = 0; r < K; ++r) {
                    if (r == p) continue;
                    const float2 f = A(r * K + p);
                    A(r * K + p) = make_float2(0.f, 0.f);
                    for (int c = 0; c < K; ++c) A(r * K + c) = csub(A(r * K + c), cmul(f, A(p * K + c)));
                }
            }
            // bias mu_j = Re (A^-1 G)_jj, PIC estimate of stream j, its effective noise variance
            for (int j = 0; j < K; ++j) {
                const float2 xj = XB(j);
                float m = 0.f;
                float2 s = make_float2(0.f, 0.f);
                for (int c = 0; c < K; ++c) {
                    const float2 a = A(j * K + c), g = G(c * K + j);
                    m += a.x * g.x - a.y * g.y;
                    s = cadd(s, cmul(a, csub(cadd(YM(c), cmul(g, xj)), TG(c))));
                }
                XT(j) = cscale(s, 1.f / m);
                const float rho = m / fmaxf(1.f - V(j).x * m, 1e-4f);
                NE(j) = make_float2(1.f / rho, 0.f);
            }
            // demapping with the prior; llr_d feeds the next iteration, the last one leaves as llr_d - llr_a
            const bool last = it == q.num_iter - 1;
            for (int k = 0; k < K; ++k) {
                float ls1[MB], ls0[MB], la[MB], ld[MB];
#pragma unroll
                for (int b = 0; b < MB; ++b) {
                    la[b] = LA(k * MB + b);
                    ls1[b] = log_sigmoidf(la[b]);
                    ls0[b] = log_sigmoidf(__fmul_rn(-1.f, la[b]));
                }
                demap_symbol<METHOD, MB>(XT(k), fmaxf(NE(k).x, tiny), pts, ls1, ls0, true, ld);
                if (!last) {
#pragma unroll
                    for (int b = 0; b < MB; ++b) LA(k * MB + b) = ld[b];
                } else if (oi[k] >= 0) {
                    float* out = q.out + oi[k] * MB;
#pragma unroll
                    for (int b = 0; b < MB; ++b) {
                        const float e = ld[b] - la[b];
                        out[b] = q.hard ? (e > 0.f ? 1.f : 0.f) : e;
                    }
                }
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------------------
// Malformed arguments are SB_EINVAL; well-formed configurations beyond the kernels' limits are SB_EUNSUPPORTED.
int it_check_common(const char* who, int M, int K, int num_points, int max_points, int hard_out) {
    if (M < 1 || K < 1 || num_points < 2 || (num_points & (num_points - 1)) || hard_out < 0 || hard_out > 1) {
        sb_set_error("%s: bad arguments (need M >= 1 antennas, K >= 1 streams, a power-of-two constellation of >= 2 "
                     "points, hard_out in {0, 1})", who);
        return SB_EINVAL;
    }
    if (K > kItMaxStreams) {
        sb_set_error("%s: %d streams, the limit is %d", who, K, kItMaxStreams);
        return SB_EUNSUPPORTED;
    }
    if (num_points > max_points) {
        sb_set_error("%s: a constellation of %d points, the limit is %d", who, num_points, max_points);
        return SB_EUNSUPPORTED;
    }
    return SB_OK;
}

int ep_check(const char* who, int M, int K, int num_points, int l, float beta, int output, int hard_out) {
    const int rc = it_check_common(who, M, K, num_points, kEpMaxPoints, hard_out);
    if (rc != SB_EINVAL && (l < 1 || !(beta >= 0.f && beta <= 1.f) || output < 0 || output > 1)) {
        sb_set_error("%s: bad arguments (need l >= 1, 0 <= beta <= 1, output in {0, 1})", who);
        return SB_EINVAL;
    }
    if (rc != SB_EINVAL && (31 - __builtin_clz((unsigned)num_points)) % 2) {
        sb_set_error("%s: bad arguments (EP needs a QAM constellation, an even number of bits; %d points given)", who,
                     num_points);
        return SB_EINVAL;
    }
    return rc;
}

int pic_check(const char* who, int M, int K, int num_points, int num_iter, int method, int hard_out) {
    const int rc = it_check_common(who, M, K, num_points, kPicMaxPoints, hard_out);
    if (rc != SB_EINVAL && (num_iter < 1 || method < 0 || method > 1)) {
        sb_set_error("%s: bad arguments (need num_iter >= 1, method in {0, 1})", who);
        return SB_EINVAL;
    }
    return rc;
}

int ep_run(const char* who, const MimoProblem& pb, const float* levels, int num_points, int l, float beta, int output,
           int hard_out, void* out, cudaStream_t stream) {
    const int m = 31 - __builtin_clz((unsigned)num_points), hb = m / 2;
    const size_t per = sizeof(float2) * it_base_size(pb.M, pb.K) + sizeof(float) * ep_real_size(pb.K);
    size_t smem = 0;
    const int th = sb_dense::detector_threads(who, 16 * sizeof(float), per, pb.M, pb.K, &smem);
    if (!th) return SB_EUNSUPPORTED;
    EpParams q{pb, levels, out, 1 << hb, hb, l, output, hard_out, beta};
    SB_CUDA(cudaFuncSetAttribute(ep_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    ep_kernel<<<sb_grid(pb.P, th, 16), th, smem, stream>>>(q);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

int pic_run(const char* who, const MimoProblem& pb, const float* prior, const float* points, int num_points, int num_iter,
            int method, int hard_out, float* out, cudaStream_t stream) {
    const int m = 31 - __builtin_clz((unsigned)num_points);
    const size_t per = sizeof(float2) * (it_base_size(pb.M, pb.K) + pic_size(pb.K)) + sizeof(float) * pb.K * m;
    size_t smem = 0;
    const int th = sb_dense::detector_threads(who, sizeof(float2) * num_points, per, pb.M, pb.K, &smem);
    if (!th) return SB_EUNSUPPORTED;
    PicParams q{pb, (const float2*)points, prior, out, num_iter, hard_out};
    return sb_dispatch<0, 1>(method, [&](auto METHOD) {
        return sb_dispatch<1, 10>(m, [&](auto MB) {
            auto kern = pic_kernel<METHOD, MB>;
            SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            kern<<<sb_grid(pb.P, th, 16), th, smem, stream>>>(q);
            SB_LAUNCH_CHECK();
            return SB_OK;
        });
    });
}

}  // namespace

extern "C" int sb_mimo_ep(const float* d_y, const float* d_h, const float* d_s, const float* d_levels, void* d_out,
                          int64_t num, int32_t M, int32_t K, int32_t num_points, int32_t l, float beta, int32_t output,
                          int32_t hard_out, void* stream) {
    const int rc = ep_check("sb_mimo_ep", M, K, num_points, l, beta, output, hard_out);
    if (rc != SB_OK) return rc;
    if (num == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_y && d_h && d_s && d_levels && d_out && num > 0, "sb_mimo_ep: bad arguments");
    return ep_run("sb_mimo_ep", sb_dense::dense_problem(d_y, d_h, d_s, num, M, K), d_levels, num_points, l, beta, output,
                  hard_out, d_out, (cudaStream_t)stream);
}

extern "C" int sb_ofdm_ep(const float* d_y, const float* d_h_hat, const float* d_err_var, const int64_t* h_ev_stride,
                          const float* d_no, const int64_t* h_no_stride, const int32_t* d_desired,
                          const int32_t* d_undesired, const int32_t* d_out_stream, const int32_t* d_data_pos,
                          const float* d_levels, void* d_out, int64_t batch, int32_t num_rx, int32_t num_rx_ant,
                          int32_t num_tx_streams, int32_t num_symbols, int32_t num_subcarriers, int32_t streams_per_rx,
                          int32_t interferers_per_rx, int32_t num_data, int32_t num_points, int32_t l, float beta,
                          int32_t output, int32_t hard_out, void* stream) {
    const int rc = ep_check("sb_ofdm_ep", num_rx_ant, streams_per_rx, num_points, l, beta, output, hard_out);
    if (rc != SB_OK) return rc;
    if (batch == 0) return SB_OK;                       // empty batch: nothing to do, pointers may be null
    const int ac = sb_dense::ofdm_check("sb_ofdm_ep", d_y, d_h_hat, d_err_var, h_ev_stride, d_no, h_no_stride, d_desired,
                                        d_undesired, d_out_stream, d_data_pos, d_levels, d_out, batch, num_rx_ant,
                                        interferers_per_rx);
    if (ac != SB_OK) return ac;
    const MimoProblem pb = sb_dense::ofdm_problem(d_y, d_h_hat, d_err_var, h_ev_stride, d_no, h_no_stride, d_desired,
                                                  d_undesired, d_out_stream, d_data_pos, batch, num_rx, num_rx_ant,
                                                  num_tx_streams, num_symbols, num_subcarriers, streams_per_rx,
                                                  interferers_per_rx, num_data);
    return ep_run("sb_ofdm_ep", pb, d_levels, num_points, l, beta, output, hard_out, d_out, (cudaStream_t)stream);
}

extern "C" int sb_mimo_mmse_pic(const float* d_y, const float* d_h, const float* d_s, const float* d_prior,
                                const float* d_points, float* d_out, int64_t num, int32_t M, int32_t K,
                                int32_t num_points, int32_t num_iter, int32_t method, int32_t hard_out, void* stream) {
    const int rc = pic_check("sb_mimo_mmse_pic", M, K, num_points, num_iter, method, hard_out);
    if (rc != SB_OK) return rc;
    if (num == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_y && d_h && d_s && d_points && d_out && num > 0, "sb_mimo_mmse_pic: bad arguments");
    return pic_run("sb_mimo_mmse_pic", sb_dense::dense_problem(d_y, d_h, d_s, num, M, K), d_prior, d_points, num_points, num_iter,
                   method, hard_out, d_out, (cudaStream_t)stream);
}

extern "C" int sb_ofdm_mmse_pic(const float* d_y, const float* d_h_hat, const float* d_err_var,
                                const int64_t* h_ev_stride, const float* d_no, const int64_t* h_no_stride,
                                const int32_t* d_desired, const int32_t* d_undesired, const int32_t* d_out_stream,
                                const int32_t* d_data_pos, const float* d_prior, const float* d_points, float* d_out,
                                int64_t batch, int32_t num_rx, int32_t num_rx_ant, int32_t num_tx_streams,
                                int32_t num_symbols, int32_t num_subcarriers, int32_t streams_per_rx,
                                int32_t interferers_per_rx, int32_t num_data, int32_t num_points, int32_t num_iter,
                                int32_t method, int32_t hard_out, void* stream) {
    const int rc = pic_check("sb_ofdm_mmse_pic", num_rx_ant, streams_per_rx, num_points, num_iter, method, hard_out);
    if (rc != SB_OK) return rc;
    if (batch == 0) return SB_OK;                       // empty batch: nothing to do, pointers may be null
    const int ac = sb_dense::ofdm_check("sb_ofdm_mmse_pic", d_y, d_h_hat, d_err_var, h_ev_stride, d_no, h_no_stride,
                                        d_desired, d_undesired, d_out_stream, d_data_pos, d_points, d_out, batch,
                                        num_rx_ant, interferers_per_rx);
    if (ac != SB_OK) return ac;
    const MimoProblem pb = sb_dense::ofdm_problem(d_y, d_h_hat, d_err_var, h_ev_stride, d_no, h_no_stride, d_desired,
                                                  d_undesired, d_out_stream, d_data_pos, batch, num_rx, num_rx_ant,
                                                  num_tx_streams, num_symbols, num_subcarriers, streams_per_rx,
                                                  interferers_per_rx, num_data);
    return pic_run("sb_ofdm_mmse_pic", pb, d_prior, d_points, num_points, num_iter, method, hard_out, d_out,
                   (cudaStream_t)stream);
}
