/* oracle/mapping_ref.c -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
 *
 * CPU restatement of /root/reference/src/sionna/phy/mapping.py:
 *   Demapper.call            :664-691   squared distance via |y - c| then pow 2, / max(no, tiny)
 *   SymbolLogits2LLRs.call   :927-967   gather into C_{i,0} / C_{i,1}, reduce_logsumexp ("app") or reduce_max
 *                                       ("maxlog"), optional prior through log_sigmoid
 * tf.reduce_logsumexp(x) = log(sum(exp(x - max))) + max with a non-finite max replaced by 0;
 * tf.math.log_sigmoid(x) = -softplus(-x), softplus with TensorFlow's threshold branches.
 * math_mode 0: glibc hypotf/expf/logf/log1pf; math_mode 1: the product's sb_math.h functions and
 * |d| = sqrt(fma(dr,dr,di*di)) -- then the CUDA demapper must agree bit for bit.
 * Pinned by the reference's own demapper test recipe (test/unit/mapping/test_mapping.py:175-225:
 * scipy.special.logsumexp / np.max over the two index sets, atol 1e-5), restated in tests/test_oracle_mapping.py.
 */
#include <math.h>
#include <stdint.h>
#include "../sionna_b200/csrc/sb_math.h"

static float m_exp(float x, int mode) { return mode ? sb_expf(x) : expf(x); }
static float m_log(float x, int mode) { return mode ? sb_logf(x) : logf(x); }
static float m_log1p_pos(float u, int mode) {
    if (!mode) return log1pf(u);
    float w = 1.f + u;
    if (w == 1.f) return u;
    return sb_logf(w) * (u / (w - 1.f));
}
static float softplus(float x, int mode) {
    const float threshold = -13.942385f;
    if (x > -threshold) return x;
    float ex = m_exp(x, mode);
    if (x < threshold) return ex;
    return m_log1p_pos(ex, mode);
}
static float log_sigmoid(float x, int mode) { return -softplus(-x, mode); }

static float exponent(float yr, float yi, float cr, float ci, float no, int mode) {
    float dr = yr - cr, di = yi - ci;
    float a = mode ? sqrtf(fmaf(dr, dr, di * di)) : hypotf(dr, di);
    return -(a * a) / no;
}

/* y [n_sym] complex64 (interleaved), no[s / no_inner], points [2^m], prior[(s / prior_inner) * m ..] or NULL,
 * method 0 app / 1 maxlog, llr [n_sym * m]. */
void sbo_demap(const float* y, const float* no, int64_t no_inner, const float* points, int m, int method,
               const float* prior, int64_t prior_inner, float* llr, int64_t n_sym, int hard_out, int math_mode) {
    const int npts = 1 << m;
    const float tiny = 1.17549435e-38f;
#pragma omp parallel for schedule(static)
    for (int64_t s = 0; s < n_sym; ++s) {
        float e[4096];
        float n0 = fmaxf(no[s / no_inner], tiny);
        const float* pr = prior ? prior + (s / prior_inner) * m : 0;
        for (int j = 0; j < npts; ++j) {
            float ex = exponent(y[2 * s], y[2 * s + 1], points[2 * j], points[2 * j + 1], n0, math_mode);
            if (pr) {
                float ps = 0.f;
                for (int k = 0; k < m; ++k) {
                    float lab = ((j >> (m - 1 - k)) & 1) ? 1.f : -1.f;
                    ps += log_sigmoid(lab * pr[k], math_mode);
                }
                ex = ps + ex;
            }
            e[j] = ex;
        }
        for (int i = 0; i < m; ++i) {
            int mask = 1 << (m - 1 - i);
            float acc[2];
            for (int v = 0; v < 2; ++v) {
                float mx = -INFINITY;
                for (int j = 0; j < npts; ++j) if (((j & mask) != 0) == (v == 1)) mx = fmaxf(mx, e[j]);
                if (method == 1) { acc[v] = mx; continue; }
                float mm = isfinite(mx) ? mx : 0.f;
                float sum = 0.f;
                for (int j = 0; j < npts; ++j) if (((j & mask) != 0) == (v == 1)) sum += m_exp(e[j] - mm, math_mode);
                acc[v] = (sum > 0.f ? m_log(sum, math_mode) : -INFINITY) + mm;
            }
            float l = acc[1] - acc[0];
            llr[s * m + i] = hard_out ? (l > 0.f ? 1.f : 0.f) : l;
        }
    }
}


/* Kernel-math restatement of the separable-QAM demapper (csrc/phy_kernels.cu demap_qam_kernel): mathematically the same
 * LLRs as sbo_demap (exp(e_j) factors into a real and an imaginary part and the other dimension's factor cancels), with
 * the operation order the CUDA kernel uses, so the two agree bit for bit. lev_re / lev_im: 2^(m/2) PAM levels indexed
 * by the even / odd label bits (MSB first). Always evaluated with sb_math.h (this path has no reference-order twin; the
 * reference-order value is sbo_demap with math_mode 0). */
void sbo_demap_qam(const float* y, const float* no, int64_t no_inner, const float* lev_re, const float* lev_im, int m,
                   int method, float* llr, int64_t n_sym, int hard_out) {
    const int H = m / 2, L = 1 << H;
    const float tiny = 1.17549435e-38f;
#pragma omp parallel for schedule(static)
    for (int64_t s = 0; s < n_sym; ++s) {
        float inv_n0 = 1.0f / fmaxf(no[s / no_inner], tiny);
        for (int d = 0; d < 2; ++d) {
            float yd = y[2 * s + d];
            float e[32];
            for (int t = 0; t < L; ++t) {
                float dd = yd - (d ? lev_im[t] : lev_re[t]);
                e[t] = -(dd * dd) * inv_n0;
            }
            float wgt[32], mx = -INFINITY;                         /* "app", H > 1: exponentials relative to the dimension's maximum */
            for (int t = 0; t < L; ++t) mx = fmaxf(mx, e[t]);
            mx = isfinite(mx) ? mx : 0.f;
            for (int t = 0; t < L; ++t) { float a = e[t] - mx; wgt[t] = a < -87.3f ? 0.f : sb_expf(a); }
            for (int u = 0; u < H; ++u) {
                int mask = 1 << (H - 1 - u);
                float mx0 = -INFINITY, mx1 = -INFINITY;
                for (int t = 0; t < L; ++t) { if (t & mask) mx1 = fmaxf(mx1, e[t]); else mx0 = fmaxf(mx0, e[t]); }
                float l;
                if (method == 1 || H == 1) {
                    l = mx1 - mx0;
                } else {
                    float s0 = 0.f, s1 = 0.f;
                    for (int t = 0; t < L; ++t) { if (t & mask) s1 += wgt[t]; else s0 += wgt[t]; }   /* ascending t */
                    if (fminf(s0, s1) >= 0x1p-92f) {              /* demap_qam.cuh DEMAP_QAM_GROUP_MIN */
                        l = sb_logf(s1) - sb_logf(s0);
                    } else {                                       /* a group's shared sum is tiny: per-group maxima */
                        mx0 = isfinite(mx0) ? mx0 : 0.f;
                        mx1 = isfinite(mx1) ? mx1 : 0.f;
                        s0 = 0.f; s1 = 0.f;
                        for (int t = 0; t < L; ++t) {
                            if (t & mask) { float a = e[t] - mx1; s1 += a < -87.3f ? 0.f : sb_expf(a); }
                            else { float a = e[t] - mx0; s0 += a < -87.3f ? 0.f : sb_expf(a); }
                        }
                        float b1 = (s1 > 0.f ? sb_logf(s1) : -INFINITY) + mx1;
                        float b0 = (s0 > 0.f ? sb_logf(s0) : -INFINITY) + mx0;
                        l = b1 - b0;
                    }
                }
                llr[s * m + 2 * u + d] = hard_out ? (l > 0.f ? 1.f : 0.f) : l;
            }
        }
    }
}
