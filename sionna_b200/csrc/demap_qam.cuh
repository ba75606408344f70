// demap_qam.cuh -- LLRs of ONE received symbol for a separable (square QAM) constellation without prior, shared by the
// stand-alone demapper kernel (phy_kernels.cu, sb_demap_qam) and the fused receive front-end (frontend.cu).
// Reference: Demapper.call + SymbolLogits2LLRs.call, /root/reference/src/sionna/phy/mapping.py:664-691, 927-967.
// Even label bits select the real PAM level, odd label bits the imaginary one (mapping.py:104-117): the 2-D sums factor,
// exp(e_j) = exp(e_re) exp(e_im), and the factor of the other dimension cancels in the LLR, so bit i only needs the
// 2^(M/2) exponents of its own dimension:
//   LLR_(2u+d) = logsumexp_{t: bit u of t = 1} e_d(t) - logsumexp_{t: bit u = 0} e_d(t),  e_d(t) = -(y_d - a_d(t))^2 * (1/no)
// (max instead of logsumexp for maxlog).
#pragma once
#include "sb_math.h"
#include "sb_math2.cuh"

// Least shared sum (relative to the dimension's maximum) of a bit group that the shared-maximum form keeps; below it the
// group is summed relative to its own maximum (derivation in demap_qam_dim). oracle/mapping_ref.c uses the same value.
constexpr float DEMAP_QAM_GROUP_MIN = 0x1p-92f;

// Slow path of "app": the shared sum of the bit group that does NOT contain the dimension's largest exponent is below
// DEMAP_QAM_GROUP_MIN (|LLR| > ~64: high SNR), so members of that group may have been flushed to 0 (e_t - max < -87.3)
// while they are still comparable to the group's own maximum, or the whole group underflowed and the shared-maximum form
// would return log(0). That group is summed relative to its OWN maximum, as the reference's per-group logsumexp does
// (mapping.py:915-918); the other group keeps its shared sum `s_ok` (its maximum IS the dimension's maximum `mx`). Out of
// line and loop-rolled on purpose: it must not bloat the callers' instruction stream. `lev` points at the 2^H levels of
// the dimension (global or kernel-parameter memory); g = the small group (value of bit u). Returns LLR =
// logsumexp(group 1) - logsumexp(group 0).
static __device__ __noinline__ float demap_qam_group_fallback(float yd, float inv_n0, const float* lev, int H, int u, int g,
                                                             float s_ok, float mx) {
    const int L = 1 << H, sh = H - 1 - u;
    float mg = -INFINITY, m2 = -INFINITY;                           // largest and second largest exponent of the group
    for (int t = 0; t < L; ++t) {
        if (((t >> sh) & 1) != g) continue;
        const float dd = __fsub_rn(yd, lev[t]);
        const float e = __fmul_rn(-__fmul_rn(dd, dd), inv_n0);
        m2 = fmaxf(m2, fminf(mg, e));
        mg = fmaxf(mg, e);
    }
    const bool finite = mg > -INFINITY && mg < INFINITY;
    mg = finite ? mg : 0.f;
    float sg = 1.f;
    // High SNR: every other member is below exp(-21) of the group's maximum. At most 15 such terms sum to < 2^-25, so the
    // reference's fp32 sum (ascending t, the maximum contributes exp(0) == 1) rounds to exactly 1 and its log to 0. Only
    // for a finite maximum: a group whose exponents are all -inf (no = 0 far from every level) sums to 0, log -inf.
    if (!(finite && __fsub_rn(m2, mg) < -21.f)) {
        sg = 0.f;
        for (int t = 0; t < L; ++t) {                               // ascending t inside the group
            if (((t >> sh) & 1) != g) continue;
            const float dd = __fsub_rn(yd, lev[t]);
            const float a = __fsub_rn(__fmul_rn(-__fmul_rn(dd, dd), inv_n0), mg);
            sg = __fadd_rn(sg, a < -87.3f ? 0.f : sb_expf(a));
        }
    }
    const float lg = __fadd_rn(sg > 0.f ? sb_logf(sg) : -INFINITY, mg);
    // s_ok == 0 only when every exponent of the dimension is -inf: then both groups are log(0) and the LLR is NaN
    const float lo = __fadd_rn(s_ok > 0.f ? sb_logf(s_ok) : -INFINITY, mx);
    return g ? __fsub_rn(lg, lo) : __fsub_rn(lo, lg);
}

// One dimension (d = 0 real, 1 imaginary) of one symbol. METHOD 0 = app, 1 = maxlog; H = bits per dimension.
// `lev(t)`: level t of this dimension (registers or constant bank); `lev_mem`: the same 2^H levels in addressable memory
// (only read by the fallback); inv_n0 = 1 / max(no, tiny); out[u] for bit u of the dimension.
template <int METHOD, int H, class Lev>
__device__ __forceinline__ void demap_qam_dim(float yd, float inv_n0, const Lev& lev, const float* lev_mem, int hard_out,
                                              float* out) {
    constexpr int L = 1 << H;
    float e[L];
#pragma unroll
    for (int t = 0; t < L; ++t) {
        const float dd = __fsub_rn(yd, lev(t));
        e[t] = __fmul_rn(-__fmul_rn(dd, dd), inv_n0);
    }
    // "app": exponentials relative to the LARGEST exponent of the dimension, evaluated once (L exps) and shared by the
    // H bits of the dimension: LLR = log(sum_{bit=1} w_t) - log(sum_{bit=0} w_t), the maximum cancels. The reference's
    // per-group logsumexp is the same number up to rounding as long as neither group's sum is tiny (fallback above).
    float wgt[L];
    float mx = -INFINITY;
    if (METHOD == 0 && H > 1) {
#pragma unroll
        for (int t = 0; t < L; ++t) mx = fmaxf(mx, e[t]);
        mx = (mx > -INFINITY && mx < INFINITY) ? mx : 0.f;
#pragma unroll
        for (int t = 0; t < L; t += 2) {
            const float a0 = __fsub_rn(e[t], mx), a1 = __fsub_rn(e[t + 1], mx);
            const float2 r = sb_expf2_inrange(make_float2(fmaxf(a0, -87.3f), fmaxf(a1, -87.3f)));
            wgt[t] = a0 < -87.3f ? 0.f : r.x;
            wgt[t + 1] = a1 < -87.3f ? 0.f : r.y;
        }
    }
#pragma unroll
    for (int u = 0; u < H; ++u) {
        float l;
        // H == 1 (QPSK / BPSK per dimension): each group has ONE member, logsumexp of one value is the value itself
        // (sb_expf(0) == 1 and sb_logf(1) == 0 exactly), so "app" equals "maxlog" bit for bit without exp / log
        if (METHOD == 1 || H == 1) {
            float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
            for (int t = 0; t < L; ++t) {
                if ((t >> (H - 1 - u)) & 1) mx1 = fmaxf(mx1, e[t]);
                else mx0 = fmaxf(mx0, e[t]);
            }
            l = __fsub_rn(mx1, mx0);
        } else {
            float s0 = 0.f, s1 = 0.f;
#pragma unroll
            for (int t = 0; t < L; ++t) {                           // ascending t inside each group
                if ((t >> (H - 1 - u)) & 1) s1 = __fadd_rn(s1, wgt[t]);
                else s0 = __fadd_rn(s0, wgt[t]);
            }
            // The group holding mx sums to >= 1. The other one may have lost members flushed at e_t - mx < -87.3; they
            // matter only if they are not negligible next to that group's own maximum e_g. With a shared sum
            // s >= DEMAP_QAM_GROUP_MIN = 2^-92 and at most 2^(H-1) <= 16 members in it, exp(e_g - mx) >= 2^-96, i.e.
            // e_g - mx >= -66.5, so every flushed member lies more than 20.7 below e_g, and the at most 15 of them add
            // < 15 e^-20.7 < 2^-26 to the group's sum relative to its maximum: below fp32 rounding of the log.
            // Smaller sums take the per-group path.
            if (fminf(s0, s1) >= DEMAP_QAM_GROUP_MIN) {
                const float2 lg = sb_logf2(make_float2(s0, s1));
                l = __fsub_rn(lg.y, lg.x);
            } else {
                const bool ok1 = s1 >= DEMAP_QAM_GROUP_MIN;
                l = demap_qam_group_fallback(yd, inv_n0, lev_mem, H, u, ok1 ? 0 : 1, ok1 ? s1 : s0, mx);
            }
        }
        out[u] = hard_out ? (l > 0.f ? 1.f : 0.f) : l;
    }
}

// Both dimensions with the levels in registers (lr / li) and in memory (lev_re / lev_im); out[2 * u + d].
template <int METHOD, int H>
__device__ __forceinline__ void demap_qam_symbol(float2 yy, float inv_n0, const float* lr, const float* li,
                                                 const float* lev_re, const float* lev_im, int hard_out, float* out) {
    struct RegLev {
        const float* v;
        __device__ __forceinline__ float operator()(int t) const { return v[t]; }
    };
    float o[2][H];
    demap_qam_dim<METHOD, H>(yy.x, inv_n0, RegLev{lr}, lev_re, hard_out, o[0]);
    demap_qam_dim<METHOD, H>(yy.y, inv_n0, RegLev{li}, lev_im, hard_out, o[1]);
#pragma unroll
    for (int u = 0; u < H; ++u) { out[2 * u] = o[0][u]; out[2 * u + 1] = o[1][u]; }
}
