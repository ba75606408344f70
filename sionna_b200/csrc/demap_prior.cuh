// demap_prior.cuh -- LLRs of ONE received symbol for any constellation, with optional bit priors, shared by the
// stand-alone demapper kernel (phy_kernels.cu, sb_demap) and the MMSE-PIC detector (mimo_iterative.cu).
// Reference: Demapper.call + SymbolLogits2LLRs.call, /root/reference/src/sionna/phy/mapping.py:664-691, 927-967.
// Every operation is an explicit IEEE-754 RN intrinsic or an sb_math.h function, so the result does not depend on the
// translation unit's -fmad setting and the CPU oracle (oracle/mapping_ref.c) reproduces it bit for bit.
#pragma once
#include "sb_math.h"
#include "sb_math2.cuh"

// log_sigmoid(x) = -softplus(-x) with TensorFlow's softplus branches (threshold = log(eps) + 2)
__device__ __forceinline__ float log1p_pos(float u) {   // u >= 0
    float w = __fadd_rn(1.f, u);
    if (w == 1.f) return u;
    return __fmul_rn(sb_logf(w), __fdiv_rn(u, __fsub_rn(w, 1.f)));
}
__device__ __forceinline__ float softplusf(float x) {
    const float threshold = -13.942385f;   // logf(FLT_EPSILON) + 2
    if (x > -threshold) return x;
    float ex = sb_expf(x);
    if (x < threshold) return ex;
    return log1p_pos(ex);
}
__device__ __forceinline__ float log_sigmoidf(float x) { return -softplusf(-x); }

// Exponent of point j with label bits MSB first: e_j = -|y - c_j|^2 / n0 (+ sum_k log_sigmoid(+-prior_k), ls1 / ls0 =
// log_sigmoid(prior) / log_sigmoid(-prior) per label bit). With the exponent term dropped this prior sum is
// LLRs2SymbolLogits (mapping.py:1045-1059).
template <int M>
__device__ __forceinline__ float demap_prior_logit(const float* ls1, const float* ls0, int j) {
    float ps = 0.f;
#pragma unroll
    for (int k = 0; k < M; ++k) ps = __fadd_rn(ps, ((j >> (M - 1 - k)) & 1) ? ls1[k] : ls0[k]);
    return ps;
}
template <int M>
__device__ __forceinline__ float demap_exponent(float2 yy, float2 c, float n0, const float* ls1, const float* ls0, int j,
                                                bool with_prior) {
    float dr = __fsub_rn(yy.x, c.x), di = __fsub_rn(yy.y, c.y);
    float a = __fsqrt_rn(__fmaf_rn(dr, dr, __fmul_rn(di, di)));     // |y - c|  (tf.abs)
    float e = __fdiv_rn(-__fmul_rn(a, a), n0);                       // -|.|^2 / no
    if (with_prior) e = __fadd_rn(demap_prior_logit<M>(ls1, ls0, j), e);
    return e;
}

// out[i] = LLR of label bit i of the symbol yy received with noise variance n0 (> 0) over the 2^M points pts.
// Exponents are evaluated once per pass and feed all 2M groups {points with bit i = v} at the same time:
//   pass 1: group maxima (METHOD 1, maxlog: done);  pass 2 (METHOD 0, app): sum_j exp(e_j - max_group) per group, two
//   groups per packed FP32x2 exp (sb_math2.cuh, bit-identical to sb_expf); LLR_i = logsumexp(bit 1) - logsumexp(bit 0).
// Per group the operation order is the one of tf.reduce_logsumexp over the points in ascending label order.
template <int METHOD, int M>
__device__ __forceinline__ void demap_symbol(float2 yy, float n0, const float2* pts, const float* ls1, const float* ls0,
                                             bool with_prior, float* out) {
    constexpr int NPTS = 1 << M;
    float mx0[M], mx1[M];
#pragma unroll
    for (int i = 0; i < M; ++i) { mx0[i] = -INFINITY; mx1[i] = -INFINITY; }
#pragma unroll 4
    for (int j = 0; j < NPTS; ++j) {
        const float e = demap_exponent<M>(yy, pts[j], n0, ls1, ls0, j, with_prior);
#pragma unroll
        for (int i = 0; i < M; ++i) {                        // label bit i, MSB first (mapping.py:894-907)
            if ((j >> (M - 1 - i)) & 1) mx1[i] = fmaxf(mx1[i], e);
            else mx0[i] = fmaxf(mx0[i], e);
        }
    }
    if (METHOD == 1) {
#pragma unroll
        for (int i = 0; i < M; ++i) out[i] = __fsub_rn(mx1[i], mx0[i]);
    } else {
        // tf.reduce_logsumexp: log(sum(exp(x - max))) + max, max replaced by 0 if not finite
        float sm0[M], sm1[M];
#pragma unroll
        for (int i = 0; i < M; ++i) {
            mx0[i] = (mx0[i] > -INFINITY && mx0[i] < INFINITY) ? mx0[i] : 0.f;
            mx1[i] = (mx1[i] > -INFINITY && mx1[i] < INFINITY) ? mx1[i] : 0.f;
            sm0[i] = 0.f; sm1[i] = 0.f;
        }
#pragma unroll 2
        for (int j = 0; j < NPTS; ++j) {
            const float e = demap_exponent<M>(yy, pts[j], n0, ls1, ls0, j, with_prior);
            float t[M + 1];
#pragma unroll
            for (int i = 0; i < M; ++i) t[i] = __fsub_rn(e, ((j >> (M - 1 - i)) & 1) ? mx1[i] : mx0[i]);
            t[M] = 0.f;
#pragma unroll
            for (int i = 0; i < M; i += 2) {                 // exp of two groups at a time (sb_math2.cuh)
                float2 a = make_float2(fmaxf(t[i], -87.3f), fmaxf(t[i + 1], -87.3f));
                float2 r = sb_expf2_inrange(a);
                if (t[i] < -87.3f) r.x = 0.f;                // sb_expf: exact 0 below -87.3
                if (t[i + 1] < -87.3f) r.y = 0.f;
                t[i] = r.x;
                t[i + 1] = r.y;
            }
#pragma unroll
            for (int i = 0; i < M; ++i) {
                if ((j >> (M - 1 - i)) & 1) sm1[i] = __fadd_rn(sm1[i], t[i]);
                else sm0[i] = __fadd_rn(sm0[i], t[i]);
            }
        }
#pragma unroll
        for (int i = 0; i < M; ++i) {
            const float2 lg = sb_logf2(make_float2(fmaxf(sm0[i], 1.17549435e-38f), fmaxf(sm1[i], 1.17549435e-38f)));
            float a1 = __fadd_rn(sm1[i] > 0.f ? lg.y : -INFINITY, mx1[i]);
            float a0 = __fadd_rn(sm0[i] > 0.f ? lg.x : -INFINITY, mx0[i]);
            out[i] = __fsub_rn(a1, a0);
        }
    }
}
