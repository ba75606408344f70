// lmmse_diag.cuh -- LMMSE (and ZF / MF: zf_diag_solve, mf_diag_solve) equalisation of one resource element whose
// interference-plus-noise covariance S is diagonal (no interfering streams): everything lives in registers. Shared by
// the OFDM equaliser kernel (ofdm_mimo.cu) and the fused receive front-end (frontend.cu), so both run the same
// arithmetic.
//   input : B = H_w^H H_w (K x K Hermitian, lower triangle, row a holds (a, 0..a), zeroed by lmmse_diag_clear) and
//           z = H_w^H y_w of the WHITENED channel H_w = S^-1/2 H, y_w = S^-1/2 y
//   A = B + I = C C^H, A^-1 = C^-H C^-1;  G y_w = A^-1 z;  diag(G H_w)_k = sum_j (A^-1)_kj B_jk
//   output: x_hat_k = (G y_w)_k / diag_k, no_eff_k = Re(1 / diag_k - 1)     (mimo/equalization.py:217-231)
#pragma once
#include "sb_common.h"

namespace sb_lmmse {
template <int K>
__device__ __forceinline__ void lmmse_diag_clear(float2* Bm, float2* z) {
#pragma unroll
    for (int e = 0; e < K * (K + 1) / 2; ++e) Bm[e] = make_float2(0.f, 0.f);
#pragma unroll
    for (int k = 0; k < K; ++k) z[k] = make_float2(0.f, 0.f);
}

// C (packed lower triangle of a Hermitian positive-definite K x K matrix, row a holds (a, 0..a)) -> its Cholesky factor
// in place, Ci = that factor's inverse (lower, packed)
template <int K>
__device__ __forceinline__ void chol_inv_packed(float2* C, float2* Ci) {
#pragma unroll
    for (int j = 0; j < K; ++j) {
        float dj = C[j * (j + 1) / 2 + j].x;
#pragma unroll
        for (int k = 0; k < j; ++k) { float2 l = C[j * (j + 1) / 2 + k]; dj -= l.x * l.x + l.y * l.y; }
        dj = sqrtf(dj);
        C[j * (j + 1) / 2 + j] = make_float2(dj, 0.f);
#pragma unroll
        for (int r = j + 1; r < K; ++r) {
            float2 v = C[r * (r + 1) / 2 + j];
#pragma unroll
            for (int k = 0; k < j; ++k) v = csub(v, cmulc(C[r * (r + 1) / 2 + k], C[j * (j + 1) / 2 + k]));
            C[r * (r + 1) / 2 + j] = make_float2(v.x / dj, v.y / dj);
        }
    }
    // Ci = C^-1 (lower), column by column
#pragma unroll
    for (int c = 0; c < K; ++c) {
#pragma unroll
        for (int r = c; r < K; ++r) {
            float2 v = make_float2(r == c ? 1.f : 0.f, 0.f);
#pragma unroll
            for (int k = c; k < r; ++k) v = csub(v, cmul(C[r * (r + 1) / 2 + k], Ci[k * (k + 1) / 2 + c]));
            float dr = C[r * (r + 1) / 2 + r].x;
            Ci[r * (r + 1) / 2 + c] = make_float2(v.x / dr, v.y / dr);
        }
    }
}

// (A^-1)_kj = sum_{r >= max(k, j)} conj(Ci[r, k]) Ci[r, j] for A^-1 = C^-H C^-1, Ci = C^-1 packed
template <int K>
__device__ __forceinline__ float2 packed_inv_entry(const float2* Ci, int k, int j) {
    float2 ainv = make_float2(0.f, 0.f);
#pragma unroll
    for (int r = (k > j ? k : j); r < K; ++r) ainv = cadd(ainv, cmulc(Ci[r * (r + 1) / 2 + j], Ci[r * (r + 1) / 2 + k]));
    return ainv;
}

// The LMMSE solve keeps its own copy of the factorisation and inversion below (the same steps as chol_inv_packed):
// calling the helper instead changes the K = 1 kernels' instruction schedule and their results in the last bits.
template <int K>
__device__ __forceinline__ void lmmse_diag_solve(const float2* Bm, const float2* z, float2* xh, float* ne) {
    // A = B + I = C C^H (lower, in registers)
    float2 C[K * (K + 1) / 2];
#pragma unroll
    for (int e = 0; e < K * (K + 1) / 2; ++e) C[e] = Bm[e];
#pragma unroll
    for (int a = 0; a < K; ++a) C[a * (a + 1) / 2 + a].x += 1.f;
#pragma unroll
    for (int j = 0; j < K; ++j) {
        float dj = C[j * (j + 1) / 2 + j].x;
#pragma unroll
        for (int k = 0; k < j; ++k) { float2 l = C[j * (j + 1) / 2 + k]; dj -= l.x * l.x + l.y * l.y; }
        dj = sqrtf(dj);
        C[j * (j + 1) / 2 + j] = make_float2(dj, 0.f);
#pragma unroll
        for (int r = j + 1; r < K; ++r) {
            float2 v = C[r * (r + 1) / 2 + j];
#pragma unroll
            for (int k = 0; k < j; ++k) v = csub(v, cmulc(C[r * (r + 1) / 2 + k], C[j * (j + 1) / 2 + k]));
            C[r * (r + 1) / 2 + j] = make_float2(v.x / dj, v.y / dj);
        }
    }
    // Ci = C^-1 (lower), column by column
    float2 Ci[K * (K + 1) / 2];
#pragma unroll
    for (int c = 0; c < K; ++c) {
#pragma unroll
        for (int r = c; r < K; ++r) {
            float2 v = make_float2(r == c ? 1.f : 0.f, 0.f);
#pragma unroll
            for (int k = c; k < r; ++k) v = csub(v, cmul(C[r * (r + 1) / 2 + k], Ci[k * (k + 1) / 2 + c]));
            float dr = C[r * (r + 1) / 2 + r].x;
            Ci[r * (r + 1) / 2 + c] = make_float2(v.x / dr, v.y / dr);
        }
    }
#pragma unroll
    for (int k = 0; k < K; ++k) {
        // row k of A^-1 = C^-H C^-1: (A^-1)_kj = sum_{r >= max(k, j)} conj(Ci[r, k]) Ci[r, j]
        float2 gy = make_float2(0.f, 0.f), dd = make_float2(0.f, 0.f);
#pragma unroll
        for (int j = 0; j < K; ++j) {
            float2 ainv = make_float2(0.f, 0.f);
#pragma unroll
            for (int r = (k > j ? k : j); r < K; ++r)
                ainv = cadd(ainv, cmulc(Ci[r * (r + 1) / 2 + j], Ci[r * (r + 1) / 2 + k]));
            gy = cadd(gy, cmul(ainv, z[j]));
            // B_jk: stored lower triangle, B_jk = conj(B_kj)
            float2 bjk = j >= k ? Bm[j * (j + 1) / 2 + k] : make_float2(Bm[k * (k + 1) / 2 + j].x, -Bm[k * (k + 1) / 2 + j].y);
            dd = cadd(dd, cmul(ainv, bjk));
        }
        float2 inv = cdiv(make_float2(1.f, 0.f), dd);
        xh[k] = cdiv(gy, dd);
        ne[k] = inv.x - 1.f;
    }
}

// ZF without interferers, from B = H^H H, z = H^H y and C = H^H D H (packed lower triangles) of the unwhitened channel:
// x_hat = B^-1 z, no_eff_k = u_k^H C u_k with u_k column k of B^-1 (= diag(G D G^H), G = B^-1 H^H, mimo/equalization.py:
// 316-342). u_k = conj(row k), so no_eff_k = sum_a C_aa |g_a|^2 + 2 Re sum_{a > b} g_a C_ab conj(g_b), g = row k.
template <int K>
__device__ __forceinline__ void zf_diag_solve(const float2* Bm, const float2* Cm, const float2* z, float2* xh, float* ne) {
    float2 C[K * (K + 1) / 2], Ci[K * (K + 1) / 2];
#pragma unroll
    for (int e = 0; e < K * (K + 1) / 2; ++e) C[e] = Bm[e];
    chol_inv_packed<K>(C, Ci);
#pragma unroll
    for (int k = 0; k < K; ++k) {
        float2 g[K], gy = make_float2(0.f, 0.f);
#pragma unroll
        for (int j = 0; j < K; ++j) {
            g[j] = packed_inv_entry<K>(Ci, k, j);
            gy = cadd(gy, cmul(g[j], z[j]));
        }
        float dg = 0.f, off = 0.f;
#pragma unroll
        for (int a = 0; a < K; ++a) {
            dg += Cm[a * (a + 1) / 2 + a].x * (g[a].x * g[a].x + g[a].y * g[a].y);
            float2 t = make_float2(0.f, 0.f);
#pragma unroll
            for (int b = 0; b < a; ++b) t = cadd(t, cmulc(Cm[a * (a + 1) / 2 + b], g[b]));
            off += g[a].x * t.x - g[a].y * t.y;
        }
        xh[k] = gy;
        ne[k] = dg + 2.f * off;
    }
}

// MF without interferers, from B = H^H H, z = H^H y (packed lower) and the diagonal Cd[k].x = (H^H D H)_kk:
// x_hat_k = z_k / B_kk, no_eff_k = (sum_{j != k} |B_kj|^2 + (H^H D H)_kk) / B_kk^2 (mimo/equalization.py:437-464)
template <int K>
__device__ __forceinline__ void mf_diag_solve(const float2* Bm, const float2* Cd, const float2* z, float2* xh, float* ne) {
#pragma unroll
    for (int k = 0; k < K; ++k) {
        float off = 0.f;
#pragma unroll
        for (int j = 0; j < K; ++j) {
            if (j == k) continue;
            const float2 b = j < k ? Bm[k * (k + 1) / 2 + j] : Bm[j * (j + 1) / 2 + k];
            off += b.x * b.x + b.y * b.y;
        }
        const float inv = 1.f / Bm[k * (k + 1) / 2 + k].x;
        xh[k] = cscale(z[k], inv);
        ne[k] = fabsf((off + Cd[k].x) * inv * inv);
    }
}
}  // namespace sb_lmmse
