// dense_mimo.cuh -- per-vector dense linear algebra and the OFDM per-resource-element problem assembly shared by the LMMSE
// kernels (ofdm_mimo.cu) and the maximum-likelihood and K-Best detectors (mimo_ml.cu, mimo_kbest.cu), so all whiten
// with the same arithmetic.
//   Scratch          per-thread view of a shared-memory matrix, interleaved by thread (element e of thread t at
//                    [e * T + t]: conflict-free); scratch_threads sizes the CTA
//   chol_lower       L = chol(S), in place                                   (utils/linalg.py:28-32)
//   whiten           y_w = L^-1 y, H_w = L^-1 H                              (mimo/utils.py:343-347)
//   qr_record        modified Gram-Schmidt of [H_w | y_w] in a given column order: R, Q^H y_w, out-of-span term
//   OfdmEqParams     OFDMEqualizer's inputs and stream-management tables (ofdm/equalization.py:109-275)
//   ofdm_re / ofdm_load_re / ofdm_out_index   addressing of one resource element, S = H_u H_u^H + diag(no) +
//                    diag(sum err_var) assembly (equalization.py:205-218), output position of stream k
#pragma once
#include "sb_common.h"

namespace sb_dense {

struct Scratch {
    float2* p;
    int T, t;
    __device__ __forceinline__ float2& operator()(int e) const { return p[(size_t)e * T + t]; }
};

// A = L L^H (lower, n x n), in place
static __device__ void chol_lower(const Scratch& A, int n) {
    for (int j = 0; j < n; ++j) {
        float d = A(j * n + j).x;
        for (int k = 0; k < j; ++k) { float2 l = A(j * n + k); d -= l.x * l.x + l.y * l.y; }
        d = sqrtf(d);
        A(j * n + j) = make_float2(d, 0.f);
        for (int i = j + 1; i < n; ++i) {
            float2 v = A(i * n + j);
            for (int k = 0; k < j; ++k) v = csub(v, cmulc(A(i * n + k), A(j * n + k)));
            A(i * n + j) = make_float2(v.x / d, v.y / d);
        }
    }
}

// forward substitution with the Cholesky factor L (M x M), in place: Y = L^-1 Y (M), H = L^-1 H (M x K)
static __device__ void whiten(const Scratch& L, const Scratch& Y, const Scratch& H, int M, int K) {
    for (int i = 0; i < M; ++i) {
        float d = L(i * M + i).x;
        float2 v = Y(i);
        for (int k = 0; k < i; ++k) v = csub(v, cmul(L(i * M + k), Y(k)));
        Y(i) = make_float2(v.x / d, v.y / d);
        for (int c = 0; c < K; ++c) {
            float2 w = H(i * K + c);
            for (int k = 0; k < i; ++k) w = csub(w, cmul(L(i * M + k), H(k * K + c)));
            H(i * K + c) = make_float2(w.x / d, w.y / d);
        }
    }
}

// Modified Gram-Schmidt on the whitened [H | y] with the columns of H taken in the order col(0), col(1), ... (H: M x K
// in scratch, column col(j) overwritten by q_j), record: R [K, K] row-major in that order, yq = Q^H y [K], the
// out-of-span term c0 = ||y - Q yq||^2 in rec[K^2 + K].x. Columns j >= M (or numerically dependent ones) get R_jj = 0
// and a zero q_j. col is a functor so that the identity order compiles to plain indexing.
template <class Col>
static __device__ void qr_record(const Scratch& Y, const Scratch& H, int M, int K, Col col, float2* __restrict__ rec) {
    for (int j = 0; j < K; ++j) {
        const int cj = col(j);
        for (int r = 0; r < j; ++r) {
            const int cr = col(r);
            float2 a = make_float2(0.f, 0.f);
            for (int m = 0; m < M; ++m) a = cadd(a, cmulc(H(m * K + cj), H(m * K + cr)));   // q_r^H h_j
            for (int m = 0; m < M; ++m) H(m * K + cj) = csub(H(m * K + cj), cmul(H(m * K + cr), a));
            rec[r * K + j] = a;
        }
        for (int r = j + 1; r < K; ++r) rec[r * K + j] = make_float2(0.f, 0.f);
        float n2 = 0.f;
        for (int m = 0; m < M; ++m) { float2 v = H(m * K + cj); n2 += v.x * v.x + v.y * v.y; }
        const float nrm = sqrtf(n2);
        const bool keep = j < M && nrm > 0.f;
        const float inv = keep ? 1.f / nrm : 0.f;
        rec[j * K + j] = make_float2(keep ? nrm : 0.f, 0.f);
        for (int m = 0; m < M; ++m) H(m * K + cj) = cscale(H(m * K + cj), inv);
    }
    for (int r = 0; r < K; ++r) {
        const int cr = col(r);
        float2 a = make_float2(0.f, 0.f);
        for (int m = 0; m < M; ++m) a = cadd(a, cmulc(Y(m), H(m * K + cr)));
        for (int m = 0; m < M; ++m) Y(m) = csub(Y(m), cmul(H(m * K + cr), a));
        rec[K * K + r] = a;
    }
    float c0 = 0.f;
    for (int m = 0; m < M; ++m) { float2 v = Y(m); c0 += v.x * v.x + v.y * v.y; }
    rec[K * K + K] = make_float2(c0, 0.f);
}

// Threads per CTA of a thread-per-vector scratch kernel: per_thread bytes of shared memory each and at most cap bytes in
// all. At most 128 and a multiple of 32 when a warp fits; otherwise the largest power of two that fits (16 ... 1), so
// large matrices still run, at low occupancy. 0 if not even one thread fits.
static inline int scratch_threads(size_t per_thread, size_t cap, size_t* smem) {
    const int fit = (int)std::min<size_t>(128, cap / per_thread);
    int t = fit / 32 * 32;
    if (t == 0)
        for (t = 16; t > fit; t /= 2) {}
    if (t == 0) return 0;
    *smem = per_thread * t;
    return t;
}

// OFDMEqualizer inputs. Per (b, rx, sym, sc):
//   y    [B, RX, ANT, S, F]          (effective subcarriers only)
//   hhat [B, RX, ANT, TXS, S, F]     TXS = num_tx * num_streams_per_tx
//   ev   err_var with strides given by ev_stride[6] elements for dims (b, rx, ant, txs, s, f) (0 = broadcast)
//   no   [B, RX, ANT] via no_stride (b, rx, ant)
//   des [RX, K], und [RX, KU]: TXS indices of the desired / interfering streams of receiver rx
//   out_ts [RX, K]: output stream row (tx*streams + st) after stream_ind re-ordering; data_pos [TXS, S*F]: position among
//   the data symbols of that stream or -1 -> outputs [B, TXS, num_data, ...]
struct OfdmEqParams {
    const float2* y; const float2* hhat; const float* ev; const float* no;
    long long ev_stride[6]; long long no_stride[3];
    const int* des; const int* und; const int* out_ts; const int* data_pos;
    float2* xh; float* ne;
    long long B; int RX, ANT, TXS, S, F, K, KU, ND;
};

// resource element i of the flattened (b, rx, symbol, subcarrier) grid
struct OfdmRe {
    long long b, re;
    int rx, s, f;
};
__device__ __forceinline__ OfdmRe ofdm_re(const OfdmEqParams& p, long long i) {
    const long long SF = (long long)p.S * p.F;
    OfdmRe e;
    e.re = i % SF;
    e.rx = (int)((i / SF) % p.RX);
    e.b = i / (SF * p.RX);
    e.s = (int)(e.re / p.F);
    e.f = (int)(e.re % p.F);
    return e;
}

// output position (b * TXS + ts) * ND + dp of the k-th stream of the element's receiver, -1 if that stream carries no
// data there
__device__ __forceinline__ long long ofdm_out_index(const OfdmEqParams& p, const OfdmRe& e, int k) {
    const long long SF = (long long)p.S * p.F;
    const int ts = p.out_ts[e.rx * p.K + k];
    const int dp = p.data_pos[(size_t)ts * SF + e.re];
    return dp >= 0 ? (e.b * p.TXS + ts) * (long long)p.ND + dp : -1;
}

// true if the element carries data for at least one of its receiver's streams
__device__ __forceinline__ bool ofdm_re_has_data(const OfdmEqParams& p, const OfdmRe& e) {
    const long long SF = (long long)p.S * p.F;
    bool any = false;
    for (int k = 0; k < p.K; ++k) any = any || p.data_pos[(size_t)p.out_ts[e.rx * p.K + k] * SF + e.re] >= 0;
    return any;
}

// Y = y [M], H = desired channel columns [M, K], lower triangle of S = H_u H_u^H + diag(no) + diag(sum_txs err_var)
// (equalization.py:205-218)
__device__ __forceinline__ void ofdm_load_re(const OfdmEqParams& p, const OfdmRe& e, const Scratch& Y, const Scratch& H,
                                             const Scratch& S) {
    const long long SF = (long long)p.S * p.F;
    const int M = p.ANT, K = p.K;
    const long long b = e.b, re = e.re;
    const int rx = e.rx, s = e.s, f = e.f;
    for (int m = 0; m < M; ++m) {
        long long ybase = ((b * p.RX + rx) * M + m) * SF + re;
        Y(m) = p.y[ybase];
        long long hb = ((b * p.RX + rx) * M + m) * (long long)p.TXS;
        for (int k = 0; k < K; ++k) H(m * K + k) = p.hhat[(hb + p.des[rx * K + k]) * SF + re];
        float evs = 0.f;
        for (int q = 0; q < p.TXS; ++q)
            evs += p.ev[b * p.ev_stride[0] + rx * p.ev_stride[1] + m * p.ev_stride[2] + q * p.ev_stride[3] +
                        s * p.ev_stride[4] + f * p.ev_stride[5]];
        float nn = p.no[b * p.no_stride[0] + rx * p.no_stride[1] + m * p.no_stride[2]];
        for (int m2 = 0; m2 <= m; ++m2) {
            float2 acc = make_float2(0.f, 0.f);
            long long hb2 = ((b * p.RX + rx) * M + m2) * (long long)p.TXS;
            for (int u = 0; u < p.KU; ++u)
                acc = cadd(acc, cmulc(p.hhat[(hb + p.und[rx * p.KU + u]) * SF + re],
                                      p.hhat[(hb2 + p.und[rx * p.KU + u]) * SF + re]));
            if (m2 == m) acc.x += nn + evs;
            S(m * M + m2) = acc;
        }
    }
}

}  // namespace sb_dense
