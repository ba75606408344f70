// dense_mimo.cuh -- per-vector dense linear algebra, the OFDM per-resource-element problem assembly and the front half
// of the MIMO detectors, shared by the LMMSE kernels (ofdm_mimo.cu), the ML, K-Best, EP and MMSE-PIC detectors
// (mimo_ml.cu, mimo_kbest.cu, mimo_iterative.cu) and the precoders (precoding.cu), so all whiten and solve with the
// same arithmetic.
//   Scratch          per-thread view of a shared-memory matrix, interleaved by thread (element e of thread t at
//                    [e * T + t]: conflict-free; ScratchOf<float> for real matrices); scratch_threads sizes the CTA,
//                    detector_threads also under kScratchSmemCap with the error message
//   chol_lower       L = chol(S), in place                                   (utils/linalg.py:28-32)
//   chol_solve_col   one column of (L L^H)^-1 B                              (tf.linalg.cholesky_solve)
//   whiten           y_w = L^-1 y, H_w = L^-1 H                              (mimo/utils.py:343-347)
//   qr_record        modified Gram-Schmidt of [H_w | y_w] in a given column order: R, Q^H y_w, out-of-span term
//                    (qr_record_size float2)
//   pam2qam_index    QAM label of a pair of PAM labels                       (mapping.py:1234-1320)
//   OfdmEqParams     OFDMEqualizer's inputs and stream-management tables (ofdm/equalization.py:109-275)
//   ofdm_re / ofdm_load_re / ofdm_out_index   addressing of one resource element, S = H_u H_u^H + diag(no) +
//                    diag(sum err_var) assembly (equalization.py:205-218), output position of stream k
//   MimoProblem / load_whitened   a detector's dense or OFDM problem set; problem i loaded, whitened and given its
//                    output positions. dense_problem / ofdm_problem build the set from the C-ABI arguments,
//                    ofdm_check tests the OFDM detectors' pointer arguments
#pragma once
#include "sb_common.h"

namespace sb_dense {

template <class E>
struct ScratchOf {
    E* p;
    int T, t;
    __device__ __forceinline__ E& operator()(int e) const { return p[(size_t)e * T + t]; }
};
using Scratch = ScratchOf<float2>;

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

// solve (C C^H) x = b for one column, b_i = b(i), x_i in X(i * ldx + col); C lower triangular n x n. b may read the
// column being solved: b(i) is read before X(i * ldx + col) is written.
template <typename BF>
__device__ void chol_solve_col(const Scratch& C, int n, const BF& b, const Scratch& X, int ldx, int col) {
    for (int i = 0; i < n; ++i) {
        float2 v = b(i);
        for (int k = 0; k < i; ++k) v = csub(v, cmul(C(i * n + k), X(k * ldx + col)));
        float d = C(i * n + i).x;
        X(i * ldx + col) = make_float2(v.x / d, v.y / d);
    }
    for (int i = n - 1; i >= 0; --i) {
        float2 v = X(i * ldx + col);
        for (int k = i + 1; k < n; ++k) { float2 c = C(k * n + i); c.y = -c.y; v = csub(v, cmul(c, X(k * ldx + col))); }
        float d = C(i * n + i).x;
        X(i * ldx + col) = make_float2(v.x / d, v.y / d);
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

// float2 per qr_record of K columns: R [K, K], yq [K], c0
__host__ __device__ constexpr int qr_record_size(int K) { return K * K + K + 1; }

// QAM label of the PAM label pair (re, im) of a QAM with m bits per symbol (m even): re on the even label bits, MSB
// first (PAM2QAM)
__device__ __forceinline__ int pam2qam_index(int re, int im, int m) {
    const int h = m >> 1;
    int idx = 0;
    for (int j = 0; j < h; ++j)
        idx |= (((re >> (h - 1 - j)) & 1) << (m - 1 - 2 * j)) | (((im >> (h - 1 - j)) & 1) << (m - 2 - 2 * j));
    return idx;
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

// dynamic shared memory per CTA of the scratch kernels
constexpr size_t kScratchSmemCap = 200 * 1024;

// CTA size of a detector kernel with per_thread bytes of scratch after fixed bytes per CTA, *smem = its shared memory;
// 0 (with an error message naming who) if not even one thread fits
static inline int detector_threads(const char* who, size_t fixed, size_t per_thread, int M, int K, size_t* smem) {
    const int th = scratch_threads(per_thread, kScratchSmemCap - fixed, smem);
    if (!th)
        sb_set_error("%s: M = %d, K = %d needs %zu bytes of shared-memory scratch per problem, the limit is %zu", who, M,
                     K, per_thread, kScratchSmemCap - fixed);
    *smem += fixed;
    return th;
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

// A detector's problem set: P dense problems (y [P, M], h [P, M, K], s [P, M, M]) or, is_ofdm, the P resource elements
// of an OFDM grid (problem i = element i of the flattened (b, rx, symbol, subcarrier) grid, M = ANT)
struct MimoProblem {
    const float2* y; const float2* h; const float2* s;  // dense inputs (is_ofdm = 0)
    OfdmEqParams ofdm;
    int is_ofdm;
    long long P;
    int M, K;
};

// Loads problem i into S [M, M], H [M, K], Y [M] and writes the output position of stream k to oi[k] (dense: i K + k;
// OFDM: ofdm_out_index, -1 where the stream carries no data). False for an OFDM element that carries no data for any
// stream; otherwise S -> L = chol(S), Y = L^-1 y, H = L^-1 H.
static __device__ bool load_whitened(const MimoProblem& q, long long i, const Scratch& S, const Scratch& H,
                                     const Scratch& Y, long long* oi) {
    const int M = q.M, K = q.K;
    if (q.is_ofdm) {
        const OfdmRe e = ofdm_re(q.ofdm, i);
        bool any = false;
        for (int k = 0; k < K; ++k) {
            oi[k] = ofdm_out_index(q.ofdm, e, k);
            any = any || oi[k] >= 0;
        }
        if (!any) return false;
        ofdm_load_re(q.ofdm, e, Y, H, S);
    } else {
        for (int k = 0; k < K; ++k) oi[k] = i * K + k;
        for (int e = 0; e < M * M; ++e) S(e) = q.s[i * M * M + e];
        for (int e = 0; e < M * K; ++e) H(e) = q.h[i * M * K + e];
        for (int e = 0; e < M; ++e) Y(e) = q.y[i * M + e];
    }
    chol_lower(S, M);
    whiten(S, Y, H, M, K);
    return true;
}

static inline MimoProblem dense_problem(const float* y, const float* h, const float* s, long long num, int M, int K) {
    MimoProblem pb{};
    pb.y = (const float2*)y; pb.h = (const float2*)h; pb.s = (const float2*)s;
    pb.is_ofdm = 0; pb.P = num; pb.M = M; pb.K = K;
    return pb;
}

// The OFDM C-ABI arguments (sb_ofdm_lmmse and the sb_ofdm_* detectors) as a problem set; ofdm.xh and ofdm.ne are unset
static inline MimoProblem ofdm_problem(const float* d_y, const float* d_h_hat, const float* d_err_var,
                                       const int64_t* h_ev_stride, const float* d_no, const int64_t* h_no_stride,
                                       const int32_t* d_desired, const int32_t* d_undesired,
                                       const int32_t* d_out_stream, const int32_t* d_data_pos, int64_t batch,
                                       int num_rx, int num_rx_ant, int num_tx_streams, int num_symbols,
                                       int num_subcarriers, int streams_per_rx, int interferers_per_rx, int num_data) {
    MimoProblem pb{};
    OfdmEqParams& p = pb.ofdm;
    p.y = (const float2*)d_y; p.hhat = (const float2*)d_h_hat; p.ev = d_err_var; p.no = d_no;
    for (int i = 0; i < 6; ++i) p.ev_stride[i] = h_ev_stride[i];
    for (int i = 0; i < 3; ++i) p.no_stride[i] = h_no_stride[i];
    p.des = d_desired; p.und = d_undesired; p.out_ts = d_out_stream; p.data_pos = d_data_pos;
    p.B = batch; p.RX = num_rx; p.ANT = num_rx_ant; p.TXS = num_tx_streams;
    p.S = num_symbols; p.F = num_subcarriers; p.K = streams_per_rx; p.KU = interferers_per_rx; p.ND = num_data;
    pb.is_ofdm = 1;
    pb.P = batch * num_rx * (long long)num_symbols * num_subcarriers;
    pb.M = num_rx_ant;
    pb.K = streams_per_rx;
    return pb;
}

// Pointer arguments of an sb_ofdm_* detector with a non-empty batch: SB_EINVAL ("who: bad arguments") unless every input,
// table, the constellation and the output are given (d_undesired only with interferers) and num_rx_ant >= 1
static inline int ofdm_check(const char* who, const float* d_y, const float* d_h_hat, const float* d_err_var,
                             const int64_t* h_ev_stride, const float* d_no, const int64_t* h_no_stride,
                             const int32_t* d_desired, const int32_t* d_undesired, const int32_t* d_out_stream,
                             const int32_t* d_data_pos, const float* d_points, const void* d_out, int64_t batch,
                             int num_rx_ant, int interferers_per_rx) {
    SB_CHECK_ARG(d_y && d_h_hat && d_err_var && h_ev_stride && d_no && h_no_stride && d_desired && d_out_stream &&
                     d_data_pos && d_points && d_out && batch > 0 && num_rx_ant >= 1 &&
                     (interferers_per_rx == 0 || d_undesired),
                 "%s: bad arguments", who);
    return SB_OK;
}

}  // namespace sb_dense
