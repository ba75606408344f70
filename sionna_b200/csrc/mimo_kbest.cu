// mimo_kbest.cu -- K-Best MIMO detection for sm_90a. Replaces (paths under /root/reference/src/sionna/phy/):
//   sb_mimo_kbest   KBestDetector.call   mimo/detection.py:539-1037 (+ complex2real_channel mimo/utils.py:194-242,
//                   List2LLRSimple mimo/utils.py:420-577, PAM2QAM mapping.py:1234-1320)
//   sb_ofdm_kbest   the same detector per OFDM resource element, with OFDMEqualizer's covariance
//                   S = H_u H_u^H + diag(no) + diag(sum err_var) assembled on chip (dense_mimo.cuh)
// The reference materialises [batch, k |C|, S] symbol and index tensors per layer and sorts them with top_k; here one
// warp keeps a problem's whole path list in shared memory and nothing per path leaves the chip.
//
// Two launches per call (as mimo_ml.cu: the prologue's scratch would otherwise cap the search's occupancy):
//   1. kbest_prologue_kernel, one thread per problem: y_w and H_w from the detectors' shared loader (load_whitened,
//      dense_mimo.cuh), the squared norm of every whitened column, the column order (descending norm, ties: lower index
//      first, an insertion sort), then the modified Gram-Schmidt of the sorted [H_w | y_w] (qr_record): R (upper
//      triangular, R_jj real >= 0) and ybar = Q^H y_w. The out-of-span term is dropped: every path metric shares it.
//      Real representation (real_rep = 1, QAM only): realify(S) / 2 = F F^T with F = realify(L) / sqrt(2), so the
//      whitened real channel is sqrt(2) [[Re H_w, -Im H_w], [Im H_w, Re H_w]] with y = sqrt(2) [Re y_w; Im y_w]. It is
//      the reference's whitened channel up to an orthogonal factor, which leaves every metric unchanged. Columns k and
//      K + k have the same norm; it is computed once per complex column, so k always sorts before K + k. The real
//      matrices are stored as float2 with a zero imaginary part, so one search kernel serves both representations.
//      Record (caller's workspace, sb_kbest_workspace_bytes): R [S, S], ybar [S], one unused slot (qr_record's layout),
//      the K output positions (int64) and the column order [S] (int32); S = K (complex) or 2 K (real) layers.
//   2. kbest_search_kernel, one warp per problem. Layers run from the last sorted stream to the first. Each kept path
//      carries its metric and the offset b = ybar_i - sum_{j > i} R_ij x_j of the next layer (O(S), once per path), so a
//      child costs 4 FMAs: d = parent + |b - R_ii x|^2. Child c = parent rank * |C| + point index (tf.repeat's layout).
//      The min(k, N) children with the smallest (metric, c) are kept, sorted ascending (tf.math.top_k(-d, sorted=True)
//      puts the lower index first on ties):
//        a) radix select over the metric's bits (metrics are >= 0, so their bits order as unsigned integers): 8-bit
//           digits from the top, a 256-bin histogram in shared memory per pass, children recomputed in every pass, until
//           the digit's bucket is taken whole or all 32 bits are fixed; equal metrics are then taken by index;
//        b) one pass compacts the selected children (ballot / popc, index order) as 64-bit keys (metric bits << 32 | c);
//        c) a warp bitonic sort of the keys, padded to a power of two.
//      Nothing is stored per child, so shared memory per problem depends on k and S only.
//      Finish step: hard decisions from path 0 (PAM2QAM interleaving in the real representation, SymbolInds2Bits for
//      bits) or List2LLRSimple over the kept paths (metrics halved in the real representation, clip to +-llr_clip), lanes
//      over (stream, bit) pairs, written straight into the caller's output layout.
#include "sb_common.h"
#include "dense_mimo.cuh"

namespace {

using sb_dense::Scratch;
using sb_dense::MimoProblem;
using sb_dense::qr_record_size;

constexpr int kKbMaxLayers = 16;
constexpr int kKbMaxK = 256;
constexpr int kKbMaxPoints = 256;
constexpr int kKbMaxChildren = 16384;

size_t kb_workspace_bytes(long long P, int K, int real_rep) {
    const int S = K << real_rep;
    return (sizeof(float2) * qr_record_size(S) + sizeof(long long) * K + sizeof(int) * S) * (size_t)P;
}

// One thread per problem (load_whitened, then the column order and qr_record); output positions to oidx [P, K].
// Scratch per thread: S [M, M], H [M, K], Y [M] and, real_rep, H_r [2M, 2K], Y_r [2M].
__global__ void kbest_prologue_kernel(const MimoProblem pb, int real_rep, float2* __restrict__ recs,
                                      long long* __restrict__ oidx, int* __restrict__ orders) {
    extern __shared__ float2 smem[];
    const int T = blockDim.x, t = threadIdx.x, M = pb.M, K = pb.K;
    const int S = K << real_rep, MR = M << real_rep;
    const size_t o_h = (size_t)M * M, o_y = o_h + (size_t)M * K, o_hr = o_y + M, o_yr = o_hr + (size_t)MR * S;
    const Scratch Sc{smem, T, t}, H{smem + o_h * T, T, t}, Y{smem + o_y * T, T, t};
    const Scratch HR{smem + o_hr * T, T, t}, YR{smem + o_yr * T, T, t};
    for (long long i = (long long)blockIdx.x * T + t; i < pb.P; i += (long long)gridDim.x * T) {
        if (!sb_dense::load_whitened(pb, i, Sc, H, Y, oidx + i * K)) continue;
        float nrm[kKbMaxLayers];
        for (int k = 0; k < K; ++k) {
            float n2 = 0.f;
            for (int m = 0; m < M; ++m) { const float2 v = H(m * K + k); n2 += v.x * v.x + v.y * v.y; }
            nrm[k] = n2;
        }
        int ord[kKbMaxLayers];                         // stable: a column moves ahead only past strictly smaller norms
        for (int d = 0; d < S; ++d) {
            const float nd = nrm[d % K];
            int j = d;
            for (; j > 0 && nrm[ord[j - 1] % K] < nd; --j) ord[j] = ord[j - 1];
            ord[j] = d;
        }
        for (int d = 0; d < S; ++d) orders[i * S + d] = ord[d];
        float2* rec = recs + i * qr_record_size(S);
        if (real_rep) {
            const float r2 = 1.41421356237309515f;
            for (int m = 0; m < M; ++m) {
                for (int k = 0; k < K; ++k) {
                    const float2 v = H(m * K + k);
                    HR(m * S + k) = make_float2(r2 * v.x, 0.f);
                    HR(m * S + K + k) = make_float2(-r2 * v.y, 0.f);
                    HR((M + m) * S + k) = make_float2(r2 * v.y, 0.f);
                    HR((M + m) * S + K + k) = make_float2(r2 * v.x, 0.f);
                }
                YR(m) = make_float2(r2 * Y(m).x, 0.f);
                YR(M + m) = make_float2(r2 * Y(m).y, 0.f);
            }
            sb_dense::qr_record(YR, HR, MR, S, [&](int j) { return ord[j]; }, rec);
        } else {
            sb_dense::qr_record(Y, H, M, K, [&](int j) { return ord[j]; }, rec);
        }
    }
}

struct KbParams {
    const float2* rec; const long long* oidx; const int* order; const void* points;
    void* out;
    long long P;
    int S, K, NP, lg, m, k, kpad, real_rep, symbol, hard;
    float clip;
    int per_warp;                                       // shared-memory bytes per warp
};

// child metric d = parent + |b - r_ii x|^2: every pass of a layer evaluates a child through this one expression, so the
// radix passes and the compaction see bit-identical values
__device__ __forceinline__ float kb_leaf(float2 b, float rii, float2 pt, float parent) {
    const float tx = fmaf(-rii, pt.x, b.x), ty = fmaf(-rii, pt.y, b.y);
    return fmaf(tx, tx, fmaf(ty, ty, parent));
}

// ascending bitonic sort of a[0, n) (n a power of two) by one warp
__device__ void kb_bitonic(unsigned long long* a, int n, int lane) {
    for (int size = 2; size <= n; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            for (int t = lane; t < (n >> 1); t += 32) {
                const int i = 2 * t - (t & (stride - 1)), j = i + stride;
                const unsigned long long x = a[i], y = a[j];
                if ((x > y) == ((i & size) == 0)) { a[i] = y; a[j] = x; }
            }
            __syncwarp();
        }
    }
}

// One warp per problem. Shared memory: points [NP] float2 per CTA, then per warp
//   keys [kpad] u64 | offsets b [k] float2 | metrics [k] float | histogram [256] u32 | paths 2 x [k, S] u8
__global__ void __launch_bounds__(256) kbest_search_kernel(const KbParams q) {
    extern __shared__ float2 smem[];
    const int T = blockDim.x, t = threadIdx.x, lane = t & 31, W = T >> 5;
    const int S = q.S, K = q.K, NP = q.NP, lg = q.lg, kk = q.k;
    const unsigned lt_mask = (1u << lane) - 1u;
    float2* spts = smem;
    for (int i = t; i < NP; i += T)
        spts[i] = q.real_rep ? make_float2(static_cast<const float*>(q.points)[i], 0.f)
                             : static_cast<const float2*>(q.points)[i];
    __syncthreads();
    char* wb = reinterpret_cast<char*>(smem + NP) + (size_t)(t >> 5) * q.per_warp;
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(wb);
    float2* bo = reinterpret_cast<float2*>(keys + q.kpad);
    float* met = reinterpret_cast<float*>(bo + kk);
    unsigned* hist = reinterpret_cast<unsigned*>(met + kk);
    unsigned char* cur = reinterpret_cast<unsigned char*>(hist + 256);
    unsigned char* nxt = cur + kk * S;
    for (long long p = (long long)blockIdx.x * W + (t >> 5); p < q.P; p += (long long)gridDim.x * W) {   // warp-uniform
        const long long* oi = q.oidx + p * K;
        bool any = false;
        for (int k = 0; k < K; ++k) any = any || oi[k] >= 0;
        if (!any) continue;
        const float2* rec = q.rec + p * qr_record_size(S);
        const int* ord = q.order + p * S;
        __syncwarp();                                   // the previous problem's finish step has read the path list
        if (lane == 0) {
            met[0] = 0.f;
            bo[0] = rec[S * S + S - 1];
        }
        __syncwarp();
        int npar = 1;
        for (int i = S - 1; i >= 0; --i) {
            const float rii = rec[i * S + i].x;
            const int N = npar * NP, need = min(kk, N);
            auto child = [&](int c) { return kb_leaf(bo[c >> lg], rii, spts[c & (NP - 1)], met[c >> lg]); };
            // a) radix select: children with (bits & mask) < prefix are taken (below of them), those equal to prefix
            //    hold the rest; full once that bucket is taken whole
            unsigned prefix = 0, mask = 0;
            int below = 0;
            bool full = need == N;
            for (int shift = 24; !full && shift >= 0; shift -= 8) {
                for (int b = lane; b < 256; b += 32) hist[b] = 0;
                __syncwarp();
                for (int base = 0; base < N; base += 32) {
                    const int c = base + lane;
                    bool in = false;
                    unsigned bin = 0;
                    if (c < N) {
                        const unsigned u = __float_as_uint(child(c));
                        in = (u & mask) == prefix;
                        bin = (u >> shift) & 255u;
                    }
                    const unsigned grp = __match_any_sync(0xffffffffu, in ? bin : 256u + lane);
                    if (in && lane == __ffs(grp) - 1) atomicAdd(&hist[bin], (unsigned)__popc(grp));
                }
                __syncwarp();
                const int rem = need - below;
                unsigned h8[8], local = 0;
#pragma unroll
                for (int j = 0; j < 8; ++j) { h8[j] = hist[lane * 8 + j]; local += h8[j]; }
                unsigned incl = local;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const unsigned v = __shfl_up_sync(0xffffffffu, incl, o);
                    if (lane >= o) incl += v;
                }
                const int L = __ffs(__ballot_sync(0xffffffffu, incl >= (unsigned)rem)) - 1;
                int sb = 0, sbelow = 0, scnt = 0;
                if (lane == L) {
                    unsigned cum = incl - local;
#pragma unroll
                    for (int j = 0; j < 8; ++j) {
                        if (cum + h8[j] >= (unsigned)rem) { sb = 8 * L + j; sbelow = (int)cum; scnt = (int)h8[j]; break; }
                        cum += h8[j];
                    }
                }
                sb = __shfl_sync(0xffffffffu, sb, L);
                sbelow = __shfl_sync(0xffffffffu, sbelow, L);
                scnt = __shfl_sync(0xffffffffu, scnt, L);
                prefix |= (unsigned)sb << shift;
                mask |= 255u << shift;
                below += sbelow;
                full = below + scnt == need;
                __syncwarp();                           // histogram read before the next pass clears it
            }
            // b) compaction in index order: equal metrics (all 32 bits fixed, bucket not whole) are taken lowest first
            const int rem = need - below;
            int taken = 0, eq_seen = 0;
            for (int base = 0; base < N; base += 32) {
                const int c = base + lane;
                bool lt = false, eq = false;
                unsigned u = 0;
                if (c < N) {
                    u = __float_as_uint(child(c));
                    lt = (u & mask) < prefix;
                    eq = (u & mask) == prefix;
                }
                const unsigned eqb = __ballot_sync(0xffffffffu, eq);
                const bool take = lt || (eq && (full || eq_seen + __popc(eqb & lt_mask) < rem));
                const unsigned tb = __ballot_sync(0xffffffffu, take);
                if (take) keys[taken + __popc(tb & lt_mask)] = ((unsigned long long)u << 32) | (unsigned)c;
                taken += __popc(tb);
                eq_seen += __popc(eqb);
            }
            // c) sort by (metric, child index)
            int n2 = 1;
            while (n2 < need) n2 <<= 1;
            for (int j = need + lane; j < n2; j += 32) keys[j] = ~0ull;
            __syncwarp();
            kb_bitonic(keys, n2, lane);
            // new path list, metrics and the next layer's offsets
            for (int r = lane; r < need; r += 32) {
                const unsigned long long key = keys[r];
                const int c = (int)(key & 0xffffffffu), par = c >> lg;
                met[r] = __uint_as_float((unsigned)(key >> 32));
                for (int j = i + 1; j < S; ++j) nxt[r * S + j] = cur[par * S + j];
                nxt[r * S + i] = (unsigned char)(c & (NP - 1));
                if (i > 0) {
                    float2 b = rec[S * S + i - 1];
                    for (int j = i; j < S; ++j) {
                        const float2 R = rec[(i - 1) * S + j], pj = spts[nxt[r * S + j]];
                        b.x = fmaf(-R.x, pj.x, fmaf(R.y, pj.y, b.x));
                        b.y = fmaf(-R.x, pj.y, fmaf(-R.y, pj.x, b.y));
                    }
                    bo[r] = b;
                }
            }
            unsigned char* sw = cur; cur = nxt; nxt = sw;
            npar = need;
            __syncwarp();
        }
        // finish: cur holds the npar kept paths, rank 0 the best
        const int m = q.m;
        if (q.hard) {
            for (int ks = lane; ks < K; ks += 32) {
                const long long o = oi[ks];
                if (o < 0) continue;
                int pos_re = 0, pos_im = 0;
                for (int s2 = 0; s2 < S; ++s2) {
                    if (ord[s2] == ks) pos_re = s2;
                    if (ord[s2] == K + ks) pos_im = s2;
                }
                int idx = cur[pos_re];
                if (q.real_rep) idx = sb_dense::pam2qam_index(cur[pos_re], cur[pos_im], m);
                if (q.symbol) {
                    reinterpret_cast<int*>(q.out)[o] = idx;
                } else {
                    for (int j = 0; j < m; ++j) reinterpret_cast<float*>(q.out)[o * m + j] = (float)((idx >> (m - 1 - j)) & 1);
                }
            }
        } else {
            const int md = m >> q.real_rep;             // bits per detection-domain symbol
            for (int it = lane; it < S * md; it += 32) {
                const int s2 = it / md, b = it % md;
                float l0 = INFINITY, l1 = INFINITY;
                for (int r = 0; r < npar; ++r) {
                    const float d = met[r];
                    if ((cur[r * S + s2] >> (md - 1 - b)) & 1) l1 = fminf(l1, d); else l0 = fminf(l0, d);
                }
                if (q.real_rep) { l0 *= 0.5f; l1 *= 0.5f; }
                const float llr = fminf(fmaxf(l0 - l1, -q.clip), q.clip);
                const int ds = ord[s2];
                const int ks = q.real_rep ? ds % K : ds, bit = q.real_rep ? 2 * b + ds / K : b;
                const long long o = oi[ks];
                if (o >= 0) reinterpret_cast<float*>(q.out)[o * m + bit] = llr;
            }
        }
    }
}

// Malformed arguments are SB_EINVAL; well-formed configurations beyond the kernels' limits (counted in the detection
// domain: S = K or 2 K layers of |C| or sqrt(|C|) points) are SB_EUNSUPPORTED.
int kb_check(const char* who, int M, int K, int num_points, int k, int real_rep, int output, int hard_out, float clip) {
    const int bits = num_points >= 2 ? 31 - __builtin_clz((unsigned)num_points) : 0;
    if (K < 1 || M < K || k < 1 || num_points < 2 || (num_points & (num_points - 1)) || real_rep < 0 || real_rep > 1 ||
        output < 0 || output > 1 || hard_out < 0 || hard_out > 1 || !(clip >= 0.f)) {
        sb_set_error("%s: bad arguments (need K >= 1 streams, M >= K antennas, k >= 1, a power-of-two constellation of "
                     ">= 2 points, real_rep / output / hard_out in {0, 1}, llr_clip >= 0)", who);
        return SB_EINVAL;
    }
    if (real_rep && (bits & 1)) {
        sb_set_error("%s: bad arguments (the real representation needs a QAM constellation, an even number of bits; "
                     "%d given)", who, bits);
        return SB_EINVAL;
    }
    if (output == 1 && !hard_out) {
        sb_set_error("%s: bad arguments (symbol output needs hard_out = 1: soft symbols are not provided)", who);
        return SB_EINVAL;
    }
    const int S = K << real_rep, NP = real_rep ? 1 << (bits / 2) : num_points;
    if (S > kKbMaxLayers) {
        sb_set_error("%s: %d streams are %d layers, the limit is %d", who, K, S, kKbMaxLayers);
        return SB_EUNSUPPORTED;
    }
    if (k > kKbMaxK) {
        sb_set_error("%s: k = %d paths, the limit is %d", who, k, kKbMaxK);
        return SB_EUNSUPPORTED;
    }
    if (NP > kKbMaxPoints) {
        sb_set_error("%s: a detection constellation of %d points, the limit is %d", who, NP, kKbMaxPoints);
        return SB_EUNSUPPORTED;
    }
    if ((long long)k * NP > kKbMaxChildren) {
        sb_set_error("%s: k = %d paths of %d points are %lld children per layer, the limit is %d", who, k, NP,
                     (long long)k * NP, kKbMaxChildren);
        return SB_EUNSUPPORTED;
    }
    return SB_OK;
}

// Both launches on the caller's workspace of P records.
int kb_run(const char* who, const MimoProblem& pb, const float* points, int num_points, int k, int real_rep, int output,
           int hard_out, float clip, void* out, void* ws, size_t ws_bytes, cudaStream_t stream) {
    const long long P = pb.P;
    const int M = pb.M, K = pb.K;
    if (!ws || ws_bytes < kb_workspace_bytes(P, K, real_rep)) {
        sb_set_error("%s: the workspace needs %zu bytes (sb_kbest_workspace_bytes), %zu given", who,
                     kb_workspace_bytes(P, K, real_rep), ws ? ws_bytes : (size_t)0);
        return SB_ENOMEM;
    }
    const int S = K << real_rep, MR = M << real_rep;
    const int bits = 31 - __builtin_clz((unsigned)num_points);
    const int NP = real_rep ? 1 << (bits / 2) : num_points;
    size_t psmem = 0;
    const size_t p_thread = sizeof(float2) * ((size_t)M * M + (size_t)M * K + M +
                                              (real_rep ? (size_t)MR * S + MR : 0));
    const int pthreads = sb_dense::detector_threads(who, 0, p_thread, M, K, &psmem);
    if (!pthreads) return SB_EUNSUPPORTED;
    int kpad = 1;
    while (kpad < k) kpad <<= 1;
    const size_t per_warp = (sizeof(unsigned long long) * kpad + sizeof(float2) * k + sizeof(float) * k +
                             sizeof(unsigned) * 256 + 2 * (size_t)k * S + 7) / 8 * 8;
    const int warps = (int)std::min<size_t>(8, (sb_dense::kScratchSmemCap - NP * sizeof(float2)) / per_warp);
    const size_t esmem = NP * sizeof(float2) + per_warp * warps;
    float2* recs = (float2*)ws;
    long long* oidx = (long long*)((char*)ws + sizeof(float2) * qr_record_size(S) * (size_t)P);
    int* orders = (int*)((char*)oidx + sizeof(long long) * K * (size_t)P);
    SB_CUDA(cudaFuncSetAttribute(kbest_prologue_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)psmem));
    kbest_prologue_kernel<<<sb_grid(P, pthreads, 16), pthreads, psmem, stream>>>(pb, real_rep, recs, oidx, orders);
    SB_LAUNCH_CHECK();
    KbParams q{recs, oidx, orders, points, out, P, S, K, NP, 31 - __builtin_clz((unsigned)NP), bits, k, kpad, real_rep,
               output, hard_out, clip, (int)per_warp};
    SB_CUDA(cudaFuncSetAttribute(kbest_search_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)esmem));
    kbest_search_kernel<<<sb_grid(P, warps, 16), 32 * warps, esmem, stream>>>(q);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

}  // namespace

extern "C" size_t sb_kbest_workspace_bytes(int64_t num_problems, int32_t K, int32_t real_rep) {
    return num_problems > 0 && K >= 1 && (real_rep == 0 || real_rep == 1) && (K << real_rep) <= kKbMaxLayers
               ? kb_workspace_bytes(num_problems, K, real_rep)
               : 0;
}

extern "C" int sb_mimo_kbest(const float* d_y, const float* d_h, const float* d_s, const float* d_points, void* d_out,
                             void* d_workspace, size_t workspace_bytes, int64_t num, int32_t M, int32_t K,
                             int32_t num_points, int32_t k, int32_t real_rep, int32_t output, int32_t hard_out,
                             float llr_clip, void* stream) {
    const int rc = kb_check("sb_mimo_kbest", M, K, num_points, k, real_rep, output, hard_out, llr_clip);
    if (rc != SB_OK) return rc;
    if (num == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_y && d_h && d_s && d_points && d_out && num > 0, "sb_mimo_kbest: bad arguments");
    return kb_run("sb_mimo_kbest", sb_dense::dense_problem(d_y, d_h, d_s, num, M, K), d_points, num_points, k, real_rep,
                  output, hard_out, llr_clip, d_out, d_workspace, workspace_bytes, (cudaStream_t)stream);
}

extern "C" int sb_ofdm_kbest(const float* d_y, const float* d_h_hat, const float* d_err_var, const int64_t* h_ev_stride,
                             const float* d_no, const int64_t* h_no_stride, const int32_t* d_desired,
                             const int32_t* d_undesired, const int32_t* d_out_stream, const int32_t* d_data_pos,
                             const float* d_points, void* d_out, void* d_workspace, size_t workspace_bytes,
                             int64_t batch, int32_t num_rx, int32_t num_rx_ant, int32_t num_tx_streams,
                             int32_t num_symbols, int32_t num_subcarriers, int32_t streams_per_rx,
                             int32_t interferers_per_rx, int32_t num_data, int32_t num_points, int32_t k,
                             int32_t real_rep, int32_t output, int32_t hard_out, float llr_clip, void* stream) {
    const int rc = kb_check("sb_ofdm_kbest", num_rx_ant, streams_per_rx, num_points, k, real_rep, output, hard_out,
                            llr_clip);
    if (rc != SB_OK) return rc;
    if (batch == 0) return SB_OK;                       // empty batch: nothing to do, pointers may be null
    const int ac = sb_dense::ofdm_check("sb_ofdm_kbest", d_y, d_h_hat, d_err_var, h_ev_stride, d_no, h_no_stride,
                                        d_desired, d_undesired, d_out_stream, d_data_pos, d_points, d_out, batch,
                                        num_rx_ant, interferers_per_rx);
    if (ac != SB_OK) return ac;
    const MimoProblem pb = sb_dense::ofdm_problem(d_y, d_h_hat, d_err_var, h_ev_stride, d_no, h_no_stride, d_desired,
                                                  d_undesired, d_out_stream, d_data_pos, batch, num_rx, num_rx_ant,
                                                  num_tx_streams, num_symbols, num_subcarriers, streams_per_rx,
                                                  interferers_per_rx, num_data);
    return kb_run("sb_ofdm_kbest", pb, d_points, num_points, k, real_rep, output, hard_out, llr_clip, d_out, d_workspace,
                  workspace_bytes, (cudaStream_t)stream);
}
