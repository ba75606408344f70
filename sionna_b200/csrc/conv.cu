// conv.cu -- rate-1/n convolutional codes: encoder, Viterbi decoder and BCJR decoder (fec/conv/encoding.py:11-292,
// fec/conv/decoding.py:19-943), DESIGN §3.11; the turbo decoder on the same BCJR passes (fec/turbo/decoding.py:15-435),
// DESIGN §3.12.
//
// Trellis. K = constraint length, ns = 2^(K-1) states, conv_n output bits per step. The newest register bit is the
// state's MSB, so the two predecessors of state s are ((s << 1) & (ns - 1)) | b, b = 0, 1, and the two successors of
// state j are (j >> 1) and (j >> 1) | ns / 2. The host passes the reference's tables (Trellis._generate_transitions):
// they fix which predecessor is listed first (the Viterbi tie rule), which input bit and which output symbol each
// transition carries. The tables are checked against the shift-register structure and packed into a kernel parameter.
//
// Decoders. A codeword is served by L = min(ns, 32) lanes of one warp, R = ns / L states per lane; for ns < 32 a warp
// serves 32 / ns codewords side by side. The forward recursions hold lane l's states l R ... l R + R - 1 ("blocked"):
// predecessor (2 s + b) mod ns of state l R + r then sits in register (2 r + b) mod R of lane (2 l + (2 r + b) / R) mod L,
// a register index that is the same on every lane, so each predecessor is one __shfl_sync. The BCJR backward recursion
// holds states r L + l ("interleaved"), in which the successors are one uniform shuffle each as well. The 2^conv_n
// distinct branch metrics of a step are computed once per chunk of steps into shared memory.
//
// Arithmetic. Built with -fmad=false. The Viterbi branch metric is the reference's sum over j = 0 ... conv_n - 1 in that
// order, the path metric one fp32 add per branch, the decision the first predecessor unless the second is strictly
// smaller (tf.argmin); no renormalisation. oracle/conv.py restates these steps in float32, so decisions and outputs
// are bit-identical to it. BCJR runs "map" and "log" in the log domain with max*(a, b) = max + log1p(exp(-|a - b|)),
// "maxlog" with max; alpha and beta are normalised per step by their state-0 value.
#include "sb_common.h"
#include <math.h>
#include <stdint.h>
#include <vector>

namespace {

constexpr int kMaxStates = 256;
constexpr int kMaxConvN = 8;
constexpr int kWarps = 4;                           // warps per CTA
constexpr int kTableFloats = 2048;                  // per-warp branch-metric table budget (floats)
constexpr size_t kOnChipBytes = 48 * 1024;          // per-CTA decisions / alpha kept in shared memory up to this size
constexpr unsigned kFull = 0xffffffffu;

// Per state s, both incoming transitions (slot 0 / 1 in the reference's from_nodes order): op0 | op1 << 8 |
// low bit of the slot-0 predecessor << 16 | input bit of slot 0 << 17 | input bit of slot 1 << 18.
// Per state j, both outgoing transitions (input 0 / 1): op | op' << 8 | (successor of input 0 has the MSB set) << 16.
struct ConvTrellis {
    uint32_t to[kMaxStates];
    uint32_t from[kMaxStates];
};

__device__ __forceinline__ uint32_t parity(uint32_t x) { return __popc(x) & 1u; }

// ---- encoder --------------------------------------------------------------------------------------------------------
struct Polys { uint32_t g[kMaxConvN]; };

// Feed-forward codes: one thread per (codeword, step); the output of step t is a function of inputs t - K + 1 ... t
// (0 before the start and in the termination steps).
__global__ void conv_encode_ff_kernel(const float* __restrict__ u, float* __restrict__ x, long long batch, int k,
                                      int T, int K, int conv_n, Polys p) {
    const long long total = batch * T;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const long long cw = i / T;
        const int t = (int)(i - cw * T);
        const float* ur = u + cw * k;
        uint32_t w = 0;
        for (int d = 0; d < K; ++d) {
            const int tau = t - d;
            const uint32_t bit = (tau >= 0 && tau < k) ? ((uint32_t)(int)__ldg(ur + tau) & 1u) : 0u;
            w |= bit << (K - 1 - d);
        }
        float* xr = x + (cw * T + t) * conv_n;
        for (int j = 0; j < conv_n; ++j) xr[j] = (float)parity(p.g[j] & w);
    }
}

// Recursive systematic codes: one thread per codeword, serial over the steps; g[0] is the feedback polynomial. The
// termination inputs equal the feedback bit, which drives the register to zero (encoding.py:262-285).
__global__ void conv_encode_rsc_kernel(const float* __restrict__ u, float* __restrict__ x, long long batch, int k,
                                       int T, int K, int conv_n, Polys p) {
    const uint32_t fb_mask = p.g[0] & ((1u << (K - 1)) - 1u);
    for (long long cw = blockIdx.x * (long long)blockDim.x + threadIdx.x; cw < batch;
         cw += (long long)gridDim.x * blockDim.x) {
        const float* ur = u + cw * k;
        float* xr = x + cw * T * conv_n;
        uint32_t st = 0;
        for (int t = 0; t < T; ++t) {
            const uint32_t fb = parity(st & fb_mask);
            const uint32_t in = t < k ? ((uint32_t)(int)__ldg(ur + t) & 1u) : fb;
            const uint32_t w = ((in ^ fb) << (K - 1)) | st;
            for (int j = 0; j < conv_n; ++j) xr[t * conv_n + j] = (float)parity(p.g[j] & w);
            st = w >> 1;
        }
    }
}

// ---- branch metrics -------------------------------------------------------------------------------------------------
enum { kSoft = 0, kHard = 1, kHalf = 2 };   // Viterbi soft_llr, Viterbi hard, BCJR (half LLRs, internal sign)

// Metric of output symbol o (bit j = bit conv_n - 1 - j of o, MSB first) from the step's conv_n inputs, summed over j
// in order. kSoft: sum llr_j (1 - 2 b_j) (decoding.py:367-373); kHard: sum |int_mod_2(llr_j) - b_j| (:375-380);
// kHalf: sum 0.5 (-llr_j) (1 - 2 b_j), the log of the reference's gamma factor (:704-720).
template <int MODE>
__device__ __forceinline__ float branch_metric(const float* __restrict__ y, int o, int conv_n) {
    float acc = 0.f;
    for (int j = 0; j < conv_n; ++j) {
        const float v = __ldg(y + j);
        const bool b = (o >> (conv_n - 1 - j)) & 1;
        float term;
        if (MODE == kSoft) {
            term = b ? -v : v;
        } else if (MODE == kHard) {
            const float y2 = fmodf(fabsf(rintf(v)), 2.f);
            term = fabsf(__fsub_rn(y2, b ? 1.f : 0.f));
        } else {
            const float h = __fmul_rn(0.5f, v);
            term = b ? h : -h;
        }
        acc = j == 0 ? term : __fadd_rn(acc, term);
    }
    return acc;
}

// Fill the warp's table for steps [t0, t0 + nt) of its G codewords: tab[(g * ch + tt) * tw + o]; codeword cw's step t
// reads llr[(cw * row_steps + t) * conv_n ...]. With a prior (tw = 2^conv_n + 1) entry 2^conv_n holds prior(g, cw, t),
// half the a-priori LLR of codeword g's step t. Lanes of codewords beyond the batch read the last codeword.
struct NoPrior {
    __device__ float operator()(int, long long, int) const { return 0.f; }
};

template <int MODE, class Prior>
__device__ void fill_table(float* tab, const float* __restrict__ llr, long long row_steps,
                                           const Prior& prior, long long cw0, long long batch, int G, int conv_n,
                                           int t0, int nt, int ch, int tw, int lane) {
    const int no = 1 << conv_n;
    const int total = G * nt * tw;
    for (int e = lane; e < total; e += 32) {
        const int o = e % tw;
        const int tt = (e / tw) % nt;
        const int g = e / (tw * nt);
        const long long cw = min(cw0 + g, batch - 1);
        const int t = t0 + tt;
        float v;
        if (o < no) v = branch_metric<MODE>(llr + (cw * row_steps + t) * conv_n, o, conv_n);
        else v = prior(g, cw, t);
        tab[(g * ch + tt) * tw + o] = v;
    }
}

// Layout shared by both decoders: lanes per codeword L = min(ns, 32), codewords per warp G = 32 / L, steps per table
// chunk ch, table width tw. step_bytes: decision words (Viterbi) or alpha (BCJR) per codeword and step.
struct WarpPlan { int G, ch, tw; size_t table_bytes, state_bytes; bool on_chip; };

static WarpPlan warp_plan(int ns, int conv_n, int T, bool prior, size_t step_bytes) {
    WarpPlan p;
    p.G = ns < 32 ? 32 / ns : 1;
    p.tw = (1 << conv_n) + (prior ? 1 : 0);
    p.ch = std::max(1, std::min(32, kTableFloats / (p.G * p.tw)));
    p.table_bytes = (size_t)p.G * p.ch * p.tw * sizeof(float);
    p.state_bytes = (size_t)p.G * T * step_bytes;
    p.on_chip = kWarps * p.state_bytes <= kOnChipBytes;
    return p;
}

static size_t viterbi_step_bytes(int ns) { return (size_t)(ns > 32 ? ns / 32 : 1) * sizeof(uint32_t); }
static size_t bcjr_step_bytes(int ns) { return (size_t)ns * sizeof(float); }

// ---- Viterbi --------------------------------------------------------------------------------------------------------
// Decisions: one bit per state and step, word (t, s mod R) bit s / R, G * T * R words per warp (shared memory or the
// caller's workspace). Lane 0 of each codeword then traces back serially.
template <int L, int R, int MODE>
__global__ void __launch_bounds__(kWarps * 32) viterbi_kernel(
    const float* __restrict__ llr, float* __restrict__ out, uint32_t* __restrict__ ws_dec, long long batch, int T,
    int conv_n, int k_out, int terminate, int info_bits, int ch, int tw, int on_chip, const __grid_constant__ ConvTrellis tr) {
    constexpr int NS = L * R, G = 32 / L;
    extern __shared__ float smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane / L, l = lane % L;
    const long long cw0 = ((long long)blockIdx.x * kWarps + warp) * G;
    if (cw0 >= batch) return;
    const size_t table_floats = (size_t)G * ch * tw;
    float* tab = smem + warp * table_floats;
    uint32_t* dec = on_chip ? reinterpret_cast<uint32_t*>(smem + kWarps * table_floats) + (size_t)warp * G * T * R
                            : ws_dec + cw0 * T * R;
    uint32_t* mydec = dec + (size_t)g * T * R;

    uint32_t trw[R];
    float pm[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        trw[r] = tr.to[l * R + r];
        pm[r] = (l * R + r) == 0 ? 0.f : 1048576.f;        // LARGEDIST = 2^20 (decoding.py:411, 430-433)
    }
    for (int t0 = 0; t0 < T; t0 += ch) {
        const int nt = min(ch, T - t0);
        __syncwarp();
        fill_table<MODE>(tab, llr, T, NoPrior{}, cw0, batch, G, conv_n, t0, nt, ch, tw, lane);
        __syncwarp();
        for (int tt = 0; tt < nt; ++tt) {
            const float* bm = tab + (g * ch + tt) * tw;
            float npm[R];
            bool d[R];
#pragma unroll
            for (int r = 0; r < R; ++r) {
                const int q0 = 2 * r, q1 = 2 * r + 1;
                const float v0 = __shfl_sync(kFull, pm[q0 % R], (2 * l + q0 / R) % L, L);
                const float v1 = __shfl_sync(kFull, pm[q1 % R], (2 * l + q1 / R) % L, L);
                const bool swap = (trw[r] >> 16) & 1u;
                const float m0 = __fadd_rn(swap ? v1 : v0, bm[trw[r] & 0xff]);
                const float m1 = __fadd_rn(swap ? v0 : v1, bm[(trw[r] >> 8) & 0xff]);
                d[r] = m1 < m0;
                npm[r] = d[r] ? m1 : m0;
            }
            uint32_t word = 0;
#pragma unroll
            for (int r = 0; r < R; ++r) {
                uint32_t m = __ballot_sync(kFull, d[r]);
                if (L < 32) m = (m >> (g * L)) & ((1u << L) - 1u);
                if (l == r) word = m;
                pm[r] = npm[r];
            }
            if (l < R) mydec[(size_t)(t0 + tt) * R + l] = word;
        }
    }
    // final state: 0 if terminated, else the first state with the least metric (decoding.py:334-337)
    float best = pm[0];
    int bs = l * R;
#pragma unroll
    for (int r = 1; r < R; ++r)
        if (pm[r] < best) { best = pm[r]; bs = l * R + r; }
#pragma unroll
    for (int off = L / 2; off > 0; off >>= 1) {
        const float ob = __shfl_xor_sync(kFull, best, off, L);
        const int os = __shfl_xor_sync(kFull, bs, off, L);
        if (ob < best || (ob == best && os < bs)) { best = ob; bs = os; }
    }
    __syncwarp();
    const long long cw = cw0 + g;
    if (l != 0 || cw >= batch) return;
    int s = terminate ? 0 : bs;
    const int n = T * conv_n;
    for (int t = T - 1; t >= 0; --t) {
        const uint32_t slot = (mydec[(size_t)t * R + (s % R)] >> (s / R)) & 1u;
        const uint32_t w = tr.to[s];
        const uint32_t op = slot ? (w >> 8) & 0xff : w & 0xff;
        const uint32_t lb = ((w >> 16) & 1u) ^ slot;
        if (info_bits) {
            if (t < k_out) out[cw * k_out + t] = (float)((w >> (17 + slot)) & 1u);
        } else {
            for (int j = 0; j < conv_n; ++j) out[cw * n + t * conv_n + j] = (float)((op >> (conv_n - 1 - j)) & 1u);
        }
        s = ((s << 1) & (NS - 1)) | (int)lb;
    }
}

// ---- BCJR -----------------------------------------------------------------------------------------------------------
template <bool MAXLOG>
__device__ __forceinline__ float max_star(float a, float b) {
    const float m = fmaxf(a, b);
    if (MAXLOG) return m;
    const float d = fabsf(__fsub_rn(a, b));
    return d < INFINITY ? __fadd_rn(m, log1pf(__expf(-d))) : m;   // d = NaN (both -inf) or inf: the max
}

// alpha_t (before step t) is stored per step, ns floats in state order: G * T * ns per warp (shared or workspace). The
// backward pass forms beta and the APP LLR of step t from alpha_t, gamma_t and beta_{t+1}. Both passes are shared by
// the BCJR and turbo kernels: `prior` supplies the a-priori LLR of a step (see fill_table) and `store(t, v)` receives the
// APP LLR v (Sionna's sign) of step t < num_out of the lane group's own codeword, on its lane 0, if it is in the batch.
// Codeword cw's channel LLRs are llr[(cw * row_steps + t) * conv_n ...]; alpha points at the group's own T * ns floats.
template <int L, int R, bool MAXLOG, class Prior>
__device__ __forceinline__ void bcjr_forward(float* tab, float* alpha, const float* __restrict__ llr, long long row_steps,
                                             const Prior& prior, long long cw0, long long batch, int T, int conv_n,
                                             int ch, int tw, int l, int g, int lane, const ConvTrellis& tr) {
    constexpr int NS = L * R, G = 32 / L;
    const int no = 1 << conv_n;
    uint32_t trw[R];
    float a[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        trw[r] = tr.to[l * R + r];
        a[r] = (l * R + r) == 0 ? 0.f : -INFINITY;
    }
    for (int t0 = 0; t0 < T; t0 += ch) {
        const int nt = min(ch, T - t0);
        __syncwarp();
        fill_table<kHalf>(tab, llr, row_steps, prior, cw0, batch, G, conv_n, t0, nt, ch, tw, lane);
        __syncwarp();
        for (int tt = 0; tt < nt; ++tt) {
            const float* bm = tab + (g * ch + tt) * tw;
            const float ha = bm[no];
            float* at = alpha + (size_t)(t0 + tt) * NS + l * R;
#pragma unroll
            for (int r = 0; r < R; ++r) at[r] = a[r];
            float na[R];
#pragma unroll
            for (int r = 0; r < R; ++r) {
                const int q0 = 2 * r, q1 = 2 * r + 1;
                const float v0 = __shfl_sync(kFull, a[q0 % R], (2 * l + q0 / R) % L, L);
                const float v1 = __shfl_sync(kFull, a[q1 % R], (2 * l + q1 / R) % L, L);
                const uint32_t w = trw[r];
                const bool swap = (w >> 16) & 1u;
                const float g0 = __fadd_rn(bm[w & 0xff], ((w >> 17) & 1u) ? ha : -ha);
                const float g1 = __fadd_rn(bm[(w >> 8) & 0xff], ((w >> 18) & 1u) ? ha : -ha);
                na[r] = max_star<MAXLOG>(__fadd_rn(swap ? v1 : v0, g0), __fadd_rn(swap ? v0 : v1, g1));
            }
            const float a0 = __shfl_sync(kFull, na[0], 0, L);
#pragma unroll
            for (int r = 0; r < R; ++r) a[r] = __fsub_rn(na[r], a0);
        }
    }
    __syncwarp();
}

template <int L, int R, bool MAXLOG, class Prior, class Store>
__device__ __forceinline__ void bcjr_backward(float* tab, const float* alpha, const float* __restrict__ llr,
                                              long long row_steps, const Prior& prior, long long cw0, long long batch,
                                              int T, int conv_n, int num_out, int terminate, int ch, int tw, int l,
                                              int g, int lane, const ConvTrellis& tr, const Store& store) {
    constexpr int NS = L * R, G = 32 / L;
    const int no = 1 << conv_n;
    uint32_t frw[R];
    float b[R];
#pragma unroll
    for (int r = 0; r < R; ++r) {
        frw[r] = tr.from[r * L + l];
        b[r] = (terminate && (r * L + l) != 0) ? -INFINITY : 0.f;   // uniform start unless terminated (decoding.py:722-741)
    }
    const long long cw = cw0 + g;
    for (int t1 = T; t1 > 0; t1 -= ch) {
        const int t0 = max(0, t1 - ch), nt = t1 - t0;
        __syncwarp();
        fill_table<kHalf>(tab, llr, row_steps, prior, cw0, batch, G, conv_n, t0, nt, ch, tw, lane);
        __syncwarp();
        for (int tt = nt - 1; tt >= 0; --tt) {
            const int t = t0 + tt;
            const float* bm = tab + (g * ch + tt) * tw;
            const float ha = bm[no];
            const float* at = alpha + (size_t)t * NS;
            float nb[R], num = -INFINITY, den = -INFINITY;
#pragma unroll
            for (int r = 0; r < R; ++r) {
                const float lo = __shfl_sync(kFull, b[r >> 1], (r & 1) * (L / 2) + (l >> 1), L);
                const float hi = __shfl_sync(kFull, b[(r + R) >> 1], ((r + R) & 1) * (L / 2) + (l >> 1), L);
                const uint32_t w = frw[r];
                const bool hi0 = (w >> 16) & 1u;
                const float e0 = __fadd_rn(__fadd_rn(bm[w & 0xff], -ha), hi0 ? hi : lo);
                const float e1 = __fadd_rn(__fadd_rn(bm[(w >> 8) & 0xff], ha), hi0 ? lo : hi);
                nb[r] = max_star<MAXLOG>(e0, e1);
                const float aj = at[r * L + l];
                num = max_star<MAXLOG>(num, __fadd_rn(aj, e0));
                den = max_star<MAXLOG>(den, __fadd_rn(aj, e1));
            }
#pragma unroll
            for (int off = L / 2; off > 0; off >>= 1) {
                num = max_star<MAXLOG>(num, __shfl_xor_sync(kFull, num, off, L));
                den = max_star<MAXLOG>(den, __shfl_xor_sync(kFull, den, off, L));
            }
            if (l == 0 && cw < batch && t < num_out) store(t, __fsub_rn(den, num));   // Sionna's sign: log p(1) / p(0)
            const float b0 = __shfl_sync(kFull, nb[0], 0, L);
#pragma unroll
            for (int r = 0; r < R; ++r) b[r] = __fsub_rn(nb[r], b0);
        }
    }
}

template <int L, int R, bool MAXLOG>
__global__ void __launch_bounds__(kWarps * 32) bcjr_kernel(
    const float* __restrict__ llr, const float* __restrict__ llr_a, float* __restrict__ out, float* __restrict__ ws_alpha,
    long long batch, int T, int conv_n, int num_out, int terminate, int hard_out, int ch, int tw, int on_chip,
    const __grid_constant__ ConvTrellis tr) {
    constexpr int NS = L * R, G = 32 / L;
    extern __shared__ float smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane / L, l = lane % L;
    const long long cw0 = ((long long)blockIdx.x * kWarps + warp) * G;
    if (cw0 >= batch) return;
    const size_t table_floats = (size_t)G * ch * tw;
    float* tab = smem + warp * table_floats;
    float* alpha = (on_chip ? smem + kWarps * table_floats + (size_t)warp * G * T * NS : ws_alpha + cw0 * T * NS) +
                   (size_t)g * T * NS;
    const auto prior = [&](int, long long cw, int t) { return llr_a ? __fmul_rn(0.5f, __ldg(llr_a + cw * T + t)) : 0.f; };
    const long long cw = cw0 + g;
    const auto store = [&](int t, float v) { out[cw * num_out + t] = hard_out ? (v > 0.f ? 1.f : 0.f) : v; };
    bcjr_forward<L, R, MAXLOG>(tab, alpha, llr, T, prior, cw0, batch, T, conv_n, ch, tw, l, g, lane, tr);
    bcjr_backward<L, R, MAXLOG>(tab, alpha, llr, T, prior, cw0, batch, T, conv_n, num_out, terminate, ch, tw, l, g,
                                lane, tr, store);
}

// ---- turbo ----------------------------------------------------------------------------------------------------------
// All num_iter iterations of both rate-1/2 component decoders in one launch (fec/turbo/decoding.py:357-435). llr holds
// the two component codewords of each turbo codeword side by side, [batch, 2, 2 T]; decoder 2's systematic LLRs are
// decoder 1's gathered through pi. The warp owns its G codewords throughout, so __syncwarp is the only barrier.
// Extrinsic buffer: k floats per codeword, always in decoder 1's (natural) order. Decoder 1 reads its prior at step t
// from position t and writes its extrinsic there; decoder 2 reads its prior at step t from position pi(t) and writes
// its extrinsic there, i.e. deinterleaved. Each position is read by exactly one step of a half-iteration (pi is a
// permutation): in that step's chunk fill of the forward pass, again in the backward pass's chunk fill, and by the
// storing lane in the same step just before it overwrites it. The fill of a backward chunk precedes (__syncwarp) every
// store of that chunk, and later chunks hold other steps, so no value is overwritten before its last read.
// Extrinsic out of decoder 1: clip((APP - L_sys) - L_a); of decoder 2: clip((APP - L_a) - L_sys), clip to +-20, the
// reference's operation order (:407-423). The termination steps' prior is 0. The last half-iteration scatters
// decoder 2's APP through pi into out: out[pi(t)] = APP_2(t).
template <int L, int R, bool MAXLOG>
__global__ void __launch_bounds__(kWarps * 32) turbo_kernel(
    const float* __restrict__ llr, const int32_t* __restrict__ perm, float* __restrict__ out, float* ws_alpha,
    float* ws_ext, long long batch, int k, int T, int num_iter, int terminate, int hard_out, int ch, int tw,
    int alpha_on_chip, int ext_on_chip, const __grid_constant__ ConvTrellis tr) {
    constexpr int NS = L * R, G = 32 / L, conv_n = 2;
    constexpr float kClip = 20.f;
    extern __shared__ float smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int g = lane / L, l = lane % L;
    const long long cw0 = ((long long)blockIdx.x * kWarps + warp) * G;
    if (cw0 >= batch) return;
    const size_t table_floats = (size_t)G * ch * tw;
    float* tab = smem + warp * table_floats;
    float* chip = smem + kWarps * table_floats;
    float* alpha = (alpha_on_chip ? chip + (size_t)warp * G * T * NS : ws_alpha + cw0 * T * NS) + (size_t)g * T * NS;
    if (alpha_on_chip) chip += (size_t)kWarps * G * T * NS;
    // written during the kernel: plain loads, not the read-only path
    float* ext = ext_on_chip ? chip + (size_t)warp * G * k : ws_ext + cw0 * k;
    float* my_ext = ext + (size_t)g * k;
    for (int i = l; i < k; i += L) my_ext[i] = 0.f;
    const long long row_steps = 2LL * T;
    const long long cw = cw0 + g;
    // half-iteration h: decoder d = h & 1 reads its prior at step t from position t (d = 0) or pi(t) (d = 1)
    for (int h = 0; h < 2 * num_iter; ++h) {
        const int d = h & 1;
        const bool last = h + 1 == 2 * num_iter;
        const float* llr_d = llr + d * 2 * T;
        const auto pos = [&](int t) { return d ? __ldg(perm + t) : t; };
        const auto prior = [&](int gg, long long, int t) {
            return t < k ? __fmul_rn(0.5f, ext[(size_t)gg * k + pos(t)]) : 0.f;
        };
        const auto store = [&](int t, float v) {
            const int p = pos(t);
            if (last) {
                out[cw * k + p] = hard_out ? (v > 0.f ? 1.f : 0.f) : v;
                return;
            }
            const float ls = __ldg(llr_d + (cw * row_steps + t) * conv_n), la = my_ext[p];
            const float e = d ? __fsub_rn(__fsub_rn(v, la), ls) : __fsub_rn(__fsub_rn(v, ls), la);
            my_ext[p] = fminf(fmaxf(e, -kClip), kClip);
        };
        bcjr_forward<L, R, MAXLOG>(tab, alpha, llr_d, row_steps, prior, cw0, batch, T, conv_n, ch, tw, l, g, lane, tr);
        bcjr_backward<L, R, MAXLOG>(tab, alpha, llr_d, row_steps, prior, cw0, batch, T, conv_n, k, terminate, ch, tw, l,
                                    g, lane, tr, store);
    }
}

// ---- host side ------------------------------------------------------------------------------------------------------
// Checks the trellis tables of Trellis._generate_transitions ([ns, 2] int32 each) and packs them.
static int pack_trellis(const char* who, int ns, int conv_n, const int32_t* from_nodes, const int32_t* op_by_tonode,
                        const int32_t* ip_by_tonode, ConvTrellis* tr) {
    SB_CHECK_ARG(ns >= 2 && (ns & (ns - 1)) == 0 && conv_n >= 1, "%s: ns must be a power of two >= 2 and conv_n >= 1",
                 who);
    if (ns > kMaxStates || conv_n > kMaxConvN) {
        sb_set_error("%s: %d states and %d output bits per step, the limits are %d states (constraint length 9) and %d",
                     who, ns, conv_n, kMaxStates, kMaxConvN);
        return SB_EUNSUPPORTED;
    }
    SB_CHECK_ARG(from_nodes && op_by_tonode && ip_by_tonode, "%s: missing trellis tables", who);
    int32_t to[kMaxStates][2], opf[kMaxStates][2];
    for (int j = 0; j < ns; ++j) to[j][0] = to[j][1] = -1;
    for (int s = 0; s < ns; ++s) {
        const int base = (s << 1) & (ns - 1);
        uint32_t w = 0;
        for (int slot = 0; slot < 2; ++slot) {
            const int p = from_nodes[2 * s + slot], op = op_by_tonode[2 * s + slot], ip = ip_by_tonode[2 * s + slot];
            SB_CHECK_ARG((p & ~1) == base && op >= 0 && op < (1 << conv_n) && (ip == 0 || ip == 1),
                         "%s: the trellis tables are not those of a rate-1/%d shift register with the newest bit as "
                         "the state's MSB (state %d)", who, conv_n, s);
            SB_CHECK_ARG(to[p][ip] < 0, "%s: state %d has two transitions for input %d", who, p, ip);
            to[p][ip] = s;
            opf[p][ip] = op;
            w |= (uint32_t)op << (8 * slot) | (uint32_t)ip << (17 + slot);
            if (slot == 0) w |= (uint32_t)(p & 1) << 16;
        }
        SB_CHECK_ARG(from_nodes[2 * s] != from_nodes[2 * s + 1], "%s: state %d lists one predecessor twice", who, s);
        tr->to[s] = w;
    }
    for (int j = 0; j < ns; ++j) {
        // both inputs lead somewhere (checked above: 2 ns transitions, none repeated) and to different states
        SB_CHECK_ARG(to[j][0] >= 0 && to[j][1] >= 0 && to[j][0] != to[j][1], "%s: state %d lacks a transition", who, j);
        tr->from[j] = (uint32_t)opf[j][0] | (uint32_t)opf[j][1] << 8 | (uint32_t)(to[j][0] >= ns / 2) << 16;
    }
    for (int s = ns; s < kMaxStates; ++s) tr->to[s] = tr->from[s] = 0;
    return SB_OK;
}

static int check_shape(const char* who, long long batch, int num_syms, int conv_n) {
    SB_CHECK_ARG(batch >= 0 && num_syms >= 1, "%s: bad arguments (batch >= 0, num_syms >= 1)", who);
    if ((long long)num_syms * conv_n > INT32_MAX) {
        sb_set_error("%s: %lld codeword bits, the limit is 2^31 - 1", who, (long long)num_syms * conv_n);
        return SB_EUNSUPPORTED;
    }
    return SB_OK;
}

template <class F>
static int dispatch_states(int ns, F&& f) {
    switch (ns) {
        case 2: return f(std::integral_constant<int, 2>{}, std::integral_constant<int, 1>{});
        case 4: return f(std::integral_constant<int, 4>{}, std::integral_constant<int, 1>{});
        case 8: return f(std::integral_constant<int, 8>{}, std::integral_constant<int, 1>{});
        case 16: return f(std::integral_constant<int, 16>{}, std::integral_constant<int, 1>{});
        case 32: return f(std::integral_constant<int, 32>{}, std::integral_constant<int, 1>{});
        case 64: return f(std::integral_constant<int, 32>{}, std::integral_constant<int, 2>{});
        case 128: return f(std::integral_constant<int, 32>{}, std::integral_constant<int, 4>{});
        case 256: return f(std::integral_constant<int, 32>{}, std::integral_constant<int, 8>{});
    }
    return SB_EUNSUPPORTED;
}

// Off-chip state of whole CTAs (groups past the batch write theirs too); 0 when it fits in shared memory.
static size_t workspace_bytes(long long batch, int num_syms, int ns, size_t step_bytes) {
    if (batch < 0 || num_syms < 1 || ns < 2 || ns > kMaxStates || (ns & (ns - 1))) return 0;
    const WarpPlan p = warp_plan(ns, 1, num_syms, false, step_bytes);
    if (p.on_chip) return 0;
    const long long per_cta = kWarps * p.G;
    return (size_t)((batch + per_cta - 1) / per_cta * per_cta) * num_syms * step_bytes;
}

static int check_workspace(const char* who, const char* fn, void* ws, size_t ws_bytes, size_t need) {
    if (need && (!ws || ws_bytes < need)) {
        sb_set_error("%s: the workspace needs %zu bytes (%s), %zu given", who, need, fn, ws ? ws_bytes : (size_t)0);
        return SB_ENOMEM;
    }
    return SB_OK;
}

}  // namespace

extern "C" int sb_conv_encode(const float* d_u, float* d_x, int64_t batch, int32_t k, const int32_t* h_gen_poly,
                              int32_t conv_n, int32_t constraint_length, int32_t rsc, int32_t terminate,
                              void* stream) {
    const char* who = "sb_conv_encode";
    const int K = constraint_length;
    SB_CHECK_ARG(batch >= 0 && k >= 1 && conv_n >= 1 && K >= 2 && (rsc == 0 || rsc == 1) &&
                 (terminate == 0 || terminate == 1) && h_gen_poly,
                 "%s: bad arguments (batch >= 0, k >= 1, conv_n >= 1, constraint_length >= 2, rsc and terminate in "
                 "{0, 1}, gen_poly given)", who);
    if (K > 9 || conv_n > kMaxConvN) {
        sb_set_error("%s: constraint length %d and %d output bits per step, the limits are 9 and %d", who, K, conv_n,
                     kMaxConvN);
        return SB_EUNSUPPORTED;
    }
    Polys p{};
    for (int j = 0; j < conv_n; ++j) {
        SB_CHECK_ARG(h_gen_poly[j] >= 0 && h_gen_poly[j] < (1 << K), "%s: polynomial %d has more than %d bits", who, j,
                     K);
        p.g[j] = (uint32_t)h_gen_poly[j];
    }
    SB_CHECK_ARG(!rsc || (p.g[0] >> (K - 1)) & 1u, "%s: the feedback polynomial of an RSC code must start with 1", who);
    const int T = k + (terminate ? K - 1 : 0);
    const int rc = check_shape(who, batch, T, conv_n);
    if (rc) return rc;
    if (batch == 0) return SB_OK;
    SB_CHECK_ARG(d_u && d_x, "%s: null pointer", who);
    if (rsc) {
        conv_encode_rsc_kernel<<<sb_grid(batch, 128, 8), 128, 0, (cudaStream_t)stream>>>(d_u, d_x, batch, k, T, K,
                                                                                         conv_n, p);
    } else {
        conv_encode_ff_kernel<<<sb_grid(batch * T, 256, 8), 256, 0, (cudaStream_t)stream>>>(d_u, d_x, batch, k, T, K,
                                                                                             conv_n, p);
    }
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" size_t sb_viterbi_workspace_bytes(int64_t batch, int32_t num_syms, int32_t ns) {
    return ns < 2 ? 0 : workspace_bytes(batch, num_syms, ns, viterbi_step_bytes(ns));
}

extern "C" int sb_viterbi_decode(const float* d_llr, float* d_out, int64_t batch, int32_t num_syms, int32_t k,
                                 int32_t method, int32_t terminate, int32_t return_info_bits,
                                 const int32_t* h_from_nodes, const int32_t* h_op_by_tonode,
                                 const int32_t* h_ip_by_tonode, int32_t ns, int32_t conv_n, void* d_workspace,
                                 size_t workspace_bytes_given, void* stream) {
    const char* who = "sb_viterbi_decode";
    ConvTrellis tr;
    int rc = pack_trellis(who, ns, conv_n, h_from_nodes, h_op_by_tonode, h_ip_by_tonode, &tr);
    if (rc) return rc;
    rc = check_shape(who, batch, num_syms, conv_n);
    if (rc) return rc;
    SB_CHECK_ARG((method == 0 || method == 1) && (terminate == 0 || terminate == 1) &&
                 (return_info_bits == 0 || return_info_bits == 1) && k >= 1 && k <= num_syms,
                 "%s: bad arguments (method, terminate and return_info_bits in {0, 1}, 1 <= k <= num_syms)", who);
    if (batch == 0) return SB_OK;
    SB_CHECK_ARG(d_llr && d_out, "%s: null pointer", who);
    const WarpPlan p = warp_plan(ns, conv_n, num_syms, false, viterbi_step_bytes(ns));
    rc = check_workspace(who, "sb_viterbi_workspace_bytes", d_workspace, workspace_bytes_given,
                         sb_viterbi_workspace_bytes(batch, num_syms, ns));
    if (rc) return rc;
    const size_t smem = kWarps * (p.table_bytes + (p.on_chip ? p.state_bytes : 0));
    const unsigned grid = (unsigned)((batch + kWarps * p.G - 1) / (kWarps * p.G));
    return dispatch_states(ns, [&](auto LC, auto RC) {
        constexpr int L = decltype(LC)::value, RR = decltype(RC)::value;
        auto kern = method == 0 ? viterbi_kernel<L, RR, kSoft> : viterbi_kernel<L, RR, kHard>;
        if (smem > 48 * 1024) SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, kWarps * 32, smem, (cudaStream_t)stream>>>(d_llr, d_out, (uint32_t*)d_workspace, batch, num_syms,
                                                                 conv_n, k, terminate, return_info_bits, p.ch, p.tw,
                                                                 p.on_chip, tr);
        SB_LAUNCH_CHECK();
        return SB_OK;
    });
}

extern "C" size_t sb_bcjr_workspace_bytes(int64_t batch, int32_t num_syms, int32_t ns) {
    return ns < 2 ? 0 : workspace_bytes(batch, num_syms, ns, bcjr_step_bytes(ns));
}

extern "C" int sb_bcjr_decode(const float* d_llr_ch, const float* d_llr_a, float* d_out, int64_t batch,
                              int32_t num_syms, int32_t num_out, int32_t algorithm, int32_t terminate, int32_t hard_out,
                              const int32_t* h_from_nodes, const int32_t* h_op_by_tonode,
                              const int32_t* h_ip_by_tonode, int32_t ns, int32_t conv_n, void* d_workspace,
                              size_t workspace_bytes_given, void* stream) {
    const char* who = "sb_bcjr_decode";
    ConvTrellis tr;
    int rc = pack_trellis(who, ns, conv_n, h_from_nodes, h_op_by_tonode, h_ip_by_tonode, &tr);
    if (rc) return rc;
    rc = check_shape(who, batch, num_syms, conv_n);
    if (rc) return rc;
    SB_CHECK_ARG(algorithm >= 0 && algorithm <= 2 && (terminate == 0 || terminate == 1) &&
                 (hard_out == 0 || hard_out == 1) && num_out >= 1 && num_out <= num_syms,
                 "%s: bad arguments (algorithm in {0, 1, 2}, terminate and hard_out in {0, 1}, 1 <= num_out <= "
                 "num_syms)", who);
    if (batch == 0) return SB_OK;
    SB_CHECK_ARG(d_llr_ch && d_out, "%s: null pointer", who);
    const WarpPlan p = warp_plan(ns, conv_n, num_syms, true, bcjr_step_bytes(ns));
    rc = check_workspace(who, "sb_bcjr_workspace_bytes", d_workspace, workspace_bytes_given,
                         sb_bcjr_workspace_bytes(batch, num_syms, ns));
    if (rc) return rc;
    const size_t smem = kWarps * (p.table_bytes + (p.on_chip ? p.state_bytes : 0));
    const unsigned grid = (unsigned)((batch + kWarps * p.G - 1) / (kWarps * p.G));
    return dispatch_states(ns, [&](auto LC, auto RC) {
        constexpr int L = decltype(LC)::value, RR = decltype(RC)::value;
        auto kern = algorithm == 2 ? bcjr_kernel<L, RR, true> : bcjr_kernel<L, RR, false>;
        if (smem > 48 * 1024) SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, kWarps * 32, smem, (cudaStream_t)stream>>>(d_llr_ch, d_llr_a, d_out, (float*)d_workspace, batch,
                                                                 num_syms, conv_n, num_out, terminate, hard_out, p.ch,
                                                                 p.tw, p.on_chip, tr);
        SB_LAUNCH_CHECK();
        return SB_OK;
    });
}

// ---- turbo decoder (host) -------------------------------------------------------------------------------------------
// The interleaver pi of a turbo code, checked on the host at creation, so that the kernel only ever reads validated
// indices.
struct sb_turbo_perm {
    int k = 0;
    std::vector<int32_t> h;
    mutable DeviceTables tables;   // device copies of h
};

namespace {

// Extrinsic buffer: k floats per codeword, in shared memory when kWarps of them fit the on-chip budget.
struct TurboPlan {
    WarpPlan w;
    size_t ext_bytes;   // per warp
    bool ext_on_chip;
};

TurboPlan turbo_plan(int ns, int k, int T) {
    TurboPlan p;
    p.w = warp_plan(ns, 2, T, true, bcjr_step_bytes(ns));
    p.ext_bytes = (size_t)p.w.G * k * sizeof(float);
    p.ext_on_chip = kWarps * p.ext_bytes <= kOnChipBytes;
    return p;
}

int turbo_syms(int k, int terminate, int ns) { return k + (terminate ? 31 - __builtin_clz((unsigned)ns) : 0); }

}  // namespace

extern "C" int sb_turbo_perm_create(sb_turbo_perm** out, const int32_t* h_perm, int32_t k) {
    const char* who = "sb_turbo_perm_create";
    SB_CHECK_ARG(out && h_perm && k >= 1, "%s: bad arguments (out and h_perm given, k >= 1)", who);
    std::vector<char> seen(k, 0);
    for (int i = 0; i < k; ++i) {
        const int32_t v = h_perm[i];
        SB_CHECK_ARG(v >= 0 && v < k, "%s: h_perm[%d] = %d is outside 0 ... %d", who, i, v, k - 1);
        SB_CHECK_ARG(!seen[v], "%s: h_perm is not a permutation (%d appears twice)", who, v);
        seen[v] = 1;
    }
    auto* p = new sb_turbo_perm();
    p->k = k;
    p->h.assign(h_perm, h_perm + k);
    p->tables.set(p->h);
    *out = p;
    return SB_OK;
}

extern "C" void sb_turbo_perm_destroy(sb_turbo_perm* p) { delete p; }

extern "C" size_t sb_turbo_workspace_bytes(int64_t batch, int32_t k, int32_t terminate, int32_t ns) {
    if (batch < 0 || k < 1 || ns < 2 || ns > kMaxStates || (ns & (ns - 1)) || (terminate != 0 && terminate != 1))
        return 0;
    const int T = turbo_syms(k, terminate, ns);
    const TurboPlan p = turbo_plan(ns, k, T);
    const long long per_cta = kWarps * p.w.G;
    const long long rows = (batch + per_cta - 1) / per_cta * per_cta;
    return (p.w.on_chip ? 0 : (size_t)rows * T * bcjr_step_bytes(ns)) +
           (p.ext_on_chip ? 0 : (size_t)rows * k * sizeof(float));
}

extern "C" int sb_turbo_decode(const float* d_llr, const sb_turbo_perm* perm, float* d_out, int64_t batch, int32_t k,
                               int32_t num_iter, int32_t algorithm, int32_t terminate, int32_t hard_out,
                               const int32_t* h_from_nodes, const int32_t* h_op_by_tonode,
                               const int32_t* h_ip_by_tonode, int32_t ns, int32_t conv_n, void* d_workspace,
                               size_t workspace_bytes_given, void* stream) {
    const char* who = "sb_turbo_decode";
    ConvTrellis tr;
    int rc = pack_trellis(who, ns, conv_n, h_from_nodes, h_op_by_tonode, h_ip_by_tonode, &tr);
    if (rc) return rc;
    if (conv_n != 2) {
        sb_set_error("%s: the component codes have %d output bits per step, turbo decoding needs rate 1/2", who, conv_n);
        return SB_EUNSUPPORTED;
    }
    SB_CHECK_ARG(batch >= 0 && k >= 1 && num_iter >= 0 && algorithm >= 0 && algorithm <= 2 &&
                 (terminate == 0 || terminate == 1) && (hard_out == 0 || hard_out == 1),
                 "%s: bad arguments (batch >= 0, k >= 1, num_iter >= 0, algorithm in {0, 1, 2}, terminate and "
                 "hard_out in {0, 1})", who);
    SB_CHECK_ARG(perm && perm->k == k, "%s: the interleaver handle is missing or not of length k = %d", who, k);
    const int T = turbo_syms(k, terminate, ns);
    rc = check_shape(who, batch, 2 * T, conv_n);
    if (rc) return rc;
    if (batch == 0) return SB_OK;
    SB_CHECK_ARG(d_llr && d_out, "%s: null pointer", who);
    const TurboPlan p = turbo_plan(ns, k, T);
    const size_t need = sb_turbo_workspace_bytes(batch, k, terminate, ns);
    rc = check_workspace(who, "sb_turbo_workspace_bytes", d_workspace, workspace_bytes_given, need);
    if (rc) return rc;
    if (num_iter == 0) {                                    // the reference returns zeros (its llr_2i starts at 0)
        SB_CUDA(cudaMemsetAsync(d_out, 0, (size_t)batch * k * sizeof(float), (cudaStream_t)stream));
        return SB_OK;
    }
    const DeviceTables::Copy* d = nullptr;
    rc = perm->tables.get(&d);
    if (rc) return rc;
    const long long per_cta = kWarps * p.w.G;
    const long long rows = (batch + per_cta - 1) / per_cta * per_cta;
    float* ws_alpha = (float*)d_workspace;
    float* ws_ext = (float*)d_workspace + (p.w.on_chip ? 0 : (size_t)rows * T * ns);
    const size_t smem = kWarps * (p.w.table_bytes + (p.w.on_chip ? p.w.state_bytes : 0) +
                                  (p.ext_on_chip ? p.ext_bytes : 0));
    const unsigned grid = (unsigned)(rows / per_cta);
    return dispatch_states(ns, [&](auto LC, auto RC) {
        constexpr int L = decltype(LC)::value, RR = decltype(RC)::value;
        auto kern = algorithm == 2 ? turbo_kernel<L, RR, true> : turbo_kernel<L, RR, false>;
        if (smem > 48 * 1024) SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, kWarps * 32, smem, (cudaStream_t)stream>>>(d_llr, d->at<int32_t>(0), d_out, ws_alpha, ws_ext, batch,
                                                                 k, T, num_iter, terminate, hard_out, p.w.ch, p.w.tw,
                                                                 p.w.on_chip, p.ext_on_chip, tr);
        SB_LAUNCH_CHECK();
        return SB_OK;
    });
}
