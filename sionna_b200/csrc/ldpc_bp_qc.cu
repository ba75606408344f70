// ldpc_bp_qc.cu -- belief-propagation fast path for quasi-cyclic (5G NR) decoding graphs on sm_90a.
//
// Same algorithm, arithmetic and results as ldpc_bp.cu (one CTA per codeword, messages resident in shared memory,
// in-place flooding; reference: /root/reference/src/sionna/phy/fec/ldpc/decoding.py:416-637, 681-1166) but the
// quasi-cyclic structure of the lifted base graph (encoding.py:322-352: every base entry (r, c, s) is a ZxZ identity
// shifted by s) replaces every index table by arithmetic:
//   * message slot of base entry `be` and check offset i (CN = r*Z + i):   be*Z + i
//     - CN (r, i) walks its edges with a constant stride of Z words: no loads of indices at all;
//     - VN (c, j) reaches the edge of entry (r, c, s) at be*Z + ((j - s) mod Z): one broadcast LDS of a table entry
//       in address form + 3 integer ops (vn_addr); 32 consecutive VNs hit 32 consecutive words (mod the wrap):
//       conflict free.
//   * a warp owns 32 consecutive checks (or variables) of ONE base row (column): degree and table entries are
//     warp-uniform, so the min-sum update keeps the whole row in registers (fully unrolled degree buckets, one
//     shared-memory read and one write per edge) and the VN update keeps addresses + messages in registers.
//   * rows / columns are processed in order of decreasing degree, dealt cyclically to the warps (load balance).
// Partial trailing blocks (pruned graphs whose size is not a multiple of Z) are handled with per-entry limits.
// Summation orders (ascending VN inside a CN, ascending CN inside a VN) are those of ldpc_bp.cu, so both kernels
// and the CPU oracle (math_mode 1, order "kernel") agree bit for bit.
#include <algorithm>
#include <climits>
#include <iterator>
#include <numeric>
#include <vector>
#include "sb_common.h"
#include "sb_math.h"
#include "sb_math2.cuh"
#include "ldpc_graph.h"
#include "ldpc_rules.cuh"

namespace {

// ---- degree classes, read by the host planner (sb_ldpc_graph_set_qc) and by the kernel ---------------------------
// Rows and columns are processed class by class, heaviest first. Class k holds the degrees d with
// kMax[k + 1] < d <= kMax[k]; its code keeps a row (column) of up to kMax[k] edges in registers. kLoop marks the
// classes that take any larger degree and run loop code instead.
constexpr int kLoop = INT_MAX;
// CN classes: > 20 (loop), <= 20, <= 12, <= 8, <= 4
constexpr int kRowMax[] = {kLoop, 20, 12, 8, 4};
// VN classes: 0...6 by degree; 7...9 for columns with an edge into a partial (pruning-cut) block row, whose edges need
// a per-entry limit; 10: degree-1 columns whose update is fused into the CN phase (the last edge of their row).
constexpr int kColCut = 7, kColFused = 10;
constexpr int kColMax[] = {kLoop, 32, 20, 12, 8, 4, 2, kLoop, 12, 4, 1};
constexpr int kRowClasses = (int)std::size(kRowMax);
constexpr int kColClasses = (int)std::size(kColMax);

constexpr bool decreasing(const int* m, int lo, int hi) {
    for (int k = lo + 1; k < hi; ++k)
        if (m[k] >= m[k - 1]) return false;
    return true;
}
static_assert(decreasing(kRowMax, 0, kRowClasses), "row class bounds must decrease");
static_assert(decreasing(kColMax, 0, kColCut) && decreasing(kColMax, kColCut, kColFused), "column class bounds must decrease");
static_assert(kColFused == kColClasses - 1 && kColMax[kColFused] == 1, "the fused class holds degree-1 columns only");

// the lightest class of [lo, hi) whose bound holds degree d
constexpr int degree_class(const int* m, int lo, int hi, int d) {
    int k = hi - 1;
    while (k > lo && d > m[k]) --k;
    return k;
}

struct QcParams {
    int Z, n_rows, n_cols, nnz, N, E, E_alloc, n_in, n_out;
    int row_cls_end[kRowClasses];   // processing order: rows of class k are [row_cls_end[k-1], row_cls_end[k])
    int col_cls_end[kColClasses];
    int row_cls_mod[kRowClasses];   // (first index of class k) mod G, G = warp groups of this launch
    int col_cls_mod[kColClasses];
    const int4* row_info;    // {first base entry, deg, zrow, fused VN base (c*Z | s << 16... see host) or -1}
    const int4* col_info;    // {first col-edge, deg, zcol, c*Z}
    const int2* col_edge;    // {be*Z*4, s*4 | (zrow*4) << 16}, ascending base row inside a column
    const int* in_idx;       // [N] natural VN order
    const int* out_pos;      // [N]
    const int* slot_of_edge; // [E] reference edge -> slot
    const float* llr;
    float* out;
    float* state_out;
    long long B;
    int num_iter, hard_out, use_tma;
    int early;               // opt-in early termination by the syndrome of the hard decisions (see the kernel)
    int* iters_out;          // [B] iterations actually run per codeword, or nullptr
    const int2* row_edge;    // [nnz] per base entry (processing order): {column * Z, shift}  (syndrome pass only)
    int tab_rep;             // copies of the phi log table in shared memory (16, 8 or 1; 0: rule does not use it)
    float offset, llr_max;
    int open;                // boxplus-phi: run the opening iterations 0 and 1 on the punctured columns (see cn_open_pass)
    const int* open_tab;     // [n_rows] punctured edge positions of each row (bit l: edge l), then [n_cols] punctured flags
};

// Message invariant of this kernel: a v2c message is never -0.0f. The initial v2c is canonicalised (llr + 0.0f) and
// the VN update clip(x_tot - c2v) cannot yield -0.0f because x_tot = (0 + sum c2v) + llr is never -0.0f. Hence in the
// CN phase  sign bit set <=> v2c < 0, which is the reference's sign() with sign(0) := +1 (decoding.py:800-804, :1129).
// (c2v messages may be -0.0f; the VN arithmetic does not depend on the sign of a zero.)

// ---- check-node updates on the edges pm[0], pm[Z], pm[2Z], ... of one check ------------------------------------
// boxplus-phi (decoding.py:1126-1166), two independent edges per step (sb_math2.cuh).
// Exact strength reductions (outputs are bit-identical, only instructions are saved), all decided warp-uniformly:
//   (1) |x| >= 16.635532 (the phi clipping bound, :1113)  =>  phi(|x|) == +0 exactly              [saturated inputs]
//       The voting variant uses the wider exact bound |x| >= 14.7117348 (SB_PHI_ZERO).
//   (2) p_e == 0  =>  P - p_e == P exactly  =>  phi(P - p_e) == phi(P), evaluated once per check
//   (3) P - p_e <= 8.5e-8 (lower clipping bound)  =>  phi(P - p_e) == phi(8.5e-8) == phi_max
// Once a codeword has converged most VN->CN messages except those of degree-1 VNs sit at +-llr_max >= 16.64, and a
// check costs ~2 phi evaluations instead of 2*deg; the per-iteration cost therefore depends on the channel SNR.
#define SB_PHI_HI 16.635532f
// Least fp32 x above which phi(x) is +0 for every x in this arithmetic: e^x + 1 and e^x - 1 round to the same float
// and the two logs cancel. Below it phi is not monotone (x = 14.7117338 gives 2^-20). Checked over every fp32 value up
// to 16.635532 against the oracle and on the device by tests/test_ldpc_qc_kernel_gpu.py.
#define SB_PHI_ZERO 14.7117348f
// The two passes of the update, written once for every variant below: pass 1 on the edge words b = bits(x), pass 2 on
// the staged words w = phi(|x|) | sign(x); one edge pair (two independent phi chains, sb_math2.cuh) or one edge.
// Pass 1: phi(|x|), summed into P in ascending VN order (:1150); returns w (phi >= 0: the sign bit carries sign(x)).
// `probe(|x0|, |x1|)` runs between the phi pair and the sum (the plain variant's saturation vote).
template <class LT, class Probe>
__device__ __forceinline__ uint2 phi_pass1_pair(unsigned b0, unsigned b1, float& P, const LT& lt, Probe probe) {
    const float a0 = __uint_as_float(b0 & 0x7fffffffu), a1 = __uint_as_float(b1 & 0x7fffffffu);
    const float2 p = sb_phif2(make_float2(a0, a1), lt);
    probe(a0, a1);
    P = __fadd_rn(P, p.x);
    P = __fadd_rn(P, p.y);
    return make_uint2(__float_as_uint(p.x) | (b0 & 0x80000000u), __float_as_uint(p.y) | (b1 & 0x80000000u));
}
template <class LT>
__device__ __forceinline__ unsigned phi_pass1(unsigned b0, float& P, const LT& lt) {
    const float p = sb_phif_s(__uint_as_float(b0 & 0x7fffffffu), lt);
    P = __fadd_rn(P, p);
    return __float_as_uint(p) | (b0 & 0x80000000u);
}
// Pass 2: phi((-p) + P) (:1155), clipped, sign(x) * prod(signs) (:1161-1163); par holds the product in bit 31.
template <class LT>
__device__ __forceinline__ uint2 phi_pass2_pair(unsigned w0, unsigned w1, float P, unsigned par, float clip, const LT& lt) {
    const float2 m = fadd2(make_float2(__uint_as_float(w0 | 0x80000000u), __uint_as_float(w1 | 0x80000000u)),
                           make_float2(P, P));
    const float2 y = sb_phif2(m, lt);
    return make_uint2(__float_as_uint(fminf(y.x, clip)) | ((w0 ^ par) & 0x80000000u),
                      __float_as_uint(fminf(y.y, clip)) | ((w1 ^ par) & 0x80000000u));
}
template <class LT>
__device__ __forceinline__ unsigned phi_pass2(unsigned w0, float P, unsigned par, float clip, const LT& lt) {
    const float y = sb_phif_s(__fadd_rn(__uint_as_float(w0 | 0x80000000u), P), lt);
    return __float_as_uint(fminf(y, clip)) | ((w0 ^ par) & 0x80000000u);
}
__device__ __forceinline__ unsigned ldw(const float* q) { return __float_as_uint(*q); }
__device__ __forceinline__ void stw(float* q, unsigned w) { *q = __uint_as_float(w); }

// Plain variant: every edge is evaluated. One vote per check on its first edge pair probes for saturation and raises
// *sat_flag, which makes the CTA run the voting pass (cn_vote_pass) from the next iteration on.
// Out of line on purpose (both this and cn_vote_row): the five degree classes then share ONE copy of the loops (the
// kernel is bound by instruction fetch as much as by issue: 12.35 -> 11.85 ms per 4096 codewords at 2 dB; making phi
// itself a call costs more than it saves, 12.8 ms). Two edge pairs per loop trip. The log table is passed by value, so
// its lane offset stays in a register instead of going through the stack.
template <class LT>
__device__ __noinline__ void cn_phi_qc(float* pm, int Z, int deg, float clip, int* sat_flag, LT lt) {
    const unsigned am = __activemask();                   // lanes of this warp working on the same block row
    float P = 0.f;
    unsigned par = 0;
    int l = 0;
#pragma unroll 2
    for (; l + 1 < deg; l += 2) {
        float* q0 = pm + l * Z;
        float* q1 = q0 + Z;
        const unsigned b0 = ldw(q0), b1 = ldw(q1);
        par ^= b0 ^ b1;
        const uint2 w = phi_pass1_pair(b0, b1, P, lt, [&](float a0, float a1) {
            if (l == 0 && __all_sync(am, a0 >= SB_PHI_HI && a1 >= SB_PHI_HI)) *sat_flag = 1;   // probe (benign race)
        });
        stw(q0, w.x);
        stw(q1, w.y);
    }
    if (l < deg) {
        float* q0 = pm + l * Z;
        const unsigned b0 = ldw(q0);
        par ^= b0;
        stw(q0, phi_pass1(b0, P, lt));
    }
    par &= 0x80000000u;
    l = 0;
#pragma unroll 2
    for (; l + 1 < deg; l += 2) {
        float* q0 = pm + l * Z;
        float* q1 = q0 + Z;
        const uint2 y = phi_pass2_pair(ldw(q0), ldw(q1), P, par, clip, lt);
        stw(q0, y.x);
        stw(q1, y.y);
    }
    if (l < deg) stw(pm + l * Z, phi_pass2(ldw(pm + l * Z), P, par, clip, lt));
}

// Voting variant (deg <= 32), for the iterations after the probe saw a saturated pair. A read pass (cn_vote_pass) builds
// the row's union mask U: bit l is set if |x_l| < SB_PHI_ZERO in any lane of the warp. U is warp-uniform, and only its
// k positions are evaluated:
//   * U holds no edge but the last (the common row once a codeword has converged): every other edge has phi = +0 (1),
//     so P = p_last exactly; those edges get phi(P) and the last edge phi(P - p_last) = phi(+0) = phi_max (3). Two phi
//     per row.
//   * otherwise (cn_vote_row), walking U in ascending order two at a time: phi(|x_l|) for l in U, summed into P in
//     that order. A position outside U has phi = +0 in every lane (1), and P + (+0) == P, so P is bit-identical to the
//     sum over all edges in ascending VN order. Then phi(P - p_l) for l in U, each lane on its own values: where (2) or
//     (3) holds the evaluation itself gives what the rule gives (-0 + P == P; the clamp of phi maps P - p_l <= 8.5e-8
//     to phi_max). Every position outside U gets phi(P - 0) = phi(P), evaluated once. 2k + 1 phi per row.
// Outputs outside U take their sign from the lane's sign mask S (bit l = sign of x_l), so those edges are written
// without being read again; the row's sign parity is popc(S) & 1.
__device__ __forceinline__ unsigned vote_sign(unsigned S, int l, unsigned par) { return ((S >> l) << 31) ^ par; }

// The 2k + 1 walk of a voting row whose U holds an edge other than the last, given this lane's sign mask S. The two-phi
// rows are handled inline in cn_vote_pass.
template <class LT>
__device__ __noinline__ void cn_vote_row(float* pm, int Z, int deg, unsigned U, unsigned S, float clip, LT lt) {
    const unsigned par = (unsigned)__popc(S) << 31;
    float P = 0.f;
    unsigned u = U;
    for (; u & (u - 1); u &= u - 1) {                     // two or more positions left: the lowest two
        float* q0 = pm + (__ffs(u) - 1) * Z;
        u &= u - 1;
        float* q1 = pm + (__ffs(u) - 1) * Z;
        const uint2 w = phi_pass1_pair(ldw(q0), ldw(q1), P, lt, [](float, float) {});
        stw(q0, w.x);
        stw(q1, w.y);
    }
    if (u) {
        float* q0 = pm + (__ffs(u) - 1) * Z;
        stw(q0, phi_pass1(ldw(q0), P, lt));
    }
    const unsigned rest = ~U & (0xffffffffu >> (32 - deg));
    if (rest) {
        const unsigned y = __float_as_uint(fminf(sb_phif_s(P, lt), clip));
        for (unsigned r = rest; r; r &= r - 1) {
            const int l = __ffs(r) - 1;
            stw(pm + l * Z, y | vote_sign(S, l, par));
        }
    }
    for (u = U; u & (u - 1); u &= u - 1) {
        float* q0 = pm + (__ffs(u) - 1) * Z;
        u &= u - 1;
        float* q1 = pm + (__ffs(u) - 1) * Z;
        const uint2 y = phi_pass2_pair(ldw(q0), ldw(q1), P, par, clip, lt);
        stw(q0, y.x);
        stw(q1, y.y);
    }
    if (u) {
        float* q0 = pm + (__ffs(u) - 1) * Z;
        stw(q0, phi_pass2(ldw(q0), P, par, clip, lt));
    }
}

// Exact-degree variant of the plain cn_phi_qc (deg == D, the degrees 3...8 of the 5G base graphs): phi(|x|) of the
// whole row stays in registers between the two passes (no STS in pass 1, no LDS / address arithmetic in pass 2), both
// passes fully unrolled. Same operation sequence per element as cn_phi_qc, hence bit-identical. The voting variant has
// no such code: skipped straight-line code still has to be fetched, a skipped loop body does not, and the kernel is
// instruction-cache bound.
template <int D, class LT>
__device__ __forceinline__ void cn_phi_qc_reg(float* pm, int Z, float clip, int* sat_flag, const LT& lt) {
    const unsigned am = __activemask();
    unsigned w[D];                                        // phi(|x|) bits | sign(x)
    float P = 0.f;
    unsigned par = 0;
#pragma unroll
    for (int l = 0; l + 1 < D; l += 2) {
        const unsigned b0 = ldw(pm + l * Z), b1 = ldw(pm + (l + 1) * Z);
        par ^= b0 ^ b1;
        const uint2 q = phi_pass1_pair(b0, b1, P, lt, [&](float a0, float a1) {
            if (l == 0 && __all_sync(am, a0 >= SB_PHI_HI && a1 >= SB_PHI_HI)) *sat_flag = 1;
        });
        w[l] = q.x;
        w[l + 1] = q.y;
    }
    if (D & 1) {
        const unsigned b0 = ldw(pm + (D - 1) * Z);
        par ^= b0;
        w[D - 1] = phi_pass1(b0, P, lt);
    }
    par &= 0x80000000u;
#pragma unroll
    for (int l = 0; l + 1 < D; l += 2) {
        const uint2 y = phi_pass2_pair(w[l], w[l + 1], P, par, clip, lt);
        stw(pm + l * Z, y.x);
        stw(pm + (l + 1) * Z, y.y);
    }
    if (D & 1) stw(pm + (D - 1) * Z, phi_pass2(w[D - 1], P, par, clip, lt));
}

// deg == one of DS: the register variant of that degree; returns whether it ran
template <class LT, int... DS>
__device__ __forceinline__ bool cn_phi_reg_of(float* pm, int Z, int deg, float clip, int* sat_flag, const LT& lt) {
    return ((deg == DS && (cn_phi_qc_reg<DS, LT>(pm, Z, clip, sat_flag, lt), true)) || ...);
}

// the plain variant of a row of class CLS
template <int CLS, class LT>
__device__ __forceinline__ void cn_phi_dispatch(float* pm, int Z, int deg, float clip, int* sat_flag, const LT& lt) {
    if (CLS == 4 && cn_phi_reg_of<LT, 3, 4>(pm, Z, deg, clip, sat_flag, lt)) return;
    if (CLS == 3 && cn_phi_reg_of<LT, 5, 6, 7, 8>(pm, Z, deg, clip, sat_flag, lt)) return;
    cn_phi_qc<LT>(pm, Z, deg, clip, sat_flag, lt);
}

// Check-node edges pm[0], pm[Z], pm[2Z], ... for the rules of ldpc_rules.cuh
struct StrideEdges {
    float* pm;
    int Z;
    __device__ __forceinline__ float in(int l) const { return pm[l * Z]; }
    __device__ __forceinline__ void out(int l, float v) const { pm[l * Z] = v; }
    __device__ __forceinline__ float staged(int l) const { return pm[l * Z]; }
};

// (offset-)min-sum with the row in registers. Preconditions checked on the host: |message| <= llr_max and
// (deg-1)*llr_max < 99000, so the reference's 1e5 sentinel logic (decoding.py:849-887) reduces exactly to
//   unique minimum -> that edge gets fl(fl(m2 - m1) + m1), all others m1;  repeated minimum -> all edges m1.
// Offset, max(.,0) and clipping act on only two distinct magnitudes and are hoisted out of the edge loop.
// minsum_mags: those two magnitudes from the row's two smallest incoming ones m1 <= m2, {elsewhere, at the minimum}.
__device__ __forceinline__ float2 minsum_mags(float m1, float m2, int deg, float clip, float offset) {
    float min_e = (m2 == m1) ? m1 : __fadd_rn(__fsub_rn(m2, m1), m1);
    if (deg == 1) min_e = __fadd_rn(100000.f, m1);
    return make_float2(fminf(fmaxf(__fsub_rn(m1, offset), 0.f), clip), fminf(fmaxf(__fsub_rn(min_e, offset), 0.f), clip));
}
// outgoing message of the edge with incoming message v; par holds the row's sign parity in bit 31
__device__ __forceinline__ float minsum_msg(float v, float m1, float2 o, unsigned par) {
    const float mag = (fabsf(v) == m1) ? o.y : o.x;
    return __uint_as_float(__float_as_uint(mag) | ((__float_as_uint(v) ^ par) & 0x80000000u));
}
template <int DMAX, bool EXACT>                           // EXACT: deg == DMAX, no per-edge guards
__device__ __forceinline__ void cn_minsum_qc(float* pm, int Z, int deg, float clip, float offset) {
    float x[DMAX];                                        // every element is assigned unconditionally (registers)
    float m1 = INFINITY, m2 = INFINITY;
    unsigned par = 0;
#pragma unroll
    for (int l = 0; l < DMAX; ++l) {
        float v = INFINITY;                               // neutral: never the minimum, sign +
        if (EXACT || l < deg) v = pm[l * Z];              // warp-uniform predicate
        x[l] = v;
        float a = fabsf(v);
        m2 = fminf(m2, fmaxf(m1, a));
        m1 = fminf(m1, a);
        par ^= __float_as_uint(v);
    }
    par &= 0x80000000u;
    const float2 o = minsum_mags(m1, m2, deg, clip, offset);
#pragma unroll
    for (int l = 0; l < DMAX; ++l) {
        const float y = minsum_msg(x[l], m1, o, par);
        if (EXACT || l < deg) pm[l * Z] = y;
    }
}

// generic-degree fallback (re-reads shared memory instead of holding the row in registers)
__device__ __forceinline__ void cn_minsum_qc_loop(float* pm, int Z, int deg, float clip, float offset) {
    float m1 = INFINITY, m2 = INFINITY;
    unsigned par = 0;
    for (int l = 0; l < deg; ++l) {
        float v = pm[l * Z];
        float a = fabsf(v);
        m2 = fminf(m2, fmaxf(m1, a));
        m1 = fminf(m1, a);
        par ^= __float_as_uint(v);
    }
    par &= 0x80000000u;
    const float2 o = minsum_mags(m1, m2, deg, clip, offset);
    for (int l = 0; l < deg; ++l) pm[l * Z] = minsum_msg(pm[l * Z], m1, o, par);
}

template <int RULE, int CLS, class LT>
__device__ __forceinline__ void cn_qc(float* pm, int Z, int deg, float clip, float offset, int* sat_flag, const LT& lt) {
    if constexpr (RULE == SB_CN_BOXPLUS_PHI) {
        cn_phi_dispatch<CLS, LT>(pm, Z, deg, clip, sat_flag, lt);
    } else if constexpr (RULE == SB_CN_BOXPLUS) {
        cn_tanh(StrideEdges{pm, Z}, deg, clip);
    } else {
        constexpr int D = kRowMax[CLS];
        const float off = (RULE == SB_CN_MINSUM) ? 0.f : offset;
        // exact-degree code for the degrees of the 5G base graphs, guarded buckets otherwise (deg is warp-uniform)
        if constexpr (D == kLoop) {
            cn_minsum_qc_loop(pm, Z, deg, clip, off);
        } else if constexpr (CLS == 4) {
            if (deg == 3) cn_minsum_qc<3, true>(pm, Z, deg, clip, off);
            else if (deg == 4) cn_minsum_qc<4, true>(pm, Z, deg, clip, off);
            else cn_minsum_qc<D, false>(pm, Z, deg, clip, off);
        } else if constexpr (CLS == 3) {                  // 5...8: every degree of the class is exact
            if (deg == 5) cn_minsum_qc<5, true>(pm, Z, deg, clip, off);
            else if (deg == 6) cn_minsum_qc<6, true>(pm, Z, deg, clip, off);
            else if (deg == 7) cn_minsum_qc<7, true>(pm, Z, deg, clip, off);
            else cn_minsum_qc<D, true>(pm, Z, deg, clip, off);
        } else if constexpr (CLS == 2) {
            if (deg == 9) cn_minsum_qc<9, true>(pm, Z, deg, clip, off);
            else if (deg == 10) cn_minsum_qc<10, true>(pm, Z, deg, clip, off);
            else cn_minsum_qc<D, false>(pm, Z, deg, clip, off);
        } else {
            if (deg == 19) cn_minsum_qc<19, true>(pm, Z, deg, clip, off);
            else cn_minsum_qc<D, false>(pm, Z, deg, clip, off);
        }
    }
}

// explicit shared-window accesses with 32-bit addresses (no generic-address arithmetic in the hot loops)
__device__ __forceinline__ float lds_f32(uint32_t a) {
    float v;
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a));
    return v;
}
__device__ __forceinline__ void sts_f32(uint32_t a, float v) {
    asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory");
}
__device__ __forceinline__ int2 lds_i2(uint32_t a) {
    int2 v;
    asm volatile("ld.shared.v2.s32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a));
    return v;
}

// ---- variable-node update (decoding.py:714-732) for VN (c, j) -------------------------------------------------
// ce_s is the 32-bit shared-window address of the column's first table entry. The shared-memory copy of the column
// table holds per edge {x, y}: x = address of message slot be*Z minus 4*s, y = 4*s << 16 | 4*zrow. With j4 = 4*j and
// jk = j4 << 16 | 0xffff (per thread, the same for every edge) the edge's message is at x + (jk < y ? j4 + 4*Z : j4):
// jk < y holds exactly when j < s, where (j - s) mod Z wraps. One compare, one select and one add per edge.
struct VnLane {
    uint32_t j4, j4w, jk;                                 // j4w = j4 + 4*Z, the offset of a wrapped edge
};
__device__ __forceinline__ uint32_t vn_addr(int2 e, const VnLane& v) {
    return (uint32_t)e.x + (v.jk < (uint32_t)e.y ? v.j4w : v.j4);
}
// the edge exists: check offset (j - s) mod Z below the block row's zrow (partial block rows only)
__device__ __forceinline__ bool vn_in_row(int2 e, uint32_t addr, const VnLane& v) {
    return addr - (uint32_t)e.x - ((uint32_t)e.y >> 16) < ((uint32_t)e.y & 0xffffu);
}

// Returns the unclipped x_tot. Branch free: table entries beyond the column's degree are not read (predicate) and their
// load, accumulate and store are predicated off.
template <int DMAX, bool CHECK, bool KEEPM, bool EXACT = false>   // EXACT: deg == DMAX and !CHECK: no guards
__device__ __forceinline__ float vn_qc(uint32_t ce_s, int deg, const VnLane& vl, float llr, float clip) {
    uint32_t addr[DMAX];
    float m[KEEPM ? DMAX : 1];
    bool on[DMAX];
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < DMAX; ++k) {
        int2 e = make_int2(0, 0);
        if (EXACT || k < deg) e = lds_i2(ce_s + 8 * k);   // warp-uniform predicate
        addr[k] = vn_addr(e, vl);
        bool ok = EXACT || ((k < deg) && (!CHECK || vn_in_row(e, addr[k], vl)));
        on[k] = ok;
        float v = 0.f;
        if (ok) v = lds_f32(addr[k]);
        if (ok) acc = __fadd_rn(acc, v);                  // :715 sequential, ascending CN
        if (KEEPM) m[KEEPM ? k : 0] = v;
    }
    float x_tot = __fadd_rn(acc, llr);                    // :716
#pragma unroll
    for (int k = 0; k < DMAX; ++k) {
        float v = 0.f;
        if (KEEPM) v = m[KEEPM ? k : 0];
        else if (on[k]) v = lds_f32(addr[k]);
        float y = clipf(__fadd_rn(-v, x_tot), clip);      // :724-729
        if (on[k]) sts_f32(addr[k], y);
    }
    return x_tot;
}

// Loop form for any degree. MODE 0: the update; MODE 1: initialisation v2c = llr (decoding.py:571), canonical +0.0 for
// punctured bits (llr = -0.0); MODE 2: `llr` stored on every edge as it is (vn_init's pass-1 words).
template <int MODE>
__device__ __forceinline__ float vn_qc_loop(uint32_t ce_s, int deg, const VnLane& vl, float llr, float clip) {
    float acc = 0.f;
    if (MODE == 0)
        for (int k = 0; k < deg; ++k) {
            const int2 e = lds_i2(ce_s + 8 * k);
            const uint32_t a = vn_addr(e, vl);
            if (vn_in_row(e, a, vl)) acc = __fadd_rn(acc, lds_f32(a));
        }
    float x_tot = __fadd_rn(acc, llr);
    for (int k = 0; k < deg; ++k) {
        const int2 e = lds_i2(ce_s + 8 * k);
        const uint32_t a = vn_addr(e, vl);
        if (vn_in_row(e, a, vl))
            sts_f32(a, (MODE == 1) ? __fadd_rn(llr, 0.f) : (MODE == 2) ? llr : clipf(__fadd_rn(-lds_f32(a), x_tot), clip));
    }
    return x_tot;
}

// VN update of a column of class CLS (kColMax). EX: exact-degree variants.
template <int CLS, bool EX>
__device__ __forceinline__ float vn_cls(uint32_t ce, int deg, const VnLane& vl, float llr, float clip) {
    constexpr int D = kColMax[CLS];
    if constexpr (D == kLoop) {
        return vn_qc_loop<0>(ce, deg, vl, llr, clip);
    } else if constexpr (CLS >= kColCut) {
        return vn_qc<D, true, true>(ce, deg, vl, llr, clip);
    } else if constexpr (D > 12) {
        // the punctured columns of base graph 1 at the rates that keep 24 block rows: exact-degree code, each message
        // read once; the guarded buckets re-read their messages instead of keeping them in registers
        if (CLS == 2 && EX && deg == 19) return vn_qc<19, false, true, true>(ce, deg, vl, llr, clip);
        if (CLS == 2 && EX && deg == 17) return vn_qc<17, false, true, true>(ce, deg, vl, llr, clip);
        return vn_qc<D, false, false>(ce, deg, vl, llr, clip);
    } else {
        // exact-degree code (no guards) for every degree up to 12; deg is warp-uniform
        if constexpr (CLS == 3) {
            if (EX && deg == 9) return vn_qc<9, false, true, true>(ce, deg, vl, llr, clip);
            if (EX && deg == 10) return vn_qc<10, false, true, true>(ce, deg, vl, llr, clip);
            if (EX && deg == 11) return vn_qc<11, false, true, true>(ce, deg, vl, llr, clip);
        } else if constexpr (CLS == 4) {
            if (EX && deg == 5) return vn_qc<5, false, true, true>(ce, deg, vl, llr, clip);
            if (EX && deg == 6) return vn_qc<6, false, true, true>(ce, deg, vl, llr, clip);
            if (EX && deg == 7) return vn_qc<7, false, true, true>(ce, deg, vl, llr, clip);
        } else if constexpr (CLS == 5) {
            if (EX && deg == 3) return vn_qc<3, false, true, true>(ce, deg, vl, llr, clip);
        } else {
            if (EX && deg == 1) return vn_qc<1, false, true, true>(ce, deg, vl, llr, clip);
        }
        return vn_qc<D, false, true, EX>(ce, deg, vl, llr, clip);
    }
}

struct WarpCtx {
    int G, grp, lane_i;
};

// first index >= start that is congruent to grp modulo G (rows/columns are dealt cyclically over ALL classes);
// start_mod = start mod G comes from the host
__device__ __forceinline__ int first_of(int start, int start_mod, const WarpCtx& w) {
    return start + (w.grp - start_mod + (w.grp < start_mod ? w.G : 0));
}

// The row's last edge goes to a degree-1 VN (row_info.w = fw >= 0): apply that VN's update right here
// (decoding.py:714-729 with the single incoming message c2v, the edge's new value at q) so the VN phase can skip the column
__device__ __forceinline__ void fused_vn(const QcParams& p, float* q, float c2v, int fw, int lane_i, const float* llr_s,
                                         float clip, unsigned char* hd) {
    int s = fw >> 16, vb = fw & 0xffff;                   // shift, column index
    int j = lane_i + s;
    j -= (j >= p.Z) ? p.Z : 0;
    float x_tot = __fadd_rn(__fadd_rn(0.f, c2v), llr_s[vb * p.Z + j]);
    *q = clipf(__fadd_rn(-c2v, x_tot), clip);
    if (hd) hd[vb * p.Z + j] = 0.f >= x_tot ? 1 : 0;
}

template <int RULE, int CLS, class LT>
__device__ __forceinline__ void cn_class(const QcParams& p, const WarpCtx& w, float* msg, const float* llr_s,
                                         const int4* s_row, int start, int end, float clip, bool fuse, int* sat_flag,
                                         const LT& lt, unsigned char* hd) {
    for (int rr = first_of(start, p.row_cls_mod[CLS], w); rr < end; rr += w.G) {
        int4 ri = s_row[rr];
        if (w.lane_i < ri.z) {
            float* pm = msg + ri.x * p.Z + w.lane_i;
            cn_qc<RULE, CLS, LT>(pm, p.Z, ri.y, clip, p.offset, sat_flag, lt);
            if (fuse && ri.w >= 0) {
                float* q = pm + (ri.y - 1) * p.Z;
                fused_vn(p, q, *q, ri.w, w.lane_i, llr_s, clip, hd);
            }
        }
    }
}

template <int RULE, class LT>
__device__ __forceinline__ void cn_all(const QcParams& p, const WarpCtx& w, float* msg, const float* llr_s,
                                       const int4* s_row, float clip, bool fuse, int* sat_flag, const LT& lt,
                                       unsigned char* hd) {
    const int* re = p.row_cls_end;
    cn_class<RULE, 0, LT>(p, w, msg, llr_s, s_row, 0, re[0], clip, fuse, sat_flag, lt, hd);
    cn_class<RULE, 1, LT>(p, w, msg, llr_s, s_row, re[0], re[1], clip, fuse, sat_flag, lt, hd);
    cn_class<RULE, 2, LT>(p, w, msg, llr_s, s_row, re[1], re[2], clip, fuse, sat_flag, lt, hd);
    cn_class<RULE, 3, LT>(p, w, msg, llr_s, s_row, re[2], re[3], clip, fuse, sat_flag, lt, hd);
    cn_class<RULE, 4, LT>(p, w, msg, llr_s, s_row, re[3], re[4], clip, fuse, sat_flag, lt, hd);
}

// bit 31 set iff |x| < SB_PHI_ZERO (b = bits(x)): fl(|x| - SB_PHI_ZERO) has the sign of the exact difference and is
// +0 when they are equal. One FADD, and a funnel shift moves the bit into a mask.
__device__ __forceinline__ unsigned unsat_bit31(unsigned b) {
    return __float_as_uint(__fadd_rn(fabsf(__uint_as_float(b)), -SB_PHI_ZERO));
}

// CN phase of the voting iterations: the warp's rows (rr = grp, grp + G, ...; the same rows as the class loops of
// cn_all), class-agnostic. Per row an inline read pass builds the lane's masks (bit l: |x_l| < SB_PHI_ZERO in own, sign
// of x_l in S), top edge first, and __reduce_or_sync the union mask U. A row whose U holds no edge but the last (the
// common row once a codeword has converged) is finished here: two phi, one loop-carried copy, then the stores; only the
// 2k + 1 walk of the other rows is the out-of-line cn_vote_row. Both loops take two edges per trip, after one single
// edge when deg - 1 is odd (measured 1.3 % faster at 2 dB than one edge per trip, H100 80GB HBM3, 700 W). Rows of more than 32 edges (none in
// the 5G base graphs) run the plain variant, whose probe then re-raises the already raised flag. A lane outside a row
// (lane_i >= zrow) reads the row's first check instead of its own (a valid slot), drops its bits from the union mask
// and stores nothing.
// Taking two rows per trip, with the phi of two converged rows as one phi pair, measured no faster at 2 dB and slower
// at 0 dB and with early termination (H100 80GB HBM3, 700 W): 12.68-12.70 against 12.65-12.67 ms, 16.72-16.74 against
// 16.55-16.57 ms, 10.69-10.71 against 10.53-10.54 ms.
template <class LT>
__device__ __forceinline__ void cn_vote_pass(const QcParams& p, const WarpCtx& w, float* msg, const float* llr_s,
                                             const int4* s_row, float clip, bool fuse, float phi_max, int* sat_flag,
                                             const LT& lt, unsigned char* hd) {
    const int Z = p.Z, Z4 = 4 * Z;
    const int msgb = (int)smem_u32(msg);
    const unsigned ylast = __float_as_uint(fminf(phi_max, clip));
    for (int rr = w.grp; rr < p.n_rows; rr += w.G) {
        const int4 ri = s_row[rr];
        const bool act = w.lane_i < ri.z;
        float c2v = 0.f;                                  // new message of the row's last edge (the fused update's input)
        if (ri.y > 32) {
            if (act) {
                float* pm = msg + ri.x * Z + w.lane_i;
                cn_phi_qc<LT>(pm, Z, ri.y, clip, sat_flag, lt);
                c2v = pm[(ri.y - 1) * Z];
            }
        } else if (ri.y > 0) {
            const int deg = ri.y;
            const int a0 = msgb + 4 * (ri.x * Z + (act ? w.lane_i : 0));   // address of edge 0
            const int top = a0 + (deg - 1) * Z4;
            const unsigned last = __float_as_uint(lds_f32(top));
            unsigned own = unsat_bit31(last) >> 31, S = last >> 31;
            int a = top - Z4;                             // edges deg - 2 ... 0
            if (!(deg & 1)) {
                const unsigned b = __float_as_uint(lds_f32(a));
                own = __funnelshift_l(unsat_bit31(b), own, 1);
                S = __funnelshift_l(b, S, 1);
                a -= Z4;
            }
            for (; a > a0; a -= 2 * Z4) {
                const unsigned b1 = __float_as_uint(lds_f32(a)), b0 = __float_as_uint(lds_f32(a - Z4));
                own = __funnelshift_l(unsat_bit31(b1), own, 1);
                own = __funnelshift_l(unsat_bit31(b0), own, 1);
                S = __funnelshift_l(b1, S, 1);
                S = __funnelshift_l(b0, S, 1);
            }
            const unsigned U = __reduce_or_sync(0xffffffffu, act ? own : 0u);
            if (!(U & ~(1u << (deg - 1)))) {
                // every edge but the last has phi = +0, so P = phi(|x_last|); the others get phi(P), the last phi_max
                float y = __uint_as_float(last & 0x7fffffffu);
#pragma unroll 1
                for (int k = 0; k < 2; ++k) y = sb_phif_s(y, lt);
                if (act) {
                    const unsigned yb = __float_as_uint(fminf(y, clip));
                    // V = S ^ parity: bit l is the output sign of edge l; v walks it up to bit 31, one edge per shift
                    unsigned v = (S ^ (0u - (__popc(S) & 1u))) << (32 - deg);
                    const unsigned wl = ylast | (v & 0x80000000u);
                    sts_f32(top, __uint_as_float(wl));
                    c2v = __uint_as_float(wl);
                    int a = top - Z4;
                    if (!(deg & 1)) {
                        v <<= 1;
                        sts_f32(a, __uint_as_float(yb | (v & 0x80000000u)));
                        a -= Z4;
                    }
                    for (; a > a0; a -= 2 * Z4) {
                        sts_f32(a, __uint_as_float(yb | ((v << 1) & 0x80000000u)));
                        sts_f32(a - Z4, __uint_as_float(yb | ((v << 2) & 0x80000000u)));
                        v <<= 2;
                    }
                }
            } else if (act) {
                cn_vote_row<LT>(msg + ri.x * Z + w.lane_i, Z, deg, U, S, clip, lt);
                c2v = lds_f32(top);
            }
        }
        if (fuse && ri.w >= 0 && act)
            fused_vn(p, msg + (ri.x + ri.y - 1) * Z + w.lane_i, c2v, ri.w, w.lane_i, llr_s, clip, hd);
    }
}

// Syndrome of the current hard decisions hd[] (one byte per VN): every warp walks its block rows like the CN phase and
// XORs the decisions of the row's variable nodes, VN of base entry (c, s) and check offset i being c * Z + (i + s) mod Z.
// Raises *unsat if any check is violated.
__device__ __forceinline__ void syndrome_pass(const QcParams& p, const WarpCtx& w, const int4* s_row,
                                              const unsigned char* hd, int* unsat) {
    for (int rr = w.grp; rr < p.n_rows; rr += w.G) {
        const int4 ri = s_row[rr];
        if (w.lane_i < ri.z) {
            unsigned par = 0;
            for (int l = 0; l < ri.y; ++l) {
                const int2 e = __ldg(p.row_edge + ri.x + l);
                int j = w.lane_i + e.y;
                j -= (j >= p.Z) ? p.Z : 0;
                par ^= hd[e.x + j];
            }
            if (par) *unsat = 1;
        }
    }
}

template <int CLS, bool EX>
__device__ __forceinline__ void vn_class(const QcParams& p, const WarpCtx& w, const VnLane& vl, const float* llr_s,
                                         const int4* s_col, uint32_t s_ce, int start, int end, float clip,
                                         bool final_pass, long long b, unsigned char* hd) {
    for (int cc = first_of(start, p.col_cls_mod[CLS], w); cc < end; cc += w.G) {
        int4 ci = s_col[cc];
        if (w.lane_i < ci.z) {
            int v = ci.w + w.lane_i;
            float x_tot = vn_cls<CLS, EX>(s_ce + 8 * ci.x, ci.y, vl, llr_s[v], clip);
            if (hd) hd[v] = 0.f >= x_tot ? 1 : 0;                                            // hard decision (:622-624)
            if (final_pass) {
                int o = p.out_pos[v];
                if (o >= 0) {
                    x_tot = clipf(x_tot, clip);                                              // :730
                    p.out[(size_t)b * p.n_out + o] = decoder_out(x_tot, p.hard_out);              // :622-626
                }
            }
        }
    }
}

template <bool EX>
__device__ __forceinline__ void vn_all(const QcParams& p, const WarpCtx& w, const VnLane& vl, const float* llr_s,
                                       const int4* s_col, uint32_t s_ce, float clip, bool final_pass,
                                       bool with_fused, long long b, unsigned char* hd) {
    const int* ce = p.col_cls_end;
    vn_class<0, EX>(p, w, vl, llr_s, s_col, s_ce, 0, ce[0], clip, final_pass, b, hd);
    vn_class<1, EX>(p, w, vl, llr_s, s_col, s_ce, ce[0], ce[1], clip, final_pass, b, hd);
    vn_class<2, EX>(p, w, vl, llr_s, s_col, s_ce, ce[1], ce[2], clip, final_pass, b, hd);
    vn_class<3, EX>(p, w, vl, llr_s, s_col, s_ce, ce[2], ce[3], clip, final_pass, b, hd);
    vn_class<4, EX>(p, w, vl, llr_s, s_col, s_ce, ce[3], ce[4], clip, final_pass, b, hd);
    vn_class<5, EX>(p, w, vl, llr_s, s_col, s_ce, ce[4], ce[5], clip, final_pass, b, hd);
    vn_class<6, EX>(p, w, vl, llr_s, s_col, s_ce, ce[5], ce[6], clip, final_pass, b, hd);
    vn_class<7, EX>(p, w, vl, llr_s, s_col, s_ce, ce[6], ce[7], clip, final_pass, b, hd);
    vn_class<8, EX>(p, w, vl, llr_s, s_col, s_ce, ce[7], ce[8], clip, final_pass, b, hd);
    vn_class<9, EX>(p, w, vl, llr_s, s_col, s_ce, ce[8], ce[9], clip, final_pass, b, hd);
    if (with_fused) vn_class<10, EX>(p, w, vl, llr_s, s_col, s_ce, ce[9], ce[10], clip, final_pass, b, hd);
}

// v2c = llr on every edge (decoding.py:571), once per codeword. One class-agnostic loop over the warp's columns in loop
// form: the unrolled classes are the iterations' code, and a second copy of them for this pass only made the kernel
// larger (it is bound by instruction fetch). The message is the canonical llr + 0 (+0.0 for punctured bits, whose llr
// is -0.0). `staged` (the opening iterations, cn_open_pass): the edges get the pass-1 word phi(|v2c|) | sign(v2c)
// instead, one phi per VN rather than one per edge.
template <class LT>
__device__ __forceinline__ void vn_init(const QcParams& p, const WarpCtx& w, const VnLane& vl, const float* llr_s,
                                        const int4* s_col, uint32_t s_ce, bool staged, const LT& lt) {
    for (int cc = w.grp; cc < p.n_cols; cc += w.G) {
        const int4 ci = s_col[cc];
        if (w.lane_i >= ci.z) continue;
        const float llr = llr_s[ci.w + w.lane_i];
        if (staged) {
            float P = 0.f;                                // unused
            const unsigned st = phi_pass1(__float_as_uint(__fadd_rn(llr, 0.f)), P, lt);
            vn_qc_loop<2>(s_ce + 8 * ci.x, ci.y, vl, __uint_as_float(st), 0.f);
        } else {
            vn_qc_loop<1>(s_ce + 8 * ci.x, ci.y, vl, llr, 0.f);
        }
    }
}

// ---- the opening iterations of boxplus-phi on graphs with punctured columns ----------------------------------------
// Rate recovery gives a punctured VN the channel LLR -0.0, so its first v2c is +0 and phi(+0) = phi_max ~ 16.97. When
// every row holds a punctured edge (the host planner decides, open_tab), iteration 0 is mostly an exact no-op:
//   * CN: for an edge e other than a row's only punctured edge, P - p_e still contains a phi_max, so P - p_e >=
//     SB_PHI_ZERO and its c2v is +-0 exactly. Only the punctured edge of a row with a single punctured edge needs
//     phi(P - p_e); the punctured edges of the other rows get +-0.
//   * VN: a non-punctured VN receives only +-0, so x_tot = (+0 + +-0 + ...) + llr = llr and its new v2c is llr + 0,
//     its first v2c again (the fused degree-1 update as well). Only the punctured columns change.
// So vn_init writes the pass-1 words of every edge, iteration 0 sums them into P without evaluating phi (the same
// values in the same ascending order as pass 1, so P is bit-identical) and writes only the punctured edges, and its VN
// phase (vn_open) updates only the punctured columns. The other edges still hold their pass-1 words in iteration 1,
// which evaluates phi(|x|) only at the punctured edges before its usual pass 2 and fused update. Iteration 0 raises no
// saturation flag: edge 0 or 1 of every row is punctured (host condition), so its first-pair probe sees |x| = 0.
// Iteration 1 probes like the plain variant, reading the first v2c of a non-punctured edge from the channel LLRs.
// One out-of-line routine for both iterations and every degree, like cn_phi_qc (the kernel is instruction-fetch bound).
template <class LT>
__device__ __noinline__ void cn_phi_open(float* pm, int Z, int deg, unsigned punct, bool second, float clip, LT lt) {
    float P = 0.f;
    unsigned u = second ? punct : 0u;                     // iteration 1: the punctured edges hold v2c, stage them
    for (; u & (u - 1); u &= u - 1) {
        float* q0 = pm + (__ffs(u) - 1) * Z;
        u &= u - 1;
        float* q1 = pm + (__ffs(u) - 1) * Z;
        const uint2 w = phi_pass1_pair(ldw(q0), ldw(q1), P, lt, [](float, float) {});
        stw(q0, w.x);
        stw(q1, w.y);
    }
    if (u) {
        float* q0 = pm + (__ffs(u) - 1) * Z;
        stw(q0, phi_pass1(ldw(q0), P, lt));
    }
    P = 0.f;
    unsigned par = 0;
    for (int l = 0; l < deg; ++l) {                       // P in ascending VN order, as pass 1 sums it
        const unsigned w = ldw(pm + l * Z);
        par ^= w;
        P = __fadd_rn(P, __uint_as_float(w & 0x7fffffffu));
    }
    par &= 0x80000000u;
    if (!second && (punct & (punct - 1))) {               // iteration 0, two or more punctured edges: outputs +-0
        for (u = punct; u; u &= u - 1) {
            float* q0 = pm + (__ffs(u) - 1) * Z;
            stw(q0, (ldw(q0) ^ par) & 0x80000000u);
        }
        return;
    }
    // pass 2 on every edge (iteration 1) or on the single punctured edge (iteration 0)
    for (u = second ? 0xffffffffu >> (32 - deg) : punct; u & (u - 1); u &= u - 1) {
        float* q0 = pm + (__ffs(u) - 1) * Z;
        u &= u - 1;
        float* q1 = pm + (__ffs(u) - 1) * Z;
        const uint2 y = phi_pass2_pair(ldw(q0), ldw(q1), P, par, clip, lt);
        stw(q0, y.x);
        stw(q1, y.y);
    }
    if (u) {
        float* q0 = pm + (__ffs(u) - 1) * Z;
        stw(q0, phi_pass2(ldw(q0), P, par, clip, lt));
    }
}

// CN phase of iteration 0 (second = false) or 1 of the opening path: the warp's rows as in cn_vote_pass.
template <class LT>
__device__ __forceinline__ void cn_open_pass(const QcParams& p, const WarpCtx& w, float* msg, const float* llr_s,
                                             const int4* s_row, float clip, bool second, int* sat_flag, const LT& lt) {
    const int Z = p.Z;
    for (int rr = w.grp; rr < p.n_rows; rr += w.G) {
        const int4 ri = s_row[rr];
        if (w.lane_i < ri.z) {
            const unsigned punct = (unsigned)__ldg(p.open_tab + rr);
            float* pm = msg + ri.x * Z + w.lane_i;
            if (second && ri.y >= 2) {                    // the plain variant's probe on |x| of edges 0 and 1
                auto mag = [&](int l) {
                    if ((punct >> l) & 1u) return fabsf(pm[l * Z]);
                    const int2 e = __ldg(p.row_edge + ri.x + l);
                    int j = w.lane_i + e.y;
                    j -= (j >= Z) ? Z : 0;
                    return fabsf(llr_s[e.x + j]);
                };
                const float a0 = mag(0), a1 = mag(1);
                if (__all_sync(__activemask(), a0 >= SB_PHI_HI && a1 >= SB_PHI_HI)) *sat_flag = 1;
            }
            cn_phi_open<LT>(pm, Z, ri.y, punct, second, clip, lt);
            if (second && ri.w >= 0) {
                float* q = pm + (ri.y - 1) * Z;
                fused_vn(p, q, *q, ri.w, w.lane_i, llr_s, clip, nullptr);
            }
        }
    }
}

// VN phase of iteration 0 of the opening path: the punctured columns only, in loop form (once per codeword)
__device__ __forceinline__ void vn_open(const QcParams& p, const WarpCtx& w, const VnLane& vl, const float* llr_s,
                                        const int4* s_col, uint32_t s_ce, float clip) {
    for (int cc = w.grp; cc < p.n_cols; cc += w.G) {
        const int4 ci = s_col[cc];
        if (__ldg(p.open_tab + p.n_rows + cc) && w.lane_i < ci.z)
            vn_qc_loop<0>(s_ce + 8 * ci.x, ci.y, vl, llr_s[ci.w + w.lane_i], clip);
    }
}

// Threads per CTA. 24 warps (80 registers/thread) for every rule: 30 warps at 64 registers were measured for the min-sum
// kernels and lost 7 % (5.32 vs 4.97 ms / 4096 codewords: more barrier and spill time than latency hiding gained).
constexpr int kQcThreads = 768;

// REP: copies of the phi log table (16, 8 or 1). EARLY: the early-termination variant (hard-decision bytes + syndrome
// pass); a separate instantiation so that the default kernel carries none of it (as a run-time flag it cost 2 %).
template <int RULE, int REP, bool EARLY>
__global__ void __launch_bounds__(kQcThreads, 1) ldpc_bp_qc_kernel(const __grid_constant__ QcParams p) {
    const int T = blockDim.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, W = T >> 5;
    const int Z = p.Z, N = p.N, Zb = (Z + 31) >> 5;
    // carve-up by byte offsets from the __shared__ base (keeps the shared address space visible to the compiler): the
    // phi log table at offset 0 (sb_math2.cuh), then the messages
    unsigned char* const smem_raw = sb_smem + (RULE == SB_CN_BOXPLUS_PHI ? LogTab<REP>::bytes : 0);
    const int off_llr = p.E_alloc * 4;
    const int off_col = (off_llr + N * 4 + 15) & ~15;
    const int off_row = off_col + p.n_cols * 16;
    const int off_ce = off_row + p.n_rows * 16;
    const int off_bar = (off_ce + p.nnz * 8 + 15) & ~15;
    float* msg = reinterpret_cast<float*>(smem_raw);
    float* llr_s = reinterpret_cast<float*>(smem_raw + off_llr);
    int4* s_col = reinterpret_cast<int4*>(smem_raw + off_col);
    int4* s_row = reinterpret_cast<int4*>(smem_raw + off_row);
    int2* s_ce_p = reinterpret_cast<int2*>(smem_raw + off_ce);
    uint64_t* bar = reinterpret_cast<uint64_t*>(smem_raw + off_bar);
    int* sat_flag = reinterpret_cast<int*>(smem_raw + off_bar + 8);
    int* unsat = reinterpret_cast<int*>(smem_raw + off_bar + 12);
    unsigned char* hd = EARLY ? smem_raw + off_bar + 16 : nullptr;   // early termination: one hard-decision byte per VN
    const uint32_t msgb = smem_u32(smem_raw);             // 32-bit shared-window addresses for the hot loops
    const uint32_t s_ce = msgb + off_ce;
    // a warp keeps one 32-lane slice `ib` of every block row/column it visits; G warp groups share the rows
    WarpCtx w;
    w.G = W / Zb;
    w.grp = warp / Zb;
    w.lane_i = (warp - w.grp * Zb) * 32 + lane;
    VnLane vl{4u * w.lane_i, 4u * (w.lane_i + Z), (4u * w.lane_i) << 16 | 0xffffu};
    asm("" : "+r"(vl.j4), "+r"(vl.j4w), "+r"(vl.jk));     // three live registers: not rebuilt from lane_i at every edge

    for (int i = tid; i < p.n_cols; i += T) s_col[i] = p.col_info[i];
    for (int i = tid; i < p.n_rows; i += T) s_row[i] = p.row_info[i];
    for (int i = tid; i < p.nnz; i += T) {                // the column table in address form (vn_addr)
        const int2 e = p.col_edge[i];
        const uint32_t s4 = (uint32_t)e.y & 0xffffu;
        s_ce_p[i] = make_int2((int)(msgb + (uint32_t)e.x - s4), (int)(s4 << 16 | (uint32_t)e.y >> 16));
    }
    const LogTab<REP> lt(lane);
    if (RULE == SB_CN_BOXPLUS_PHI) LogTab<REP>::fill(tid, T);
    if (p.use_tma && tid == 0) mbar_init(bar);
    __syncthreads();

    const float clip = p.llr_max;
    const float phi_max = sb_phif(0.f);                   // phi at its lower clipping bound (global-memory table)
    uint32_t tma_phase = 0;
    // opening iterations 0 and 1 (cn_open_pass); neither is the final one. The early-termination variant keeps the
    // plain path: its hard decisions come from the VN phase of every column.
    const bool open = RULE == SB_CN_BOXPLUS_PHI && !EARLY && p.open && p.num_iter >= 3;

    for (long long b = blockIdx.x; b < p.B; b += gridDim.x) {
        // ---- channel LLRs in natural VN order, staged in the message array ---------------------------------------
        load_channel_llr(llr_s, p.llr + (size_t)b * p.n_in, p.in_idx, N, p.n_in, clip, p.use_tma, msg, bar, tma_phase,
                         tid, T);
        __syncthreads();
        if (tid == 0) *sat_flag = 0;
        // ---- v2c = llr of the edge's VN (decoding.py:571) ---------------------------------------------------------
        vn_init(p, w, vl, llr_s, s_col, s_ce, open, lt);
        __syncthreads();
        if (p.num_iter == 0) {                           // x_hat = llr_ch (decoding.py:603-608)
            for (int v = tid; v < N; v += T) {
                int o = p.out_pos[v];
                if (o >= 0) p.out[(size_t)b * p.n_out + o] = decoder_out(llr_s[v], p.hard_out);
            }
        }
        // Early termination (opt-in; the reference always runs num_iter iterations, decoding.py:105-107). The VN phase
        // keeps the hard decision of every VN in hd[]; before iteration `it` (it >= 1) a syndrome pass checks H * hd = 0.
        // If it holds, iteration `it` becomes the final one (its CN phase does not fuse the degree-1 updates, its VN phase
        // writes the outputs): the outputs equal a fixed-iteration decode with num_iter = it + 1 bit for bit.
        int limit = p.num_iter;
        for (int it = 0; it < limit; ++it) {
            if (EARLY && it > 0 && it < limit - 1) {
                if (tid == 0) *unsat = 0;
                __syncthreads();
                syndrome_pass(p, w, s_row, hd, unsat);
                __syncthreads();
                if (*unsat == 0) limit = it + 1;               // CTA-uniform: read between barriers
            }
            const bool final_pass = it == limit - 1;
            const bool sc = *sat_flag != 0;                // CTA-uniform: read after the barrier that ended the last phase
            // ---- CN phase (degree-1 VN updates fused in, except in the final iteration) -------------------------
            if (final_pass && tid == 0 && p.use_tma && b + gridDim.x < p.B)   // pull the next codeword's logits into L2 early
                asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p.llr + (size_t)(b + gridDim.x) * p.n_in),
                             "r"((uint32_t)p.n_in * 4u) : "memory");
            if constexpr (RULE == SB_CN_BOXPLUS_PHI) {
                if (open && it < 2) cn_open_pass(p, w, msg, llr_s, s_row, clip, it == 1, sat_flag, lt);
                else if (sc) cn_vote_pass(p, w, msg, llr_s, s_row, clip, !final_pass, phi_max, sat_flag, lt, hd);
                else cn_all<RULE>(p, w, msg, llr_s, s_row, clip, !final_pass, sat_flag, lt, hd);
            } else {
                cn_all<RULE>(p, w, msg, llr_s, s_row, clip, !final_pass, sat_flag, lt, hd);
            }
            __syncthreads();
            // ---- VN phase ---------------------------------------------------------------------------------------
            if (open && it == 0) vn_open(p, w, vl, llr_s, s_col, s_ce, clip);
            else vn_all<true>(p, w, vl, llr_s, s_col, s_ce, clip, final_pass, final_pass, b, hd);
            __syncthreads();
        }
        if (EARLY && p.iters_out && tid == 0) p.iters_out[b] = limit;
        if (p.state_out) {
            store_state(p.state_out + (size_t)b * p.E, msg, p.slot_of_edge, p.E, tid, T);
            __syncthreads();
        }
    }
}

size_t qc_smem_bytes(const sb_ldpc_graph* g, int tab_rep, int early = 0) {
    return (early ? (size_t)g->N + 16 : 0) + ((size_t)g->qc_nnz * g->qc_Z + g->N) * 4 + 16 + (size_t)g->qc_cols * 16 + (size_t)g->qc_rows * 16 +
           (size_t)g->qc_nnz * 8 + 16 + 16 + (size_t)tab_rep * SB_LOGTAB_N * 8;
}

template <int RULE, bool EARLY>
int launch_qc(const QcParams& p, int num_sms, int threads, size_t smem, cudaStream_t stream) {
    auto kern = ldpc_bp_qc_kernel<RULE, 16, EARLY>;
    if constexpr (RULE == SB_CN_BOXPLUS_PHI) {
        if (p.tab_rep == 8) kern = ldpc_bp_qc_kernel<RULE, 8, EARLY>;
        if (p.tab_rep == 1) kern = ldpc_bp_qc_kernel<RULE, 1, EARLY>;
    }
    return sb_launch_decoder(kern, p, num_sms, threads, smem, LLONG_MAX, stream, "sb_ldpc_decode(qc)");
}

}  // namespace

// Attach the quasi-cyclic description of the graph: base entries (row, col, shift) of the lifted matrix with lifting
// size Z; entries outside ceil(C/Z) x ceil(N/Z) are ignored (pruned away). The description is verified against the
// handle's edge list; on mismatch the handle is left unchanged and SB_EINVAL is returned.
extern "C" int sb_ldpc_graph_set_qc(sb_ldpc_graph* g, int32_t Z, int32_t n_entries, const int32_t* base_row,
                                    const int32_t* base_col, const int32_t* shift) {
    SB_CHECK_ARG(g && Z > 0 && Z <= 16383 && n_entries > 0 && base_row && base_col && shift, "sb_ldpc_graph_set_qc: bad arguments");
    SB_CHECK_ARG((int)g->h_cn.size() == g->E, "sb_ldpc_graph_set_qc: handle holds no edge list");
    SB_CHECK_ARG(!g->ref_order, "sb_ldpc_graph_set_qc: the QC kernel sums in ascending neighbour order; graphs created with "
                                "sb_ldpc_graph_create_ordered stay on the generic kernel");
    const int C = g->C, N = g->N, E = g->E;
    const int n_rows = (C + Z - 1) / Z, n_cols = (N + Z - 1) / Z;
    auto zrow = [&](int r) { return std::min(Z, C - r * Z); };
    auto zcol = [&](int c) { return std::min(Z, N - c * Z); };
    struct Ent { int r, c, s; };
    std::vector<Ent> ents;
    for (int k = 0; k < n_entries; ++k) {
        if (base_row[k] < 0 || base_col[k] < 0 || shift[k] < 0) { sb_set_error("sb_ldpc_graph_set_qc: negative entry"); return SB_EINVAL; }
        if (base_row[k] >= n_rows || base_col[k] >= n_cols) continue;
        ents.push_back({base_row[k], base_col[k], shift[k] % Z});
    }
    // verify against the edge list
    std::vector<long long> keys(E);
    for (int e = 0; e < E; ++e) keys[e] = ((long long)g->h_cn[e] << 32) | (unsigned)g->h_vn[e];
    std::sort(keys.begin(), keys.end());
    long long total = 0;
    for (const Ent& en : ents)
        for (int i = 0; i < zrow(en.r); ++i) {
            int j = (i + en.s) % Z;
            long long key = ((long long)(en.r * Z + i) << 32) | (unsigned)(en.c * Z + j);
            if (j >= zcol(en.c) || !std::binary_search(keys.begin(), keys.end(), key)) {
                sb_set_error("sb_ldpc_graph_set_qc: base entry (%d,%d,%d) does not match the graph", en.r, en.c, en.s);
                return SB_EINVAL;
            }
            ++total;
        }
    if (total != E) { sb_set_error("sb_ldpc_graph_set_qc: %lld lifted edges != %d graph edges", total, E); return SB_EINVAL; }
    // classes (see the kernel): rows by degree bucket, heaviest first; columns by bucket / pruning-cut rows / fused
    std::vector<int> rdeg(n_rows, 0), cdeg(n_cols, 0);
    for (const Ent& en : ents) { ++rdeg[en.r]; ++cdeg[en.c]; }
    std::vector<std::vector<Ent>> by_row(n_rows), by_col(n_cols);
    for (const Ent& en : ents) { by_row[en.r].push_back(en); by_col[en.c].push_back(en); }
    for (auto& v : by_row) std::sort(v.begin(), v.end(), [](const Ent& a, const Ent& b) { return a.c < b.c; });
    for (auto& v : by_col) std::sort(v.begin(), v.end(), [](const Ent& a, const Ent& b) { return a.r < b.r; });
    // a degree-1 column whose single entry is the LAST entry of its row is updated inside the CN phase
    std::vector<int> fused_col_of_row(n_rows, -1);
    std::vector<char> col_fused(n_cols, 0);
    for (int r = 0; r < n_rows; ++r) {
        if (by_row[r].empty()) continue;
        const Ent& last = by_row[r].back();
        if (cdeg[last.c] == 1 && rdeg[r] >= 2 && last.c < 65536 && zcol(last.c) == zrow(r)) {
            fused_col_of_row[r] = last.c;
            col_fused[last.c] = 1;
        }
    }
    auto row_class = [&](int r) { return degree_class(kRowMax, 0, kRowClasses, rdeg[r]); };
    auto col_class = [&](int c) {
        if (col_fused[c]) return kColFused;
        bool check = false;
        for (const Ent& en : by_col[c]) check = check || zrow(en.r) < Z;
        return check ? degree_class(kColMax, kColCut, kColFused, cdeg[c]) : degree_class(kColMax, 0, kColCut, cdeg[c]);
    };
    std::vector<int> rorder(n_rows), corder(n_cols);
    std::iota(rorder.begin(), rorder.end(), 0);
    std::iota(corder.begin(), corder.end(), 0);
    std::stable_sort(rorder.begin(), rorder.end(), [&](int a, int b) {
        return row_class(a) != row_class(b) ? row_class(a) < row_class(b) : rdeg[a] > rdeg[b]; });
    std::stable_sort(corder.begin(), corder.end(), [&](int a, int b) {
        return col_class(a) != col_class(b) ? col_class(a) < col_class(b) : cdeg[a] > cdeg[b]; });
    // Inside a class the order is free. Rows / columns are dealt cyclically to the G warp groups of a launch over ALL
    // classes (position i -> group i mod G), so the order decides the load balance: walk the positions in rounds of G
    // consecutive ones (a round gives every group at most one item) and hand the round's heaviest item to the group with
    // the smallest load so far. Degree order alone left the benchmark graph's four groups with 56/53/52/49 edges per lane
    // in the CN phase and 56/53/41/40 in the VN phase; this gives 54/54/53/49 and 48/48/47/47. G is fixed by Z and the CTA
    // size (kQcThreads / 32 / ceil(Z / 32)), the same for every rule.
    {
        const int Zb_ = (Z + 31) / 32;
        const int G = std::max(1, (kQcThreads / 32) / Zb_);
        auto balance = [&](std::vector<int>& order, const std::vector<int>& deg, auto cls_of) {
            std::vector<long long> load(G, 0);
            size_t pos = 0;
            while (pos < order.size()) {
                size_t end = pos;
                const int c = cls_of(order[pos]);
                while (end < order.size() && cls_of(order[end]) == c) ++end;      // one class: positions [pos, end)
                std::vector<int> items(order.begin() + pos, order.begin() + end);
                std::stable_sort(items.begin(), items.end(), [&](int a, int b) { return deg[a] > deg[b]; });
                size_t next = 0;
                for (size_t r0 = pos; r0 < end; r0 += G) {
                    const size_t r1 = std::min(end, r0 + (size_t)G);
                    std::vector<size_t> slots;
                    for (size_t q = r0; q < r1; ++q) slots.push_back(q);
                    std::stable_sort(slots.begin(), slots.end(), [&](size_t a, size_t b) { return load[a % G] < load[b % G]; });
                    for (size_t q : slots) {
                        order[q] = items[next++];
                        load[q % G] += deg[order[q]];
                    }
                }
                pos = end;
            }
        };
        balance(rorder, rdeg, row_class);
        balance(corder, cdeg, col_class);
    }
    std::vector<int> row_cls_end(kRowClasses, 0), col_cls_end(kColClasses, 0);
    for (int r = 0; r < n_rows; ++r) for (int k = row_class(r); k < kRowClasses; ++k) ++row_cls_end[k];
    for (int c = 0; c < n_cols; ++c) for (int k = col_class(c); k < kColClasses; ++k) ++col_cls_end[k];
    // base-entry numbering: rows in processing order, ascending column inside a row
    std::vector<int> be_of((size_t)n_rows * n_cols, -1);
    std::vector<int> row_info(4 * n_rows), row_edge;
    int be = 0;
    for (int rr = 0; rr < n_rows; ++rr) {
        int r = rorder[rr];
        row_info[4 * rr] = be;
        row_info[4 * rr + 1] = rdeg[r];
        row_info[4 * rr + 2] = zrow(r);
        row_info[4 * rr + 3] = fused_col_of_row[r] >= 0 ? (fused_col_of_row[r] | (by_row[r].back().s << 16)) : -1;
        for (const Ent& en : by_row[r]) {
            if (be_of[(size_t)en.r * n_cols + en.c] != -1) { sb_set_error("sb_ldpc_graph_set_qc: duplicate base entry"); return SB_EINVAL; }
            be_of[(size_t)en.r * n_cols + en.c] = be++;
            row_edge.push_back(en.c * Z);
            row_edge.push_back(en.s);
        }
    }
    const int nnz = be;
    std::vector<int> col_info(4 * n_cols), col_edge(2 * (size_t)nnz);
    int ce = 0;
    for (int cc = 0; cc < n_cols; ++cc) {
        int c = corder[cc];
        col_info[4 * cc] = ce;
        for (const Ent& en : by_col[c]) {
            col_edge[2 * ce] = be_of[(size_t)en.r * n_cols + en.c] * Z * 4;
            col_edge[2 * ce + 1] = (en.s * 4) | ((zrow(en.r) * 4) << 16);
            ++ce;
        }
        col_info[4 * cc + 1] = cdeg[c];
        col_info[4 * cc + 2] = zcol(c);
        col_info[4 * cc + 3] = c * Z;
    }
    // natural-order I/O maps and the reference-edge -> slot map
    std::vector<int> in_nat(N), out_nat(N), slot(E);
    for (int r = 0; r < N; ++r) { in_nat[g->vn_order[r]] = g->in_idx[r]; out_nat[g->vn_order[r]] = g->out_pos[r]; }
    for (int e = 0; e < E; ++e) {
        int r = g->h_cn[e] / Z, i = g->h_cn[e] % Z, c = g->h_vn[e] / Z;
        slot[e] = be_of[(size_t)r * n_cols + c] * Z + i;
    }
    // Opening iterations of boxplus-phi (cn_open_pass): the punctured columns are those whose every VN gets no channel
    // input (in_idx -1, LLR 0). The path is on when every row has a punctured edge at position 0 or 1 (which keeps the
    // first-pair probe of iteration 0 silent) and at most 32 edges (one mask word), and no punctured column is fused.
    std::vector<int> open_tab(n_rows + n_cols, 0);
    bool open = true;
    std::vector<char> punct(n_cols, 1);
    for (int c = 0; c < n_cols; ++c)
        for (int v = c * Z; v < c * Z + zcol(c); ++v) punct[c] = punct[c] && in_nat[v] == -1;
    for (int rr = 0; rr < n_rows; ++rr) {
        const int r = rorder[rr];
        unsigned m = 0;
        for (size_t l = 0; l < by_row[r].size() && l < 32; ++l) m |= (unsigned)punct[by_row[r][l].c] << l;
        open = open && rdeg[r] <= 32 && (m & 3u);
        open_tab[rr] = (int)m;
    }
    for (int cc = 0; cc < n_cols; ++cc) {
        open_tab[n_rows + cc] = punct[corder[cc]];
        open = open && !(punct[corder[cc]] && col_fused[corder[cc]]);
    }
    g->qc = true;
    g->qc_open = open;
    g->qc_open_tab.swap(open_tab); g->qc_Z = Z; g->qc_rows = n_rows; g->qc_cols = n_cols; g->qc_nnz = nnz;
    g->qc_max_row_deg = *std::max_element(rdeg.begin(), rdeg.end());
    g->qc_max_col_deg = *std::max_element(cdeg.begin(), cdeg.end());
    g->qc_row_info.swap(row_info); g->qc_col_info.swap(col_info); g->qc_col_edge.swap(col_edge);
    g->qc_row_cls_end = row_cls_end; g->qc_col_cls_end = col_cls_end;
    g->qc_in_idx.swap(in_nat); g->qc_out_pos.swap(out_nat); g->qc_slot_of_edge.swap(slot); g->qc_row_edge.swap(row_edge);
    g->qc_tables.set(g->qc_row_info, g->qc_col_info, g->qc_col_edge, g->qc_in_idx, g->qc_out_pos, g->qc_slot_of_edge,
                     g->qc_row_edge, g->qc_open_tab);
    return SB_OK;
}

// Test hook: evaluates phi on the device with the scalar (sb_math.h) and the packed (sb_math2.cuh) implementation.
namespace {
__global__ void debug_phi_kernel(const float* x, float* o1, float* o2, long long n) {
    LogTab<16>::fill(threadIdx.x, blockDim.x);            // the 16-copy layout of the decoder
    __syncthreads();
    const LogTab<16> lt(threadIdx.x & 31);
    long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (2 * i + 1 < n) {
        float2 r = sb_phif2(make_float2(x[2 * i], x[2 * i + 1]), lt);
        o2[2 * i] = r.x; o2[2 * i + 1] = r.y;
        o1[2 * i] = sb_phif(x[2 * i]); o1[2 * i + 1] = sb_phif(x[2 * i + 1]);
    }
}
}  // namespace
extern "C" int sb_debug_phi(const float* d_x, float* d_scalar, float* d_packed, int64_t n, void* stream) {
    if (n == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_x && d_scalar && d_packed && n >= 0 && n % 2 == 0, "sb_debug_phi: bad arguments");
    debug_phi_kernel<<<(unsigned)((n / 2 + 255) / 256), 256, LogTab<16>::bytes, (cudaStream_t)stream>>>(d_x, d_scalar,
                                                                                                         d_packed, n);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_ldpc_graph_is_qc(const sb_ldpc_graph* g) { return g && g->qc ? 1 : 0; }
extern "C" int sb_ldpc_graph_qc_opening(const sb_ldpc_graph* g) { return g && g->qc && g->qc_open ? 1 : 0; }

int sb_qc_try_decode(const sb_ldpc_graph* g, const DeviceTables::Copy& dev, const float* d_llr, int64_t batch,
                     int32_t num_iter, int32_t cn_rule, int32_t vn_rule, float offset, float llr_max, int32_t hard_out,
                     const float* d_state_in, float* d_state_out, float* d_out, cudaStream_t stream, bool* handled,
                     int32_t early, int32_t* d_iters) {
    *handled = false;
    if (!g->qc || !g->flooding || vn_rule != SB_VN_SUM || d_state_in || cn_rule > SB_CN_OFFSET_MINSUM) return SB_OK;
    // boxplus-phi keeps the log table of phi in shared memory: one copy per bank pair if it fits, else 8 copies or one
    int tab_rep = cn_rule == SB_CN_BOXPLUS_PHI ? 16 : 0;
    if (tab_rep && qc_smem_bytes(g, tab_rep, early) > (size_t)dev.smem_optin) tab_rep = 8;
    if (tab_rep && qc_smem_bytes(g, tab_rep, early) > (size_t)dev.smem_optin) tab_rep = 1;
    const size_t smem = qc_smem_bytes(g, tab_rep, early);
    if (smem > (size_t)dev.smem_optin) return SB_OK;
    if ((cn_rule == SB_CN_MINSUM || cn_rule == SB_CN_OFFSET_MINSUM) &&
        !(llr_max < 100000.f && (float)(g->qc_max_row_deg - 1) * llr_max < 99000.f))
        return SB_OK;                                      // the generic kernel has the literal 1e5-sentinel path
    const DeviceTables::Copy* d = nullptr;
    int rc = g->qc_tables.get(&d);
    if (rc) return rc;
    QcParams p{};
    p.Z = g->qc_Z; p.n_rows = g->qc_rows; p.n_cols = g->qc_cols; p.nnz = g->qc_nnz; p.N = g->N; p.E = g->E;
    p.E_alloc = g->qc_nnz * g->qc_Z; p.n_in = g->n_in; p.n_out = g->n_out;
    for (int k = 0; k < kRowClasses; ++k) p.row_cls_end[k] = g->qc_row_cls_end[k];
    for (int k = 0; k < kColClasses; ++k) p.col_cls_end[k] = g->qc_col_cls_end[k];
    p.row_info = d->at<int4>(0); p.col_info = d->at<int4>(1);
    p.col_edge = d->at<int2>(2); p.in_idx = d->at<int>(3); p.out_pos = d->at<int>(4);
    p.slot_of_edge = d->at<int>(5);
    p.llr = d_llr; p.out = d_out; p.state_out = d_state_out; p.B = batch; p.num_iter = num_iter; p.hard_out = hard_out;
    p.offset = offset; p.llr_max = llr_max; p.tab_rep = tab_rep;
    p.early = early; p.iters_out = d_iters; p.row_edge = d->at<int2>(6);
    // the opening path needs c2v = fminf(+0, clip) = +0, i.e. a clipping bound >= 0
    p.open = cn_rule == SB_CN_BOXPLUS_PHI && g->qc_open && llr_max >= 0.f;
    p.open_tab = d->at<int>(7);
    p.use_tma = (g->n_in % 4 == 0) && (g->n_in <= p.E_alloc) && ((reinterpret_cast<uintptr_t>(d_llr) & 15) == 0);
    const int Zb = (g->qc_Z + 31) / 32;                    // 32-lane slices per block row (<= 12 for Z <= 384)
    const int max_warps = kQcThreads / 32;
    int groups = std::max(1, std::min(max_warps / Zb, std::max(g->qc_rows, g->qc_cols)));
    const int threads = groups * Zb * 32;                  // every warp owns one slice index for the whole launch
    for (int k = 0; k < kRowClasses; ++k) p.row_cls_mod[k] = (k ? g->qc_row_cls_end[k - 1] : 0) % groups;
    for (int k = 0; k < kColClasses; ++k) p.col_cls_mod[k] = (k ? g->qc_col_cls_end[k - 1] : 0) % groups;
    rc = sb_dispatch<SB_CN_BOXPLUS_PHI, SB_CN_OFFSET_MINSUM>(cn_rule, [&](auto R) {
        return p.early ? launch_qc<R, true>(p, dev.num_sms, threads, smem, stream)
                       : launch_qc<R, false>(p, dev.num_sms, threads, smem, stream);
    });
    *handled = (rc == SB_OK);
    return rc;
}
