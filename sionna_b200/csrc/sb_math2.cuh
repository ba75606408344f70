// sb_math2.cuh -- two-at-a-time versions of sb_expf / sb_logf / sb_phif for sm_90a. The two independent element
// chains are interleaved so that each instruction has a second, independent one to issue beside it (two-way ILP).
// sm_90 has no packed fp32x2 arithmetic, so ffma2 / fadd2 / fmul2 below are one IEEE-754 RN FFMA / FADD / FMUL per
// element. Every element goes through exactly the operation sequence of the scalar functions in sb_math.h, so results
// are bit-identical to them (and to the CPU oracle).
#pragma once
#include "sb_math.h"

// Bit casts of the halves of a pair go through an explicit PTX mov, which pins each half to its own register
// (tests/test_ldpc_decoder_gpu.py::test_device_phi_scalar_and_packed_equal_oracle checks both paths bit for bit).
__device__ __forceinline__ int f2i_mov(float x) { int r; asm("mov.b32 %0, %1;" : "=r"(r) : "f"(x)); return r; }
__device__ __forceinline__ float i2f_mov(int x) { float r; asm("mov.b32 %0, %1;" : "=f"(r) : "r"(x)); return r; }
__device__ __forceinline__ float2 f2(float a, float b) { return make_float2(a, b); }
__device__ __forceinline__ float2 f2s(float a) { return make_float2(a, a); }
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
    return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y));
}
__device__ __forceinline__ float2 fadd2(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 fmul2(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }

// e^x for x in [-87.3, 88.7] (callers guarantee the range: no special cases)
__device__ __forceinline__ float2 sb_expf2_inrange(float2 x) {
    float2 t = ffma2(x, f2s(1.44269504088896341f), f2s(12582912.0f));
    float2 nf = fadd2(t, f2s(-12582912.0f));
    float2 r = ffma2(nf, f2s(-0.693145751953125f), x);
    r = ffma2(nf, f2s(-1.42860677e-06f), r);
    float2 g = ffma2(f2s(0x1.a124e4p-13f), r, f2s(0x1.6d4316p-10f));
    g = ffma2(g, r, f2s(0x1.1110e0p-7f));
    g = ffma2(g, r, f2s(0x1.5554eap-5f));
    g = ffma2(g, r, f2s(0x1.555556p-3f));
    g = ffma2(g, r, f2s(0.5f));
    float2 r2 = fmul2(r, r);
    float2 s = ffma2(r2, g, r);
    float2 p = fadd2(f2s(1.0f), s);
    // bits(p) + (n << 23) with n = bits(t) - 0x4B400000: 0x4B400000 << 23 vanishes mod 2^32, so one LEA per element
    return f2(i2f_mov((int)((unsigned)f2i_mov(p.x) + ((unsigned)f2i_mov(t.x) << 23))),
              i2f_mov((int)((unsigned)f2i_mov(p.y) + ((unsigned)f2i_mov(t.y) << 23))));
}

// e^x for x in [-87.3, 88.7], one element: sb_expf's operation sequence without its range tests
__device__ __forceinline__ float sb_expf_inrange(float x) {
    float t = __fmaf_rn(x, 1.44269504088896341f, 12582912.0f);
    float nf = __fadd_rn(t, -12582912.0f);
    float r = __fmaf_rn(nf, -0.693145751953125f, x);
    r = __fmaf_rn(nf, -1.42860677e-06f, r);
    float g = __fmaf_rn(0x1.a124e4p-13f, r, 0x1.6d4316p-10f);
    g = __fmaf_rn(g, r, 0x1.1110e0p-7f);
    g = __fmaf_rn(g, r, 0x1.5554eap-5f);
    g = __fmaf_rn(g, r, 0x1.555556p-3f);
    g = __fmaf_rn(g, r, 0.5f);
    float s = __fmaf_rn(__fmul_rn(r, r), g, r);
    float p = __fadd_rn(1.0f, s);
    return i2f_mov((int)((unsigned)f2i_mov(p) + ((unsigned)f2i_mov(t) << 23)));
}

// log(y) for positive normal y
__device__ __forceinline__ float2 sb_logf2(float2 y) {
    int ix0 = f2i_mov(y.x), ix1 = f2i_mov(y.y);
    int e0 = (ix0 - 0x3f3504f3) >> 23, e1 = (ix1 - 0x3f3504f3) >> 23;
    float2 m = f2(i2f_mov(ix0 - (e0 << 23)), i2f_mov(ix1 - (e1 << 23)));
    float2 ef = f2((float)e0, (float)e1);
    float2 r = fadd2(m, f2s(-1.0f));
    float2 p = ffma2(f2s(0x1.1d8ea6p-4f), r, f2s(-0x1.d635bcp-4f));
    p = ffma2(p, r, f2s(0x1.dea282p-4f));
    p = ffma2(p, r, f2s(-0x1.fcf4c6p-4f));
    p = ffma2(p, r, f2s(0x1.23d21ap-3f));
    p = ffma2(p, r, f2s(-0x1.555b4ap-3f));
    p = ffma2(p, r, f2s(0x1.999d5ap-3f));
    p = ffma2(p, r, f2s(-0x1.fffffcp-3f));
    p = ffma2(p, r, f2s(0x1.555554p-2f));
    float2 r2 = fmul2(r, r);
    float2 r3 = fmul2(r2, r);
    float2 nh = fmul2(f2s(-0.5f), r2);                  // == -(0.5 * r2) exactly
    float2 tl = ffma2(r3, p, nh);
    float2 lo = ffma2(ef, f2s(1.42860677e-06f), tl);
    float2 t2 = fadd2(r, lo);
    return ffma2(ef, f2s(0.693145751953125f), t2);
}

// Dynamic shared memory of the kernels that use the table below; the table sits at its offset 0.
extern __shared__ __align__(16) unsigned char sb_smem[];

// Shared-memory copy of the sb_logf_tab table (sb_math.h) at offset 0 of the dynamic shared memory: entry i is the
// pair {inv_c, log c}, read with one 64-bit LDS. REP copies are interleaved per entry (entry i, copy c at byte
// (i * REP + c) * 8) and lane l reads copy l % REP, so the lookup offset is ((bits(y) >> rs) & mask) | lane_off. A 64-bit
// warp access is served as two half-warps, so 16 copies (one per bank pair, 8 KB: rs 10, mask 0x1f80, lane_off
// 8 * (lane % 16)) are conflict-free. The host falls back to 8 copies or a single one when the table does not fit next
// to the messages.
template <int REP>                                        // REP = 16, 8 or 1 copies: compile-time shift and mask
struct LogTab {
    uint32_t lane_off;
    static constexpr int bytes = SB_LOGTAB_N * REP * 8;
    static constexpr int log_stride = REP == 16 ? 7 : (REP == 8 ? 6 : 3);   // log2(REP * 8 bytes)
    static constexpr int rs = SB_LOGTAB_SHIFT - log_stride;
    static constexpr int mask = (SB_LOGTAB_N - 1) << log_stride;
    // every thread of the CTA stores a share of the table; a barrier must follow before the first lookup
    __device__ static void fill(int tid, int T) {
        float2* tab = reinterpret_cast<float2*>(sb_smem);
        for (int i = tid; i < SB_LOGTAB_N * REP; i += T)
            tab[i] = make_float2(sb_logtab_dev[2 * (i / REP)], sb_logtab_dev[2 * (i / REP) + 1]);
    }
    __device__ explicit LogTab(int lane) : lane_off(8 * (lane & (REP - 1))) {}
};

// (a & MASK) | c in one LOP3 (c in a register; nvcc otherwise emits two LOP3 when both constants are immediates)
template <int MASK>
__device__ __forceinline__ int and_or(int a, int c) {
    int d;
    asm("lop3.b32 %0, %1, %2, %3, 0xEA;" : "=r"(d) : "r"(a), "n"(MASK), "r"(c));
    return d;
}

// {inv_c, log c} of bits(y) = ix from this lane's copy of the table. The base address of the dynamic shared memory is
// CTA-uniform, so it folds into the LDS address operand.
template <class LT>
__device__ __forceinline__ float2 logtab_entry(int ix, const LT& lt) {
    float2 v;
    asm("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y)      // read-only after the prologue barrier
        : "r"((uint32_t)__cvta_generic_to_shared(sb_smem) + and_or<LT::mask>(ix >> LT::rs, lt.lane_off)));
    return v;
}

// E - 127 of bits(y) = ix > 0 as 12582912 + E before the subtraction: float(0x4B400000 + E) is exact, and
// (ix >> 23) + 0x4B400000 is one LEA.HI
__device__ __forceinline__ float logtab_expf(int ix) { return i2f_mov((int)(((unsigned)ix >> 23) + 0x4B400000u)); }

// sb_logf_tab, two at a time (same operation sequence per element)
template <class LT>
__device__ __forceinline__ float2 sb_logf2_tab(float2 y, const LT& lt) {
    int ix0 = f2i_mov(y.x), ix1 = f2i_mov(y.y);
    float2 c0 = logtab_entry(ix0, lt), c1 = logtab_entry(ix1, lt);
    float2 inv_c = f2(c0.x, c1.x);
    float2 logc = f2(c0.y, c1.y);
    float2 m = f2(i2f_mov(and_or<0x007fffff>(ix0, 0x3f800000)), i2f_mov(and_or<0x007fffff>(ix1, 0x3f800000)));
    float2 F = f2(logtab_expf(ix0), logtab_expf(ix1));
    float2 ef = fadd2(F, f2s(-12583039.0f));
    float2 r = ffma2(m, inv_c, f2s(-1.0f));
    float2 q = ffma2(r, f2s(-0.25f), f2s(0x1.555556p-2f));
    q = ffma2(q, r, f2s(-0.5f));
    float2 r2 = fmul2(r, r);
    float2 s = ffma2(r2, q, r);
    float2 lo = ffma2(ef, f2s(1.42860677e-06f), s);
    float2 t2 = fadd2(logc, lo);
    return ffma2(ef, f2s(0.693145751953125f), t2);
}

template <class LT>
__device__ __forceinline__ float sb_logf_tab_s(float y, const LT& lt) {
    int ix = __float_as_int(y);
    float2 c = logtab_entry(ix, lt);
    return sb_logf_tab_core(ix, c.x, c.y);
}

// phi(x) = log(e^x + 1) - log(e^x - 1) with the reference's fp32 clipping (see sb_phif)
template <class LT>
__device__ __forceinline__ float2 sb_phif2(float2 x, const LT& lt) {
    x.x = fminf(fmaxf(x.x, 8.5e-8f), 16.635532f);
    x.y = fminf(fmaxf(x.y, 8.5e-8f), 16.635532f);
    float2 t = sb_expf2_inrange(x);
    float2 la = sb_logf2_tab(fadd2(t, f2s(1.0f)), lt);
    float2 lb = sb_logf2_tab(fadd2(t, f2s(-1.0f)), lt);
    return ffma2(lb, f2s(-1.0f), la);                   // la - lb, one rounding
}

template <class LT>
__device__ __forceinline__ float sb_phif_s(float x, const LT& lt) {
    x = fminf(fmaxf(x, 8.5e-8f), 16.635532f);
    float t = sb_expf_inrange(x);
    return __fsub_rn(sb_logf_tab_s(__fadd_rn(t, 1.0f), lt), sb_logf_tab_s(__fadd_rn(t, -1.0f), lt));
}
