// ldpc_graph.h -- decoding-graph handle shared by ldpc_bp.cu (generic kernel, graph construction) and
// ldpc_bp_qc.cu (quasi-cyclic fast path), plus small device helpers used by both kernels.
#pragma once
#include <stdint.h>
#include <algorithm>
#include <vector>
#include "sb_common.h"

struct sb_ldpc_graph {
    int C = 0, N = 0, E = 0, Lc = 0, Lv = 0, n_in = 0, n_out = 0, n_sub = 1, n_active = 0;
    bool flooding = true;
    bool ref_order = false;   // node sums follow the reference's list orders (sb_ldpc_graph_create_ordered)
    std::vector<int> cn_off, cn_cnt, vn_off, vn_cnt, in_idx, out_pos, slot_of_edge, sched, cn_order, vn_order;
    std::vector<uint32_t> vn_slot;
    std::vector<uint16_t> vn_slot16;   // vn_slot for the on-chip kernel (E <= 65535)
    std::vector<int> h_cn, h_vn;   // the caller's edge list (reference VN order), kept for sb_ldpc_graph_set_qc
    // device copies of cn_off, cn_cnt, vn_off, vn_cnt, in_idx, out_pos, slot_of_edge, sched, vn_slot, vn_slot16
    mutable DeviceTables tables;
    // ---- quasi-cyclic description (optional, set by sb_ldpc_graph_set_qc; used by ldpc_bp_qc.cu) ----------
    bool qc = false;
    int qc_Z = 0, qc_rows = 0, qc_cols = 0, qc_nnz = 0, qc_max_row_deg = 0, qc_max_col_deg = 0;
    std::vector<int> qc_row_info;   // int4 per base row (processing order): {first base entry, deg, zrow, fused col | s << 16 or -1}
    std::vector<int> qc_col_info;   // int4 per base col (processing order): {first col-edge, deg, zcol, c*Z}
    std::vector<int> qc_col_edge;   // int2 per (col, entry), ascending base row: {be*Z*4, s*4 | (zrow*4) << 16}
    std::vector<int> qc_in_idx, qc_out_pos, qc_slot_of_edge;   // natural VN order / reference edge order
    std::vector<int> qc_row_edge;   // int2 per base entry (processing order): {column * Z, shift} for the syndrome pass
    std::vector<int> qc_row_cls_end, qc_col_cls_end;   // class boundaries in processing order (ldpc_bp_qc.cu)
    bool qc_open = false;           // boxplus-phi runs its opening iterations on the punctured columns (ldpc_bp_qc.cu)
    std::vector<int> qc_open_tab;   // per row (processing order): punctured edge positions as a bit mask; then per col: punctured
    // device copies of qc_row_info, qc_col_info, qc_col_edge, qc_in_idx, qc_out_pos, qc_slot_of_edge, qc_row_edge,
    // qc_open_tab
    mutable DeviceTables qc_tables;
};

// H100 (sm_90) opt-in shared memory per block (227 KB); used for planning when no device is present.
static const int kSmemOptinH100 = 232448;

// ldpc_bp_qc.cu: runs the QC kernel if the graph / call qualifies; *handled tells the dispatcher. `dev` is the
// current device's copy of the generic tables.
int sb_qc_try_decode(const sb_ldpc_graph* g, const DeviceTables::Copy& dev, const float* d_llr, int64_t batch,
                     int32_t num_iter, int32_t cn_rule, int32_t vn_rule, float offset, float llr_max, int32_t hard_out,
                     const float* d_state_in, float* d_state_out, float* d_out, cudaStream_t stream, bool* handled,
                     int32_t early = 0, int32_t* d_iters = nullptr);

#if defined(__CUDACC__)
// Launch of a persistent decoder kernel: opts in to `smem` bytes of dynamic shared memory, checks that a CTA of
// `threads` fits on an SM, and runs min(batch, resident CTAs, max_grid) CTAs that stride over the codewords.
template <class Kernel, class Params>
int sb_launch_decoder(Kernel kern, const Params& p, int num_sms, int threads, size_t smem, long long max_grid,
                      cudaStream_t stream, const char* who) {
    SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ = 0;
    SB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, smem));
    if (occ < 1) { sb_set_error("%s: kernel does not fit (threads %d, smem %zu)", who, threads, smem); return SB_EUNSUPPORTED; }
    long long grid = std::min<long long>(p.B, std::min<long long>((long long)num_sms * occ, max_grid));
    kern<<<(unsigned)grid, threads, smem, stream>>>(p);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

__device__ __forceinline__ float clipf(float x, float c) { return fminf(fmaxf(x, -c), c); }

// ---- mbarrier / TMA bulk-copy helpers (cp.async.bulk, 1-D) ------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
// one-arrival barrier, made visible to the async proxy before the first bulk copy
__device__ __forceinline__ void mbar_init(uint64_t* bar) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(1));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                     smem_u32(dst_smem)),
                 "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
                 : "memory");
}

// ---- per-codeword steps of the fused decoder kernels (ldpc_bp.cu, ldpc_bp_qc.cu); thread tid of T ------------------
// Decoder output of a VN from its internal LLR (positive: bit 0): hard decision or logit (decoding.py:622-626).
__device__ __forceinline__ float decoder_out(float x, int hard_out) {
    return hard_out ? (0.f >= x ? 1.f : 0.f) : __fmul_rn(x, -1.f);
}

// Channel LLRs of one codeword, clipped and negated (decoding.py:552-565), with rate recovery (:1444-1475): in_idx[v] is
// the input column of VN v, -1 for a punctured VN (0) and -2 for a filler VN (-clip). With `tma`, thread 0 first copies
// the n_in inputs into `stage`, shared memory that is free until the messages are initialised.
__device__ __forceinline__ void load_channel_llr(float* llr_s, const float* row, const int* in_idx, int N, int n_in,
                                                 float clip, bool tma, float* stage, uint64_t* bar, uint32_t& phase,
                                                 int tid, int T) {
    if (tma) {
        if (tid == 0) {
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
            mbar_expect_tx(bar, (uint32_t)n_in * 4u);
            tma_bulk_g2s(stage, row, (uint32_t)n_in * 4u, bar);
        }
        mbar_wait(bar, phase);
        phase ^= 1u;
        for (int v = tid; v < N; v += T) {
            int ii = in_idx[v];
            float l = ii >= 0 ? stage[ii] : (ii == -1 ? 0.f : -clip);
            llr_s[v] = __fmul_rn(clipf(l, clip), -1.f);
        }
    } else {
        for (int v = tid; v < N; v += T) {
            int ii = in_idx[v];
            float l = ii >= 0 ? __ldg(row + ii) : (ii == -1 ? 0.f : -clip);
            llr_s[v] = __fmul_rn(clipf(l, clip), -1.f);
        }
    }
}

// Decoder state (decoding.py:636): the v2c message of every reference edge, as a logit.
__device__ __forceinline__ void store_state(float* st, const float* v2c, const int* slot_of_edge, int E, int tid, int T) {
    for (int e = tid; e < E; e += T) st[e] = __fmul_rn(v2c[slot_of_edge[e]], -1.f);
}

#endif
