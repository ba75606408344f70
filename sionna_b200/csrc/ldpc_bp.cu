// ldpc_bp.cu -- LDPC belief-propagation decoder for sm_90a, one CTA per codeword, all edge messages
// of the codeword resident in shared memory for every iteration.
//
// Replaces (all under /root/reference/src/sionna/phy/fec/ldpc/decoding.py):
//   graph set-up :277-345, LDPCBPDecoder.call :544-637, _bp_iter :416-524, vn_update_sum :681-732,
//   cn_update_offset_minsum :755-909, cn_update_minsum :911-953, cn_update_tanh :955-1043,
//   cn_update_phi :1045-1166, LDPC5GDecoder.call rate recovery :1427-1536.
//
// Data layout (see DESIGN.md "LDPC BP"):
//   * Edge messages live in "slots". CNs are ranked by degree (descending, stable); slot of the l-th
//     edge (ascending VN) of the CN with rank r is cn_off[l] + r  (jagged-diagonal storage). A warp
//     handling 32 consecutive ranks touches 32 consecutive slots per level: bank-conflict free.
//   * VNs are ranked the same way; vn_slot[vn_off[l] + r] is the slot of the l-th edge (ascending CN) of
//     the VN with rank r. For quasi-cyclic codes (5G) consecutive VNs of a circulant hit consecutive
//     slots (mod the wrap), so the gather is conflict free as well.
//   * Flooding keeps ONE message array: the CN phase overwrites v2c by c2v in place, the VN phase
//     overwrites c2v by v2c in place (every edge belongs to exactly one CN and one VN). A custom CN
//     schedule (layered) needs both arrays (decoding.py:489-497 updates a subset of c2v only).
//   * The codeword's input row is fetched with one TMA bulk copy (cp.async.bulk + mbarrier) into the
//     not-yet-used message array, then scattered into the rank-ordered channel-LLR array.
//   * Graphs whose messages do not fit in shared memory run the same kernel with the message arrays in
//     an L2-resident per-CTA global workspace (SMEM=false instantiation).
// Arithmetic: fp32, reductions run sequentially in list order, transcendental functions from sb_math.h
// so that the CPU oracle (oracle/ldpc_bp_ref.c, math_mode 1) reproduces the results bit for bit.
#include <algorithm>
#include <numeric>
#include <vector>
#include "sb_common.h"
#include "sb_math.h"
#include "ldpc_graph.h"
#include "ldpc_rules.cuh"

namespace {

struct BpParams {
    int C, N, E, Lc, Lv;
    const int* cn_off;       // [Lc+1]
    const int* cn_cnt;       // [Lc]
    const int* vn_off;       // [Lv+1]
    const int* vn_cnt;       // [Lv]
    const void* vn_slot;     // uint16_t[E] (SMEM) or uint32_t[E]
    const int* in_idx;       // [N] by VN rank: >=0 input column, -1 punctured, -2 filler
    const int* out_pos;      // [N] by VN rank: output column or -1
    const int* slot_of_edge; // [E] reference edge number -> slot
    const int* sched;        // [n_sub*n_active] CN ranks, or nullptr (flooding)
    int n_sub, n_active, n_in, n_out;
    const float* llr;
    float* out;
    const float* state_in;
    float* state_out;
    long long B;
    int num_iter, vn_rule, hard_out, two_arrays, use_tma;
    float offset, llr_max;
    float* ws;
};

// ---- check-node updates (ldpc_rules.cuh) on the slot layout: l-th edge of the CN with rank r at off[l] + r ---------
struct SlotEdges {
    const float* v2c;
    float* c2v;
    const int* off;
    int r;
    __device__ __forceinline__ float in(int l) const { return v2c[off[l] + r]; }
    __device__ __forceinline__ void out(int l, float v) const { c2v[off[l] + r] = v; }
    __device__ __forceinline__ float staged(int l) const { return c2v[off[l] + r]; }
};

// degree of rank r given non-increasing level counts; `deg` is a hint from the previous (smaller) rank
__device__ __forceinline__ int rank_degree(const int* cnt, int L, int r, int deg) {
    while (deg > 0 && r >= cnt[deg - 1]) --deg;
    (void)L;
    return deg;
}

template <int RULE, bool SMEM>
__global__ void __launch_bounds__(1024, 1) ldpc_bp_kernel(const __grid_constant__ BpParams p) {
    using SlotT = typename std::conditional<SMEM, uint16_t, uint32_t>::type;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int T = blockDim.x, tid = threadIdx.x;
    const int E = p.E, N = p.N, C = p.C;

    // shared memory carve-up: [v2c E][c2v E (two_arrays)] (SMEM only) | llr N | tables | mbarrier
    float* sm = reinterpret_cast<float*>(smem_raw);
    float* v2c;
    float* c2v;
    float* llr_s;
    if (SMEM) {
        v2c = sm;
        c2v = p.two_arrays ? sm + E : sm;
        llr_s = sm + (p.two_arrays ? 2 : 1) * (size_t)E;
    } else {
        float* base = p.ws + (size_t)blockIdx.x * (size_t)(p.two_arrays ? 2 : 1) * (size_t)E;
        v2c = base;
        c2v = p.two_arrays ? base + E : base;
        llr_s = sm;
    }
    int* s_cn_off = reinterpret_cast<int*>(llr_s + N);
    int* s_cn_cnt = s_cn_off + p.Lc + 1;
    int* s_vn_off = s_cn_cnt + p.Lc;
    int* s_vn_cnt = s_vn_off + p.Lv + 1;
    uint64_t* bar = reinterpret_cast<uint64_t*>((reinterpret_cast<uintptr_t>(s_vn_cnt + p.Lv) + 15) & ~(uintptr_t)15);

    for (int i = tid; i <= p.Lc; i += T) s_cn_off[i] = p.cn_off[i];
    for (int i = tid; i < p.Lc; i += T) s_cn_cnt[i] = p.cn_cnt[i];
    for (int i = tid; i <= p.Lv; i += T) s_vn_off[i] = p.vn_off[i];
    for (int i = tid; i < p.Lv; i += T) s_vn_cnt[i] = p.vn_cnt[i];
    if (SMEM && p.use_tma && tid == 0) mbar_init(bar);
    __syncthreads();

    const SlotT* __restrict__ vn_slot = reinterpret_cast<const SlotT*>(p.vn_slot);
    const float clip = p.llr_max;
    uint32_t tma_phase = 0;
    const int n_cn_items = p.sched ? p.n_active : C;

    for (long long b = blockIdx.x; b < p.B; b += gridDim.x) {
        // ---- channel LLRs by VN rank, staged in the message array -----------------------------------
        load_channel_llr(llr_s, p.llr + (size_t)b * p.n_in, p.in_idx, N, p.n_in, clip, SMEM && p.use_tma, v2c, bar,
                         tma_phase, tid, T);
        __syncthreads();
        // ---- initial messages: v2c = llr of the edge's VN (:571) or the caller's state (:573); c2v = 0
        if (p.state_in) {
            const float* st = p.state_in + (size_t)b * E;
            for (int e = tid; e < E; e += T) v2c[p.slot_of_edge[e]] = __fmul_rn(st[e], -1.f);
        } else {
            int deg = p.Lv;
            for (int r = tid; r < N; r += T) {
                deg = rank_degree(s_vn_cnt, p.Lv, r, deg);
                float l = llr_s[r];
                for (int k = 0; k < deg; ++k) v2c[vn_slot[s_vn_off[k] + r]] = l;
            }
        }
        if (p.two_arrays)
            for (int e = tid; e < E; e += T) c2v[e] = 0.f;
        __syncthreads();

        if (p.num_iter == 0) {                           // x_hat = llr_ch (decoding.py:603-608)
            for (int v = tid; v < N; v += T) {
                int o = p.out_pos[v];
                if (o >= 0) p.out[(size_t)b * p.n_out + o] = decoder_out(llr_s[v], p.hard_out);
            }
        }

        for (int it = 0; it < p.num_iter; ++it) {
            for (int j = 0; j < p.n_sub; ++j) {
                // ---- CN phase (:479-500) -----------------------------------------------------------
                {
                    int deg = p.Lc;
                    for (int i = tid; i < n_cn_items; i += T) {
                        int r = p.sched ? p.sched[(size_t)j * p.n_active + i] : i;
                        if (p.sched) { deg = 0; while (deg < p.Lc && r < s_cn_cnt[deg]) ++deg; }
                        else deg = rank_degree(s_cn_cnt, p.Lc, r, deg);
                        cn_node<RULE>(SlotEdges{v2c, c2v, s_cn_off, r}, deg, clip, p.offset);
                    }
                }
                __syncthreads();
                // ---- VN phase (:506-519, vn_update_sum :714-732) -----------------------------------
                const bool final_pass = (it == p.num_iter - 1) && (j == p.n_sub - 1);
                {
                    int deg = p.Lv;
                    for (int r = tid; r < N; r += T) {
                        deg = rank_degree(s_vn_cnt, p.Lv, r, deg);
                        float acc = 0.f;
#pragma unroll 4
                        for (int k = 0; k < deg; ++k) acc = __fadd_rn(acc, c2v[vn_slot[s_vn_off[k] + r]]);   // :715
                        float x_tot = __fadd_rn(acc, llr_s[r]);                                               // :716
                        if (p.vn_rule == SB_VN_SUM) {
#pragma unroll 4
                            for (int k = 0; k < deg; ++k) {
                                int s = vn_slot[s_vn_off[k] + r];
                                v2c[s] = clipf(__fadd_rn(-c2v[s], x_tot), clip);                              // :724-729
                            }
                            x_tot = clipf(x_tot, clip);                                                       // :730
                        } else if (p.two_arrays) {
                            for (int k = 0; k < deg; ++k) {
                                int s = vn_slot[s_vn_off[k] + r];
                                v2c[s] = c2v[s];                                                              // :679
                            }
                        }
                        if (final_pass) {
                            int o = p.out_pos[r];
                            if (o >= 0) p.out[(size_t)b * p.n_out + o] = decoder_out(x_tot, p.hard_out);
                        }
                    }
                }
                __syncthreads();
            }
        }
        if (p.state_out) {
            store_state(p.state_out + (size_t)b * E, v2c, p.slot_of_edge, E, tid, T);
            __syncthreads();
        }
    }
}

}  // namespace

// ------------------------------------------------------------------------------------------------------
// Host side: graph plan (pure host), launch.
// ------------------------------------------------------------------------------------------------------

static size_t bp_smem_bytes(const sb_ldpc_graph* g, bool smem_msgs) {
    size_t arrays = g->flooding ? 1 : 2;
    size_t floats = (smem_msgs ? arrays * (size_t)g->E : 0) + (size_t)g->N;
    size_t ints = (size_t)(2 * g->Lc + 2 * g->Lv + 2);
    return floats * 4 + ints * 4 + 16 + 16;
}

// h_cn_view (optional, [E]): the reference's CN-view permutation v2c_perm = np.argsort(cn_idx) (decoding.py:329): the
// edges of a CN are then walked in that order and the edges of a VN in ascending edge number (the reference's VN order,
// decoding.py:286-288) instead of ascending neighbour index, so that every sequential sum runs in the reference's order.
static int graph_create_impl(sb_ldpc_graph** out, int32_t num_cn, int32_t num_vn, int32_t num_edges,
                             const int32_t* h_cn, const int32_t* h_vn, const int32_t* h_in_map, int32_t n_in,
                             const int32_t* h_out_vn, int32_t n_out, const int32_t* h_sched, int32_t n_sub,
                             int32_t n_active, const int32_t* h_cn_view) {
    SB_CHECK_ARG(out && num_cn > 0 && num_vn > 0 && num_edges >= 0 && (num_edges == 0 || (h_cn && h_vn)),
                 "sb_ldpc_graph_create: bad sizes/pointers");
    auto* g = new sb_ldpc_graph();
    g->C = num_cn; g->N = num_vn; g->E = num_edges;
    g->h_cn.assign(h_cn, h_cn + num_edges); g->h_vn.assign(h_vn, h_vn + num_edges);
    const int C = num_cn, N = num_vn, E = num_edges;
    std::vector<int> cdeg(C, 0), vdeg(N, 0);
    for (int e = 0; e < E; ++e) {
        if (h_cn[e] < 0 || h_cn[e] >= C || h_vn[e] < 0 || h_vn[e] >= N) {
            delete g;
            sb_set_error("sb_ldpc_graph_create: edge %d out of range", e);
            return SB_EINVAL;
        }
        ++cdeg[h_cn[e]]; ++vdeg[h_vn[e]];
    }
    // rank nodes by degree, descending, stable
    g->cn_order.resize(C); std::iota(g->cn_order.begin(), g->cn_order.end(), 0);
    std::stable_sort(g->cn_order.begin(), g->cn_order.end(), [&](int a, int b) { return cdeg[a] > cdeg[b]; });
    g->vn_order.resize(N); std::iota(g->vn_order.begin(), g->vn_order.end(), 0);
    std::stable_sort(g->vn_order.begin(), g->vn_order.end(), [&](int a, int b) { return vdeg[a] > vdeg[b]; });
    std::vector<int> crank(C), vrank(N);
    for (int r = 0; r < C; ++r) crank[g->cn_order[r]] = r;
    for (int r = 0; r < N; ++r) vrank[g->vn_order[r]] = r;
    g->Lc = C ? cdeg[g->cn_order[0]] : 0;
    g->Lv = N ? vdeg[g->vn_order[0]] : 0;
    g->cn_cnt.assign(g->Lc, 0); g->vn_cnt.assign(g->Lv, 0);
    for (int c = 0; c < C; ++c) for (int l = 0; l < cdeg[c]; ++l) ++g->cn_cnt[l];
    for (int v = 0; v < N; ++v) for (int l = 0; l < vdeg[v]; ++l) ++g->vn_cnt[l];
    g->cn_off.assign(g->Lc + 1, 0); g->vn_off.assign(g->Lv + 1, 0);
    for (int l = 0; l < g->Lc; ++l) g->cn_off[l + 1] = g->cn_off[l] + g->cn_cnt[l];
    for (int l = 0; l < g->Lv; ++l) g->vn_off[l + 1] = g->vn_off[l] + g->vn_cnt[l];
    // per-CN edge lists: ascending VN, or (reference order) the position in the caller's CN view
    std::vector<std::vector<std::pair<int, int>>> cl(C), vl(N);
    g->ref_order = h_cn_view != nullptr;
    if (h_cn_view) {
        std::vector<char> seen(E, 0);
        for (int j = 0; j < E; ++j) {
            int e = h_cn_view[j];
            if (e < 0 || e >= E || seen[e]) { delete g; sb_set_error("sb_ldpc_graph_create_ordered: cn_view is not a permutation"); return SB_EINVAL; }
            seen[e] = 1;
            cl[h_cn[e]].push_back({j, e});
        }
    } else {
        for (int e = 0; e < E; ++e) cl[h_cn[e]].push_back({h_vn[e], e});
    }
    g->slot_of_edge.assign(E, 0);
    {
        std::vector<long long> keys(E);
        for (int e = 0; e < E; ++e) keys[e] = ((long long)h_cn[e] << 32) | (unsigned)h_vn[e];
        std::sort(keys.begin(), keys.end());
        for (int e = 1; e < E; ++e)
            if (keys[e] == keys[e - 1]) {
                delete g;
                sb_set_error("sb_ldpc_graph_create: duplicate edge (cn %d, vn %d)", (int)(keys[e] >> 32), (int)(keys[e] & 0xffffffff));
                return SB_EINVAL;
            }
    }
    for (int c = 0; c < C; ++c) {
        std::sort(cl[c].begin(), cl[c].end());
        for (size_t l = 0; l < cl[c].size(); ++l) g->slot_of_edge[cl[c][l].second] = g->cn_off[l] + crank[c];
    }
    // per-VN slot lists: ascending CN, or (reference order) ascending edge number
    for (int e = 0; e < E; ++e) vl[h_vn[e]].push_back({h_cn_view ? e : h_cn[e], g->slot_of_edge[e]});
    g->vn_slot.assign(E, 0);
    for (int v = 0; v < N; ++v) {
        std::sort(vl[v].begin(), vl[v].end());
        for (size_t l = 0; l < vl[v].size(); ++l) g->vn_slot[g->vn_off[l] + vrank[v]] = (uint32_t)vl[v][l].second;
    }
    // rate-recovery maps
    g->n_in = h_in_map ? n_in : N;
    g->n_out = h_out_vn ? n_out : N;
    if ((!h_in_map && n_in != N && n_in != 0) || (!h_out_vn && n_out != N && n_out != 0) || g->n_in <= 0 || g->n_out <= 0) {
        delete g;
        sb_set_error("sb_ldpc_graph_create: identity maps need n_in == n_out == num_vn");
        return SB_EINVAL;
    }
    g->in_idx.resize(N); g->out_pos.assign(N, -1);
    for (int r = 0; r < N; ++r) {
        int v = g->vn_order[r];
        int ii = h_in_map ? h_in_map[v] : v;
        if (ii < -2 || ii >= g->n_in) { delete g; sb_set_error("sb_ldpc_graph_create: in_map[%d]=%d out of range", v, ii); return SB_EINVAL; }
        g->in_idx[r] = ii;
    }
    for (int j = 0; j < g->n_out; ++j) {
        int v = h_out_vn ? h_out_vn[j] : j;
        if (v < 0 || v >= N) { delete g; sb_set_error("sb_ldpc_graph_create: out_vn[%d]=%d out of range", j, v); return SB_EINVAL; }
        if (g->out_pos[vrank[v]] != -1) { delete g; sb_set_error("sb_ldpc_graph_create: VN %d appears twice in out_vn", v); return SB_EINVAL; }
        g->out_pos[vrank[v]] = j;
    }
    // schedule
    if (h_sched) {
        if (n_sub <= 0 || n_active <= 0) { delete g; sb_set_error("sb_ldpc_graph_create: bad schedule shape"); return SB_EINVAL; }
        g->flooding = false; g->n_sub = n_sub; g->n_active = n_active;
        g->sched.resize((size_t)n_sub * n_active);
        for (size_t i = 0; i < g->sched.size(); ++i) {
            if (h_sched[i] < 0 || h_sched[i] >= C) { delete g; sb_set_error("sb_ldpc_graph_create: schedule entry out of range"); return SB_EINVAL; }
            g->sched[i] = crank[h_sched[i]];
        }
    } else {
        g->flooding = true; g->n_sub = 1; g->n_active = C;
    }
    g->vn_slot16.assign(g->vn_slot.begin(), g->vn_slot.end());
    g->tables.set(g->cn_off, g->cn_cnt, g->vn_off, g->vn_cnt, g->in_idx, g->out_pos, g->slot_of_edge, g->sched, g->vn_slot,
                  g->vn_slot16);
    *out = g;
    return SB_OK;
}

extern "C" int sb_ldpc_graph_create(sb_ldpc_graph** out, int32_t num_cn, int32_t num_vn, int32_t num_edges,
                                    const int32_t* h_cn, const int32_t* h_vn, const int32_t* h_in_map, int32_t n_in,
                                    const int32_t* h_out_vn, int32_t n_out, const int32_t* h_sched, int32_t n_sub,
                                    int32_t n_active) {
    return graph_create_impl(out, num_cn, num_vn, num_edges, h_cn, h_vn, h_in_map, n_in, h_out_vn, n_out, h_sched, n_sub,
                             n_active, nullptr);
}

extern "C" int sb_ldpc_graph_create_ordered(sb_ldpc_graph** out, int32_t num_cn, int32_t num_vn, int32_t num_edges,
                                            const int32_t* h_cn, const int32_t* h_vn, const int32_t* h_in_map,
                                            int32_t n_in, const int32_t* h_out_vn, int32_t n_out, const int32_t* h_sched,
                                            int32_t n_sub, int32_t n_active, const int32_t* h_cn_view) {
    SB_CHECK_ARG(h_cn_view || num_edges == 0, "sb_ldpc_graph_create_ordered: null cn_view");
    return graph_create_impl(out, num_cn, num_vn, num_edges, h_cn, h_vn, h_in_map, n_in, h_out_vn, n_out, h_sched, n_sub,
                             n_active, h_cn_view);
}

extern "C" void sb_ldpc_graph_destroy(sb_ldpc_graph* g) { delete g; }

static bool graph_on_chip(const sb_ldpc_graph* g, int smem_optin) {
    return g->E <= 65535 && bp_smem_bytes(g, true) <= (size_t)smem_optin;
}

// The current device's opt-in shared memory once the graph has been used there, else the H100's.
static int planning_smem_optin(const sb_ldpc_graph* g) {
    const DeviceTables::Copy* d = g->tables.find();
    return d ? d->smem_optin : kSmemOptinH100;
}

extern "C" int sb_ldpc_graph_on_chip(const sb_ldpc_graph* g) {
    if (!g) return 0;
    return graph_on_chip(g, planning_smem_optin(g)) ? 1 : 0;
}

// upper bound on resident CTAs the launcher will ever use (grid is capped to it)
static const int kMaxGrid = 132 * 8;

static size_t workspace_bytes(const sb_ldpc_graph* g, int smem_optin) {
    if (graph_on_chip(g, smem_optin)) return 0;
    return (size_t)kMaxGrid * (g->flooding ? 1 : 2) * (size_t)g->E * sizeof(float);
}

extern "C" size_t sb_ldpc_workspace_bytes(const sb_ldpc_graph* g) {
    return g ? workspace_bytes(g, planning_smem_optin(g)) : 0;
}

static int pick_threads(const sb_ldpc_graph* g) {
    int m = std::max(g->flooding ? g->C : g->n_active, g->N);
    if (m <= 1024) return std::max(32, (m + 31) / 32 * 32);
    int best = 1024;
    double best_cost = 1e30;
    for (int t = 1024; t >= 512; t -= 64) {
        auto waste = [&](int items) { return (double)((items + t - 1) / t) * t / items; };
        double cost = waste(g->flooding ? g->C : g->n_active) + waste(g->N);
        if (cost < best_cost - 1e-9) { best_cost = cost; best = t; }
    }
    return best;
}

static int ldpc_decode_impl(const sb_ldpc_graph* g, const float* d_llr, int64_t batch, int32_t num_iter, int32_t cn_rule,
                            int32_t vn_rule, float offset, float llr_max, int32_t hard_out, const float* d_state_in,
                            float* d_state_out, float* d_out, void* d_ws, size_t ws_bytes, void* stream, int32_t early,
                            int32_t* d_iters);

extern "C" int sb_ldpc_decode(const sb_ldpc_graph* gc, const float* d_llr, int64_t batch, int32_t num_iter,
                              int32_t cn_rule, int32_t vn_rule, float offset, float llr_max, int32_t hard_out,
                              const float* d_state_in, float* d_state_out, float* d_out, void* d_ws,
                              size_t ws_bytes, void* stream) {
    return ldpc_decode_impl(gc, d_llr, batch, num_iter, cn_rule, vn_rule, offset, llr_max, hard_out, d_state_in, d_state_out,
                            d_out, d_ws, ws_bytes, stream, 0, nullptr);
}

extern "C" int sb_ldpc_decode_early(const sb_ldpc_graph* gc, const float* d_llr, int64_t batch, int32_t max_iter,
                                    int32_t cn_rule, float offset, float llr_max, int32_t hard_out, float* d_out,
                                    int32_t* d_num_iter, void* stream) {
    return ldpc_decode_impl(gc, d_llr, batch, max_iter, cn_rule, SB_VN_SUM, offset, llr_max, hard_out, nullptr, nullptr, d_out,
                            nullptr, 0, stream, 1, d_num_iter);
}

static int ldpc_decode_impl(const sb_ldpc_graph* g, const float* d_llr, int64_t batch, int32_t num_iter, int32_t cn_rule,
                            int32_t vn_rule, float offset, float llr_max, int32_t hard_out, const float* d_state_in,
                            float* d_state_out, float* d_out, void* d_ws, size_t ws_bytes, void* stream, int32_t early,
                            int32_t* d_iters) {
    if (batch == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(g && d_llr && d_out, "sb_ldpc_decode: null graph/input/output");
    SB_CHECK_ARG(batch >= 0 && num_iter >= 0, "sb_ldpc_decode: negative batch or num_iter");
    SB_CHECK_ARG(cn_rule >= SB_CN_BOXPLUS_PHI && cn_rule <= SB_CN_IDENTITY, "sb_ldpc_decode: unknown cn_rule %d", cn_rule);
    SB_CHECK_ARG(vn_rule == SB_VN_SUM || vn_rule == SB_VN_IDENTITY, "sb_ldpc_decode: unknown vn_rule %d", vn_rule);
    SB_CHECK_ARG(llr_max >= 0.f, "sb_ldpc_decode: llr_max must be >= 0");
    const DeviceTables::Copy* d = nullptr;
    int rc = g->tables.get(&d);
    if (rc) return rc;
    {   // quasi-cyclic fast path (ldpc_bp_qc.cu) when the graph carries a QC description and the call qualifies
        bool handled = false;
        rc = sb_qc_try_decode(g, *d, d_llr, batch, num_iter, cn_rule, vn_rule, offset, llr_max, hard_out, d_state_in,
                              d_state_out, d_out, (cudaStream_t)stream, &handled, early, d_iters);
        if (rc || handled) return rc;
    }
    if (early) {
        sb_set_error("sb_ldpc_decode_early: early termination needs the quasi-cyclic on-chip path (5G codes, flooding)");
        return SB_EUNSUPPORTED;
    }
    const bool on_chip = graph_on_chip(g, d->smem_optin);
    BpParams p{};
    p.C = g->C; p.N = g->N; p.E = g->E; p.Lc = g->Lc; p.Lv = g->Lv;
    p.cn_off = d->at<int>(0); p.cn_cnt = d->at<int>(1); p.vn_off = d->at<int>(2); p.vn_cnt = d->at<int>(3);
    p.vn_slot = on_chip ? (const void*)d->at<uint16_t>(9) : (const void*)d->at<uint32_t>(8);
    p.in_idx = d->at<int>(4); p.out_pos = d->at<int>(5); p.slot_of_edge = d->at<int>(6);
    p.sched = g->flooding ? nullptr : d->at<int>(7);
    p.n_sub = g->n_sub; p.n_active = g->n_active; p.n_in = g->n_in; p.n_out = g->n_out;
    p.llr = d_llr; p.out = d_out; p.state_in = d_state_in; p.state_out = d_state_out;
    p.B = batch; p.num_iter = num_iter; p.vn_rule = vn_rule; p.hard_out = hard_out;
    // the identity VN rule leaves messages untouched: it needs c2v and v2c to be the same storage only
    // in flooding mode, where that is already the case
    p.two_arrays = g->flooding ? 0 : 1;
    p.offset = offset; p.llr_max = llr_max;
    p.ws = (float*)d_ws;
    p.use_tma = on_chip && (g->n_in % 4 == 0) && (g->n_in <= g->E) && ((reinterpret_cast<uintptr_t>(d_llr) & 15) == 0);
    if (!on_chip) {
        size_t need = workspace_bytes(g, d->smem_optin);
        if (!d_ws || ws_bytes < need) { sb_set_error("sb_ldpc_decode: workspace %zu < %zu bytes", ws_bytes, need); return SB_ENOMEM; }
    }
    const int threads = pick_threads(g);
    const size_t smem = bp_smem_bytes(g, on_chip);
    cudaStream_t st = (cudaStream_t)stream;
    return sb_dispatch<SB_CN_BOXPLUS_PHI, SB_CN_IDENTITY>(cn_rule, [&](auto R) {
        return sb_launch_decoder(on_chip ? ldpc_bp_kernel<R, true> : ldpc_bp_kernel<R, false>, p, d->num_sms, threads,
                                 smem, kMaxGrid, st, "sb_ldpc_decode");
    });
}

// Debug / test export of the host-side plan (no device needed): copies the tables into caller arrays.
// Any pointer may be NULL. Sizes: cn_order[C], vn_order[N], slot_of_edge[E], vn_slot[E],
// cn_off[Lc+1], vn_off[Lv+1]; dims = {C, N, E, Lc, Lv, n_in, n_out, n_sub, n_active, flooding}.
extern "C" int sb_ldpc_graph_export(const sb_ldpc_graph* g, int32_t* dims, int32_t* cn_order, int32_t* vn_order,
                                    int32_t* slot_of_edge, int32_t* vn_slot, int32_t* cn_off, int32_t* vn_off) {
    SB_CHECK_ARG(g, "sb_ldpc_graph_export: null graph");
    if (dims) {
        int v[10] = {g->C, g->N, g->E, g->Lc, g->Lv, g->n_in, g->n_out, g->n_sub, g->n_active, g->flooding ? 1 : 0};
        for (int i = 0; i < 10; ++i) dims[i] = v[i];
    }
    if (cn_order) std::copy(g->cn_order.begin(), g->cn_order.end(), cn_order);
    if (vn_order) std::copy(g->vn_order.begin(), g->vn_order.end(), vn_order);
    if (slot_of_edge) std::copy(g->slot_of_edge.begin(), g->slot_of_edge.end(), slot_of_edge);
    if (vn_slot) for (size_t i = 0; i < g->vn_slot.size(); ++i) vn_slot[i] = (int32_t)g->vn_slot[i];
    if (cn_off) std::copy(g->cn_off.begin(), g->cn_off.end(), cn_off);
    if (vn_off) std::copy(g->vn_off.begin(), g->vn_off.end(), vn_off);
    return SB_OK;
}
