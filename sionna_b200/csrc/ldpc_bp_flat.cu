// ldpc_bp_flat.cu -- the UNFUSED belief-propagation path: one launch per half-iteration on message tensors of shape
// [num_edges, batch] in the reference's own layouts, so that Python callbacks and user-supplied node updates can see and
// modify the messages between the half-iterations exactly where the reference calls them
// (/root/reference/src/sionna/phy/fec/ldpc/decoding.py:464-524: CN update -> c2v_callbacks -> VN update ->
// v2c_callbacks). The fused kernels (ldpc_bp.cu / ldpc_bp_qc.cu) keep messages in shared memory and never use this file.
//
// Layouts (decoding.py:277-345):
//   msg_v2c [E, B]   VN order: edge e belongs to VN vn_of_edge[e]; edges of VN v are vn_ptr[v] .. vn_ptr[v+1]
//   msg_c2v [E, B]   CN-view order: position j holds the message of edge v2c_perm[j]; CN c owns positions
//                    cn_ptr[c] .. cn_ptr[c+1]; the VN side finds its message at c2v_perm[e]
//   llr_ch / x_hat [N, B]
// A thread owns one (node, batch column) pair, batch columns are consecutive in memory: every access is coalesced over b.
// Node reductions run sequentially in the REFERENCE's list orders (the arithmetic is ldpc_rules.cuh, the same code the
// shared-memory kernel runs), so this path equals the fused generic kernel with sum_order="reference" bit for bit.
#include <algorithm>
#include "sb_common.h"
#include "ldpc_rules.cuh"

namespace {

// llr[v, b] = -x[b, v] (decoding.py:565), 32 x 32 tiles through shared memory
__global__ void flat_transpose_neg_kernel(const float* __restrict__ x, float* __restrict__ llr, long long B, int N) {
    __shared__ float tile[32][33];
    const long long tiles_b = (B + 31) / 32;
    const int tiles_n = (N + 31) / 32;
    for (long long t = blockIdx.x; t < tiles_b * tiles_n; t += gridDim.x) {
        const long long b0 = (t / tiles_n) * 32;
        const int n0 = (int)(t % tiles_n) * 32;
        __syncthreads();
        for (int i = threadIdx.y; i < 32; i += blockDim.y) {
            const long long b = b0 + i;
            const int v = n0 + threadIdx.x;
            tile[i][threadIdx.x] = (b < B && v < N) ? x[b * N + v] : 0.f;
        }
        __syncthreads();
        for (int i = threadIdx.y; i < 32; i += blockDim.y) {
            const int v = n0 + i;
            const long long b = b0 + threadIdx.x;
            if (v < N && b < B) llr[(long long)v * B + b] = __fmul_rn(tile[threadIdx.x][i], -1.f);
        }
    }
}

// msg_v2c[e, b] = llr[vn_of_edge[e], b] (decoding.py:571) or -state[e, b] (:573)
__global__ void flat_init_v2c_kernel(const float* __restrict__ llr, const int* __restrict__ vn_of_edge,
                                     const float* __restrict__ state, float* __restrict__ v2c, long long B, int E) {
    const long long total = (long long)E * B;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long e = i / B, b = i - e * B;
        v2c[i] = state ? __fmul_rn(state[i], -1.f) : llr[(long long)vn_of_edge[e] * B + b];
    }
}

struct FlatEdges {                                               // edges of one CN, one batch column
    const float* v2c;                                            // + b
    float* c2v;                                                  // + (first position) * B + b
    const int* perm;                                             // v2c_perm + first position
    long long B;
    __device__ __forceinline__ float in(int l) const { return v2c[(long long)perm[l] * B]; }
    __device__ __forceinline__ void out(int l, float v) const { c2v[(long long)l * B] = v; }
    __device__ __forceinline__ float staged(int l) const { return c2v[(long long)l * B]; }
};

// CN update of the listed check nodes (cn_list == nullptr: all C of them, flooding)
template <int RULE>
__global__ void flat_cn_kernel(const float* __restrict__ v2c, float* __restrict__ c2v, const int* __restrict__ cn_ptr,
                               const int* __restrict__ v2c_perm, const int* __restrict__ cn_list, int n_nodes, long long B,
                               float clip, float offset) {
    const long long total = (long long)n_nodes * B;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long a = i / B, b = i - a * B;
        const int c = cn_list ? cn_list[a] : (int)a;
        const int j0 = cn_ptr[c], deg = cn_ptr[c + 1] - j0;
        FlatEdges e{v2c + b, c2v + (long long)j0 * B + b, v2c_perm + j0, B};
        cn_node<RULE>(e, deg, clip, offset);
    }
}

// VN update (decoding.py:714-732) of every variable node; vn_rule 1 = identity (:677-679)
__global__ void flat_vn_kernel(const float* __restrict__ c2v, const float* __restrict__ llr, const int* __restrict__ vn_ptr,
                               const int* __restrict__ c2v_perm, float* __restrict__ v2c, float* __restrict__ xhat, int N,
                               long long B, int vn_rule, float clip) {
    const long long total = (long long)N * B;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long v = i / B, b = i - v * B;
        const int e0 = vn_ptr[v], deg = vn_ptr[v + 1] - e0;
        float acc = 0.f;
        for (int k = 0; k < deg; ++k) acc = __fadd_rn(acc, c2v[(long long)c2v_perm[e0 + k] * B + b]);   // :715
        float x_tot = __fadd_rn(acc, llr[i]);                                                          // :716
        if (vn_rule == SB_VN_SUM) {
            for (int k = 0; k < deg; ++k) {
                const float m = c2v[(long long)c2v_perm[e0 + k] * B + b];
                v2c[(long long)(e0 + k) * B + b] = clipf(__fadd_rn(-m, x_tot), clip);                  // :724-729
            }
            x_tot = clipf(x_tot, clip);                                                                // :730
        } else {
            for (int k = 0; k < deg; ++k) v2c[(long long)(e0 + k) * B + b] = c2v[(long long)c2v_perm[e0 + k] * B + b];
        }
        xhat[i] = x_tot;
    }
}

// out[b, o] from x_hat[out_vn[o], b]: hard decision (decoding.py:622-624) or soft logit (:626)
__global__ void flat_out_kernel(const float* __restrict__ xhat, const int* __restrict__ out_vn, float* __restrict__ out,
                                long long B, int n_out, int hard_out) {
    const long long total = B * n_out;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long b = i / n_out;
        const int o = (int)(i - b * n_out);
        const float x = xhat[(long long)out_vn[o] * B + b];
        out[i] = hard_out ? (0.f >= x ? 1.f : 0.f) : __fmul_rn(x, -1.f);
    }
}

__global__ void flat_negate_kernel(const float* __restrict__ x, float* __restrict__ y, long long n) {
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
        y[i] = __fmul_rn(x[i], -1.f);
}

}  // namespace

extern "C" int sb_ldpc_flat_init(const float* d_x, const int32_t* d_vn_of_edge, const float* d_state_in, float* d_llr,
                                 float* d_v2c, int64_t batch, int32_t num_vn, int32_t num_edges, void* stream) {
    if (batch == 0) return SB_OK;
    SB_CHECK_ARG(d_x && d_vn_of_edge && d_llr && d_v2c && batch > 0 && num_vn > 0 && num_edges >= 0, "sb_ldpc_flat_init: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    const long long tiles = ((batch + 31) / 32) * ((num_vn + 31) / 32);
    flat_transpose_neg_kernel<<<sb_grid(tiles, 1, 16), dim3(32, 8, 1), 0, st>>>(d_x, d_llr, batch, num_vn);
    SB_LAUNCH_CHECK();
    if (num_edges > 0) {
        flat_init_v2c_kernel<<<sb_grid((long long)num_edges * batch, 256, 16), 256, 0, st>>>(d_llr, d_vn_of_edge, d_state_in,
                                                                                                d_v2c, batch, num_edges);
        SB_LAUNCH_CHECK();
    }
    return SB_OK;
}

extern "C" int sb_ldpc_flat_cn(const float* d_v2c, float* d_c2v, const int32_t* d_cn_ptr, const int32_t* d_v2c_perm,
                               const int32_t* d_cn_list, int32_t num_nodes, int64_t batch, int32_t cn_rule, float offset,
                               float llr_max, void* stream) {
    if (batch == 0 || num_nodes == 0) return SB_OK;
    SB_CHECK_ARG(d_v2c && d_c2v && d_cn_ptr && d_v2c_perm && num_nodes > 0 && batch > 0 && llr_max >= 0.f,
                 "sb_ldpc_flat_cn: bad arguments");
    SB_CHECK_ARG(cn_rule >= SB_CN_BOXPLUS_PHI && cn_rule <= SB_CN_IDENTITY, "sb_ldpc_flat_cn: unknown cn_rule %d", cn_rule);
    cudaStream_t st = (cudaStream_t)stream;
    const int grid = sb_grid((long long)num_nodes * batch, 128, 16);
    sb_dispatch<SB_CN_BOXPLUS_PHI, SB_CN_IDENTITY>(cn_rule, [&](auto R) {
        flat_cn_kernel<R><<<grid, 128, 0, st>>>(d_v2c, d_c2v, d_cn_ptr, d_v2c_perm, d_cn_list, num_nodes, batch, llr_max, offset);
        return SB_OK;
    });
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_ldpc_flat_vn(const float* d_c2v, const float* d_llr, const int32_t* d_vn_ptr, const int32_t* d_c2v_perm,
                               float* d_v2c, float* d_xhat, int32_t num_vn, int64_t batch, int32_t vn_rule, float llr_max,
                               void* stream) {
    if (batch == 0) return SB_OK;
    SB_CHECK_ARG(d_c2v && d_llr && d_vn_ptr && d_c2v_perm && d_v2c && d_xhat && num_vn > 0 && batch > 0 && llr_max >= 0.f &&
                     (vn_rule == SB_VN_SUM || vn_rule == SB_VN_IDENTITY), "sb_ldpc_flat_vn: bad arguments");
    flat_vn_kernel<<<sb_grid((long long)num_vn * batch, 128, 16), 128, 0, (cudaStream_t)stream>>>(
        d_c2v, d_llr, d_vn_ptr, d_c2v_perm, d_v2c, d_xhat, num_vn, batch, vn_rule, llr_max);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_ldpc_flat_out(const float* d_xhat, const int32_t* d_out_vn, float* d_out, const float* d_v2c,
                                float* d_state_out, int64_t batch, int32_t n_out, int32_t num_edges, int32_t hard_out,
                                void* stream) {
    if (batch == 0) return SB_OK;
    SB_CHECK_ARG(d_xhat && d_out_vn && d_out && batch > 0 && n_out > 0, "sb_ldpc_flat_out: bad arguments");
    cudaStream_t st = (cudaStream_t)stream;
    flat_out_kernel<<<sb_grid(batch * n_out, 256, 16), 256, 0, st>>>(d_xhat, d_out_vn, d_out, batch, n_out, hard_out);
    SB_LAUNCH_CHECK();
    if (d_state_out && d_v2c && num_edges > 0) {
        const long long n = (long long)num_edges * batch;
        flat_negate_kernel<<<sb_grid(n, 256, 16), 256, 0, st>>>(d_v2c, d_state_out, n);       // :636
        SB_LAUNCH_CHECK();
    }
    return SB_OK;
}
