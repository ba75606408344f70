// ldpc_enc.cu -- 5G NR LDPC encoder with rate matching, 32 codewords per CTA, bit-sliced (sm_90a).
// Replaces LDPC5GEncoder.call / _encode_fast / _matmul_gather
// (/root/reference/src/sionna/phy/fec/ldpc/encoding.py:599-668, 572-591, 559-570).
//
// Richardson-Urbanke encoding over GF(2): with H = [[A B 0],[C1 C2 I]] and s the k_ldpc information bits
// (fillers = 0),  p_a = B^-1 (A s),  p_b = C1 s + C2 p_a.  The reference evaluates each product as
// "gather columns, reduce_sum, finally AND 1"; parity of a sum == XOR of its terms, so every row is an XOR over
// its CSR column list. The whole codeword (n_ldpc bits, one 32-bit word per bit holding 32 codewords) lives in shared
// memory; the output gather
// applies filler removal, 2Z puncturing, truncation to n and the optional 38.212 5.4.2.2 interleaver
// (encoding.py:645-661) through one precomputed index list. HBM traffic per codeword: 4k bytes in, 4n out.
#include <algorithm>
#include <vector>
#include "sb_common.h"

struct sb_ldpc5g_encoder {
    int k = 0, n = 0, k_ldpc = 0, n_ldpc = 0, g = 0, m_rest = 0;   // g = 4Z rows of A / B^-1, m_rest rows of C1|C2
    std::vector<int> a_ptr, a_idx, b_ptr, b_idx, c1_ptr, c1_idx, c2_ptr, c2_idx, tx_vn;
    int rows_needed = 0;   // number of p_b rows any transmitted bit depends on
    mutable DeviceTables tables;   // device copies of the nine tables above, in that order
};

namespace {

struct EncParams {
    int k, n, k_ldpc, n_ldpc, g, rows_needed;
    const int *a_ptr, *a_idx, *b_ptr, *b_idx, *c1_ptr, *c1_idx, *c2_ptr, *c2_idx, *tx_vn;
    const float* u;
    float* c;
    long long B;
};

// Bit-sliced over the batch: a CTA encodes 32 codewords at once, word i of shared memory holds bit i of all 32 (lane b =
// codeword b), so every XOR of the sparse products serves 32 codewords and the CSR index lists are read once per 32
// codewords instead of once per codeword (the one-codeword-per-CTA version was bound by exactly that: 19.6 % of HBM).
// Global traffic stays the compulsory 4k bytes in + 4n bytes out per codeword, all of it coalesced.
__global__ void __launch_bounds__(512) ldpc5g_encode_kernel(const __grid_constant__ EncParams p) {
    extern __shared__ unsigned cw[];               // [n_ldpc] bit-sliced codeword words, then [g] scratch t = A s
    unsigned* t = cw + p.n_ldpc;
    const int tid = threadIdx.x, T = blockDim.x;
    const long long groups = (p.B + 31) / 32;
    for (long long gi = blockIdx.x; gi < groups; gi += gridDim.x) {
        const long long b0 = gi * 32;
        const int nb = (int)min((long long)32, p.B - b0);
        const float* u = p.u + (size_t)b0 * p.k;
        for (int i = tid; i < p.k_ldpc; i += T) {                                            // :637 (fillers = 0)
            unsigned w = 0;
            if (i < p.k)
                for (int b = 0; b < nb; ++b) w |= (unsigned)((int)u[(size_t)b * p.k + i] & 1) << b;
            cw[i] = w;
        }
        __syncthreads();
        for (int r = tid; r < p.g; r += T) {       // t = A s
            unsigned v = 0;
            for (int j = p.a_ptr[r]; j < p.a_ptr[r + 1]; ++j) v ^= cw[p.a_idx[j]];
            t[r] = v;
        }
        __syncthreads();
        for (int r = tid; r < p.g; r += T) {       // p_a = B^-1 t
            unsigned v = 0;
            for (int j = p.b_ptr[r]; j < p.b_ptr[r + 1]; ++j) v ^= t[p.b_idx[j]];
            cw[p.k_ldpc + r] = v;
        }
        __syncthreads();
        for (int r = tid; r < p.rows_needed; r += T) {   // p_b = C1 s + C2 p_a
            unsigned v = 0;
            for (int j = p.c1_ptr[r]; j < p.c1_ptr[r + 1]; ++j) v ^= cw[p.c1_idx[j]];
            for (int j = p.c2_ptr[r]; j < p.c2_ptr[r + 1]; ++j) v ^= cw[p.k_ldpc + p.c2_idx[j]];
            cw[p.k_ldpc + p.g + r] = v;
        }
        __syncthreads();
        float* c = p.c + (size_t)b0 * p.n;
        for (int j = tid; j < p.n; j += T) {
            const unsigned w = cw[p.tx_vn[j]];
            for (int b = 0; b < nb; ++b) c[(size_t)b * p.n + j] = (float)((w >> b) & 1u);
        }
        __syncthreads();
    }
}

bool check_csr(const int32_t* ptr, const int32_t* idx, int rows, int cols) {
    if (!ptr || ptr[0] != 0) return false;
    for (int r = 0; r < rows; ++r) if (ptr[r + 1] < ptr[r]) return false;
    for (int j = 0; j < ptr[rows]; ++j) if (!idx || idx[j] < 0 || idx[j] >= cols) return false;
    return true;
}

}  // namespace

extern "C" int sb_ldpc5g_encoder_create(sb_ldpc5g_encoder** out, int32_t k, int32_t n, int32_t k_ldpc, int32_t n_ldpc,
                                        int32_t g_rows, const int32_t* a_ptr, const int32_t* a_idx,
                                        const int32_t* binv_ptr, const int32_t* binv_idx, const int32_t* c1_ptr,
                                        const int32_t* c1_idx, const int32_t* c2_ptr, const int32_t* c2_idx,
                                        const int32_t* tx_vn) {
    SB_CHECK_ARG(out && k > 0 && n > 0 && k <= k_ldpc && k_ldpc + g_rows <= n_ldpc && g_rows > 0 && tx_vn,
                 "sb_ldpc5g_encoder_create: bad sizes");
    const int m_rest = n_ldpc - k_ldpc - g_rows;
    SB_CHECK_ARG(check_csr(a_ptr, a_idx, g_rows, k_ldpc) && check_csr(binv_ptr, binv_idx, g_rows, g_rows) &&
                     check_csr(c1_ptr, c1_idx, m_rest, k_ldpc) && check_csr(c2_ptr, c2_idx, m_rest, g_rows),
                 "sb_ldpc5g_encoder_create: malformed CSR input");
    auto* e = new sb_ldpc5g_encoder();
    e->k = k; e->n = n; e->k_ldpc = k_ldpc; e->n_ldpc = n_ldpc; e->g = g_rows; e->m_rest = m_rest;
    e->a_ptr.assign(a_ptr, a_ptr + g_rows + 1); e->a_idx.assign(a_idx, a_idx + a_ptr[g_rows]);
    e->b_ptr.assign(binv_ptr, binv_ptr + g_rows + 1); e->b_idx.assign(binv_idx, binv_idx + binv_ptr[g_rows]);
    e->c1_ptr.assign(c1_ptr, c1_ptr + m_rest + 1); e->c1_idx.assign(c1_idx, c1_idx + c1_ptr[m_rest]);
    e->c2_ptr.assign(c2_ptr, c2_ptr + m_rest + 1); e->c2_idx.assign(c2_idx, c2_idx + c2_ptr[m_rest]);
    e->tx_vn.assign(tx_vn, tx_vn + n);
    int max_vn = 0;
    for (int j = 0; j < n; ++j) {
        if (tx_vn[j] < 0 || tx_vn[j] >= n_ldpc) { delete e; sb_set_error("sb_ldpc5g_encoder_create: tx_vn out of range"); return SB_EINVAL; }
        if (tx_vn[j] > max_vn) max_vn = tx_vn[j];
    }
    e->rows_needed = std::max(0, std::min(m_rest, max_vn + 1 - k_ldpc - g_rows));
    e->tables.set(e->a_ptr, e->a_idx, e->b_ptr, e->b_idx, e->c1_ptr, e->c1_idx, e->c2_ptr, e->c2_idx, e->tx_vn);
    *out = e;
    return SB_OK;
}

extern "C" void sb_ldpc5g_encoder_destroy(sb_ldpc5g_encoder* e) { delete e; }

extern "C" int sb_ldpc5g_encode(const sb_ldpc5g_encoder* e, const float* d_u, int64_t batch, float* d_c, void* stream) {
    if (batch == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(e && d_u && d_c && batch >= 0, "sb_ldpc5g_encode: bad arguments");
    const DeviceTables::Copy* d = nullptr;
    int rc = e->tables.get(&d);
    if (rc) return rc;
    EncParams p{};
    p.k = e->k; p.n = e->n; p.k_ldpc = e->k_ldpc; p.n_ldpc = e->n_ldpc; p.g = e->g; p.rows_needed = e->rows_needed;
    p.a_ptr = d->at<int>(0); p.a_idx = d->at<int>(1); p.b_ptr = d->at<int>(2); p.b_idx = d->at<int>(3);
    p.c1_ptr = d->at<int>(4); p.c1_idx = d->at<int>(5); p.c2_ptr = d->at<int>(6); p.c2_idx = d->at<int>(7);
    p.tx_vn = d->at<int>(8);
    p.u = d_u; p.c = d_c; p.B = batch;
    size_t smem = 4 * ((size_t)e->n_ldpc + (size_t)e->g) + 16;
    SB_CUDA(cudaFuncSetAttribute(ldpc5g_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int occ = 0;
    SB_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, ldpc5g_encode_kernel, 512, smem));
    if (occ < 1) occ = 1;
    long long grid = std::min<long long>((batch + 31) / 32, (long long)d->num_sms * occ);
    ldpc5g_encode_kernel<<<(unsigned)grid, 512, smem, (cudaStream_t)stream>>>(p);
    SB_LAUNCH_CHECK();
    return SB_OK;
}
