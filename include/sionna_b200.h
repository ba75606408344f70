/* sionna_b200.h -- C-ABI of libsionna_b200.so (H100 / sm_90a kernels for the Sionna PHY hot path).
 *
 * The reference (NVlabs/sionna v1.2.1) has no FFI or plugin registry: its boundary is the Python
 * `Block.__call__ -> build(shapes) -> call()` protocol (/root/reference/src/sionna/phy/block.py:82-155)
 * and every op below is a chain of TensorFlow calls inside a `call()` method. Each entry point here
 * replaces the body of one such `call()`; the comment above it names the reference method
 * (file:line under /root/reference/src/sionna/phy/). The Python host layer (`sionna_b200/phy/...`)
 * keeps the reference's class names, constructor arguments, shapes and sign conventions and calls
 * these functions through ctypes on the current torch CUDA stream.
 *
 * Conventions
 *   - plain C types only: device pointers, sizes, a `void* stream` (cudaStream_t; NULL = default stream).
 *   - every function returns 0 on success or a negative SB_E* code; `sb_last_error()` returns a
 *     thread-local human-readable message for the last failure on the calling thread.
 *   - outputs and workspaces are allocated by the caller; no function synchronises the stream or
 *     allocates device memory, except that the first call using a handle on a device copies the
 *     handle's tables there (one copy per device, kept until `*_destroy` frees them all). That is the
 *     library's only device allocation and only synchronous copy.
 *   - all pointers named `d_*` are device pointers, `h_*` host pointers.
 *   - real tensors are fp32, complex tensors interleaved (re, im) fp32 ("single" precision).
 */
#ifndef SIONNA_B200_H
#define SIONNA_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SB_OK 0
#define SB_EINVAL (-1)   /* bad argument */
#define SB_ECUDA (-2)    /* CUDA runtime error (message holds cudaGetErrorString) */
#define SB_ENOMEM (-3)   /* workspace too small / allocation failed */
#define SB_EUNSUPPORTED (-4)

const char* sb_last_error(void);
/* Library / device sanity: returns SB_OK and fills sm count, compute capability major/minor, and the
 * opt-in shared memory per block of the CURRENT device. */
int sb_device_info(int* sm_count, int* cc_major, int* cc_minor, int* smem_optin_bytes);
int sb_version(void);
/* Number of kernels this library has launched from the calling thread since it was loaded (bench.py reports the
 * difference over its timed region as gpu_launches). */
int64_t sb_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * LDPC belief propagation
 * replaces LDPCBPDecoder.__init__ graph set-up   fec/ldpc/decoding.py:277-345
 *          LDPCBPDecoder.call / _bp_iter          fec/ldpc/decoding.py:416-637
 *          vn_update_sum / cn_update_*            fec/ldpc/decoding.py:681-1166
 *          LDPC5GDecoder.call rate recovery       fec/ldpc/decoding.py:1427-1536
 * ---------------------------------------------------------------------------------------------- */
typedef struct sb_ldpc_graph sb_ldpc_graph;

enum { SB_CN_BOXPLUS_PHI = 0, SB_CN_BOXPLUS = 1, SB_CN_MINSUM = 2, SB_CN_OFFSET_MINSUM = 3, SB_CN_IDENTITY = 4 };
enum { SB_VN_SUM = 0, SB_VN_IDENTITY = 1 };

/* Build a decoding graph.
 *   h_cn_of_edge, h_vn_of_edge [num_edges]: the reference's edge list in its VN order, i.e.
 *       `self._cn_idx`, `self._vn_idx` after `idx = np.argsort(vn_idx)` (decoding.py:282-288). Edge e of
 *       this list is row e of the `msg_v2c` decoder state ([num_edges, batch], decoding.py:575-579).
 *   h_in_map [num_vn] or NULL: where VN v takes its channel logit from: >= 0 index into the caller's
 *       input row (length n_in); -1 punctured (logit 0, decoding.py:1444-1458); -2 filler / shortened
 *       (logit -llr_max, decoding.py:1472-1475). NULL = identity (n_in must equal num_vn).
 *   h_out_vn [n_out] or NULL: VN whose estimate is written to output column j (systematic slice,
 *       filler / 2Z removal and output interleaver of decoding.py:1486-1536 folded into one gather).
 *       NULL = identity (n_out must equal num_vn).
 *   h_schedule [n_sub * n_active] or NULL: CN indices updated in each sub-iteration
 *       (`cn_schedule`, decoding.py:253-271, 464-497). NULL = flooding.
 * The graph's tables are copied to a device by the first decode there.
 */
int sb_ldpc_graph_create(sb_ldpc_graph** out, int32_t num_cn, int32_t num_vn, int32_t num_edges,
                         const int32_t* h_cn_of_edge, const int32_t* h_vn_of_edge,
                         const int32_t* h_in_map, int32_t n_in,
                         const int32_t* h_out_vn, int32_t n_out,
                         const int32_t* h_schedule, int32_t n_sub, int32_t n_active);
/* Same, but every per-node reduction runs in the REFERENCE's list order instead of ascending neighbour index:
 *   h_cn_view [num_edges]: `v2c_perm = np.argsort(cn_idx)` (decoding.py:329) - position j of the CN view holds edge
 *   h_cn_view[j]; a CN combines its edges in that order, a VN sums its edges in ascending edge number (the argsort
 *   order of decoding.py:286-288). fp32 sums depend on their order, and below the decoding threshold BP amplifies a
 *   last-bit difference into different hard decisions, so bit-exact agreement with the reference's arithmetic needs
 *   this order. Such graphs always run the generic kernel (sb_ldpc_graph_set_qc refuses them). */
int sb_ldpc_graph_create_ordered(sb_ldpc_graph** out, int32_t num_cn, int32_t num_vn, int32_t num_edges,
                                 const int32_t* h_cn_of_edge, const int32_t* h_vn_of_edge,
                                 const int32_t* h_in_map, int32_t n_in,
                                 const int32_t* h_out_vn, int32_t n_out,
                                 const int32_t* h_schedule, int32_t n_sub, int32_t n_active,
                                 const int32_t* h_cn_view);
void sb_ldpc_graph_destroy(sb_ldpc_graph* g);
/* Optional: declare the graph quasi-cyclic (lifted base graph, fec/ldpc/encoding.py:322-352): n_entries base entries
 * (h_base_row, h_base_col, h_shift) with lifting size Z, meaning CN r*Z+i is connected to VN c*Z+(i+s) mod Z. Entries
 * beyond the (possibly pruned) graph are ignored. The description is verified against the edge list given at
 * creation (SB_EINVAL on mismatch, handle unchanged); a new description drops the device copies of the previous one.
 * Qualifying decodes (flooding, "sum" VN rule, no input state, graph fits in shared memory) then run the index-free
 * QC kernel; results are identical either way. */
int sb_ldpc_graph_set_qc(sb_ldpc_graph* g, int32_t Z, int32_t n_entries, const int32_t* h_base_row,
                         const int32_t* h_base_col, const int32_t* h_shift);
int sb_ldpc_graph_is_qc(const sb_ldpc_graph* g);
/* 1 if boxplus-phi decodes of this QC graph skip the work that the punctured columns make exact in iterations 0 and 1:
 * every block row has a punctured column (no channel input) among its first two entries. */
int sb_ldpc_graph_qc_opening(const sb_ldpc_graph* g);
/* Test hook: phi(x) of decoding.py:1110-1120 evaluated on the device by the scalar and by the packed-fp32x2 code path
 * (n even); both must equal the CPU oracle bit for bit. */
int sb_debug_phi(const float* d_x, float* d_scalar, float* d_packed, int64_t n, void* stream);
/* 1 if one codeword's messages + channel LLRs fit in one SM's shared memory (the on-chip path),
 * 0 if the decoder will keep messages in an L2-resident global workspace. Judged for the current device once the graph
 * has decoded there, else for an H100. */
int sb_ldpc_graph_on_chip(const sb_ldpc_graph* g);
/* Bytes of device workspace `sb_ldpc_decode` needs for this graph (0 on the on-chip path), on the same device as
 * sb_ldpc_graph_on_chip. */
size_t sb_ldpc_workspace_bytes(const sb_ldpc_graph* g);
/* Test hook (no device needed): copies the host-side plan into caller arrays; any pointer may be NULL.
 * dims[10] = {C, N, E, Lc, Lv, n_in, n_out, n_sub, n_active, flooding}; cn_order[C], vn_order[N], slot_of_edge[E],
 * vn_slot[E], cn_off[Lc + 1], vn_off[Lv + 1]. */
int sb_ldpc_graph_export(const sb_ldpc_graph* g, int32_t* dims, int32_t* cn_order, int32_t* vn_order,
                         int32_t* slot_of_edge, int32_t* vn_slot, int32_t* cn_off, int32_t* vn_off);

/* Decode `batch` codewords.
 *   d_llr    [batch, n_in]   channel logits log p(1)/p(0) (decoding.py:159-164); clipped to +-llr_max and
 *                            negated internally (decoding.py:552-565).
 *   d_out    [batch, n_out]  hard_out != 0: 1.0f where the internal LLR <= 0 else 0.0f (decoding.py:622-624);
 *                            hard_out == 0: soft logits (decoding.py:626).
 *   d_state_in / d_state_out [batch, num_edges] or NULL: the `msg_v2c` decoder state, one row per
 *       codeword, columns in the reference's edge order (the host layer transposes to/from the
 *       reference's [num_edges, batch] layout, decoding.py:569-573, 633-637).
 *   offset: only for SB_CN_OFFSET_MINSUM (decoding.py:755).
 */
int sb_ldpc_decode(const sb_ldpc_graph* g, const float* d_llr, int64_t batch, int32_t num_iter,
                   int32_t cn_rule, int32_t vn_rule, float offset, float llr_max, int32_t hard_out,
                   const float* d_state_in, float* d_state_out, float* d_out,
                   void* d_workspace, size_t workspace_bytes, void* stream);

/* Same decode with opt-in EARLY TERMINATION (SURVEY.md section 8 row f4; the reference always runs num_iter iterations,
 * decoding.py:105-107): a codeword stops as soon as the hard decisions of all its variable nodes satisfy every parity check
 * (H x_hat = 0, evaluated on chip before each iteration), at most max_iter iterations.
 * d_num_iter [batch] (optional) receives the iterations run per codeword; the outputs of a codeword equal those of
 * sb_ldpc_decode with num_iter = d_num_iter[b] bit for bit. Only for graphs on the quasi-cyclic on-chip path (flooding,
 * "sum" VN rule); SB_EUNSUPPORTED otherwise. */
int sb_ldpc_decode_early(const sb_ldpc_graph* g, const float* d_llr, int64_t batch, int32_t max_iter, int32_t cn_rule,
                         float offset, float llr_max, int32_t hard_out, float* d_out, int32_t* d_num_iter, void* stream);

/* Unfused belief propagation (csrc/ldpc_bp_flat.cu): one call per half-iteration on [num_edges, batch] message tensors
 * in the reference's layouts, for decoders with Python callbacks (`v2c_callbacks` / `c2v_callbacks`, decoding.py:484-486,
 * 513-515) or user-supplied node updates. msg_v2c is in VN order (edge e of decoding.py:286-288), msg_c2v in CN-view
 * order (position j holds edge v2c_perm[j], decoding.py:329); node reductions run in those list orders.
 *   sb_ldpc_flat_init: d_x [batch, num_vn] channel logits after rate recovery and clipping (a 0-iteration sb_ldpc_decode)
 *       -> d_llr [num_vn, batch] = -x (decoding.py:565), d_v2c [num_edges, batch] = llr of the edge's VN (:571) or
 *       -d_state_in [num_edges, batch] (:573).
 *   sb_ldpc_flat_cn: CN update (rule as in sb_ldpc_decode) of the check nodes d_cn_list[num_nodes] (NULL: nodes
 *       0..num_nodes-1), reading d_v2c, writing those nodes' positions of d_c2v.
 *   sb_ldpc_flat_vn: VN update of every variable node: d_v2c, d_xhat [num_vn, batch] (clipped x_tot, internal sign).
 *   sb_ldpc_flat_out: d_out [batch, n_out] from d_xhat rows d_out_vn[n_out] (hard / soft as sb_ldpc_decode); optional
 *       d_state_out [num_edges, batch] = -d_v2c (:636). */
int sb_ldpc_flat_init(const float* d_x, const int32_t* d_vn_of_edge, const float* d_state_in, float* d_llr, float* d_v2c,
                      int64_t batch, int32_t num_vn, int32_t num_edges, void* stream);
int sb_ldpc_flat_cn(const float* d_v2c, float* d_c2v, const int32_t* d_cn_ptr, const int32_t* d_v2c_perm,
                    const int32_t* d_cn_list, int32_t num_nodes, int64_t batch, int32_t cn_rule, float offset,
                    float llr_max, void* stream);
int sb_ldpc_flat_vn(const float* d_c2v, const float* d_llr, const int32_t* d_vn_ptr, const int32_t* d_c2v_perm,
                    float* d_v2c, float* d_xhat, int32_t num_vn, int64_t batch, int32_t vn_rule, float llr_max,
                    void* stream);
int sb_ldpc_flat_out(const float* d_xhat, const int32_t* d_out_vn, float* d_out, const float* d_v2c, float* d_state_out,
                     int64_t batch, int32_t n_out, int32_t num_edges, int32_t hard_out, void* stream);

/* ------------------------------------------------------------------------------------------------
 * 5G NR LDPC encoder with rate matching
 * replaces LDPC5GEncoder.call / _encode_fast / _matmul_gather   fec/ldpc/encoding.py:599-668, 572-591, 559-570
 * ---------------------------------------------------------------------------------------------- */
typedef struct sb_ldpc5g_encoder sb_ldpc5g_encoder;
/* CSR (row pointer, ascending column index) of the binary Richardson-Urbanke sub-matrices of the lifted
 * parity-check matrix H = [[A B 0],[C1 C2 I]] (encoding.py:411-434): A [g_rows x k_ldpc], B^-1 [g_rows x g_rows],
 * C1 [(n_ldpc-k_ldpc-g_rows) x k_ldpc], C2 [same rows x g_rows]; h_tx_vn[n]: index into the n_ldpc-bit codeword
 * [s | p_a | p_b] transmitted at output position j (filler removal, 2Z puncturing, truncation, interleaver of
 * encoding.py:645-661 folded into one gather). The tables are copied to a device by the first encode there. */
int sb_ldpc5g_encoder_create(sb_ldpc5g_encoder** out, int32_t k, int32_t n, int32_t k_ldpc, int32_t n_ldpc,
                             int32_t g_rows, const int32_t* h_a_ptr, const int32_t* h_a_idx,
                             const int32_t* h_binv_ptr, const int32_t* h_binv_idx, const int32_t* h_c1_ptr,
                             const int32_t* h_c1_idx, const int32_t* h_c2_ptr, const int32_t* h_c2_idx,
                             const int32_t* h_tx_vn);
void sb_ldpc5g_encoder_destroy(sb_ldpc5g_encoder* e);
/* d_u [batch, k] information bits as 0.0f/1.0f -> d_c [batch, n] codeword bits as 0.0f/1.0f. */
int sb_ldpc5g_encode(const sb_ldpc5g_encoder* e, const float* d_u, int64_t batch, float* d_c, void* stream);

/* ------------------------------------------------------------------------------------------------
 * Sources, mapping, channel noise, metrics
 * ---------------------------------------------------------------------------------------------- */
/* BinarySource.call (mapping.py:1350-1352): n i.i.d. uniform bits as 0.0f/1.0f from Philox4x32-10(seed, offset). */
int sb_binary_source(float* d_out, int64_t n, uint64_t seed, uint64_t offset, void* stream);
/* out = mean + stddev * N(0,1) (GaussianPriorSource, fec/utils.py:71-114). */
int sb_normal(float* d_out, int64_t n, float mean, float stddev, uint64_t seed, uint64_t offset, void* stream);
/* config.tf_rng.uniform(shape, lo, hi) as used by TDL.__call__ (channel/tr38901/tdl.py:379-413): d_out[i] uniform in
 * [lo, hi), Philox4x32-10 stream (seed, offset). */
int sb_uniform(float* d_out, int64_t n, float lo, float hi, uint64_t seed, uint64_t offset, void* stream);
/* Mapper.call (mapping.py:497-519): d_bits [n_sym, m] 0/1 floats, MSB first -> d_out [n_sym] complex64 =
 * d_points[index]; d_idx_out (optional, int32 [n_sym]) receives the symbol indices (return_indices). */
int sb_qam_map(const float* d_bits, const float* d_points, int32_t m, float* d_out, int32_t* d_idx_out,
               int64_t n_sym, void* stream);
/* Demapper.call + SymbolLogits2LLRs.call (mapping.py:664-691, 927-967).
 *   d_y [n_sym] complex64; d_no: noise variance, element s uses d_no[s / no_inner] (no_inner = n_sym for a scalar,
 *   1 for per-symbol); d_points [2^m] complex64; method 0 = "app", 1 = "maxlog";
 *   d_prior (optional): prior logits, symbol s uses d_prior[(s / prior_inner) * m .. +m);
 *   d_llr [n_sym * m] logits log p(1)/p(0), or hard decisions (llr > 0) when hard_out != 0. */
int sb_demap(const float* d_y, const float* d_no, int64_t no_inner, const float* d_points, int32_t m, int32_t method,
             const float* d_prior, int64_t prior_inner, float* d_llr, int64_t n_sym, int32_t hard_out, void* stream);
/* Demapper.call for separable constellations (all square QAMs of mapping.py:104-117), no prior: the label's even bits
 * select the real level d_levels_re[t], the odd bits the imaginary level d_levels_im[t] (t = those m/2 bits, MSB
 * first). Same LLRs as sb_demap up to fp32 rounding with 2^(m/2) instead of 2^m exponents per dimension. */
int sb_demap_qam(const float* d_y, const float* d_no, int64_t no_inner, const float* d_levels_re,
                 const float* d_levels_im, int32_t m, int32_t method, float* d_llr, int64_t n_sym, int32_t hard_out,
                 void* stream);
/* SymbolDemapper.call (mapping.py:776-792): e_c = -|y - c|^2 / no + prior_c over the num_points points d_points
 * (complex, any constellation, 2 <= num_points <= 1024). Symbol s uses d_no[s / no_inner] and, if d_prior is given,
 * the prior logits d_prior[(s / prior_inner) * num_points ...]. d_out: log_softmax(e) [n_sym, num_points] (float), or
 * with hard_out = 1 the index of the first maximum [n_sym] (int32). Malformed arguments return SB_EINVAL before any
 * device access. */
int sb_symbol_demap(const float* d_y, const float* d_no, int64_t no_inner, const float* d_points, int32_t num_points,
                    const float* d_prior, int64_t prior_inner, void* d_out, int64_t n_sym, int32_t hard_out,
                    void* stream);
/* AWGN.call (channel/awgn.py:63-78, utils/misc.py:19-54): y = x + sqrt(no) * CN(0,1), complex64 [n];
 * element i uses d_no[i / no_inner]. */
int sb_awgn(const float* d_x, const float* d_no, int64_t no_inner, float* d_y, int64_t n, uint64_t seed,
            uint64_t offset, void* stream);
/* count_errors / count_block_errors (utils/metrics.py:94-144) fused: for b, b_hat [rows, k] (0/1 floats)
 * d_counters[0] += #(b != b_hat); [1] += #rows with any difference; [2] += rows*k; [3] += rows  (int64[4], device). */
int sb_count_errors(const float* d_b, const float* d_b_hat, int64_t rows, int32_t k, int64_t* d_counters, void* stream);

/* CRCEncoder.call (fec/crc.py:175-215): d_bits [rows, k] -> d_out [rows, k + crc_length] = [bits | CRC parity];
 * d_gen_rows[k]: row i of the reference's generator matrix (crc.py:126-156) packed MSB-first into 32 bits. */
int sb_crc_encode(const float* d_bits, const uint32_t* d_gen_rows, int32_t k, int32_t crc_length, float* d_out,
                  int64_t rows, void* stream);
/* CRCDecoder.call (fec/crc.py:300-327): d_x [rows, n] = [information bits | CRC parity]; d_gen_rows[n]: generator rows for
 * an n-bit input (as for sb_crc_encode with k = n); d_valid[rows] = 1 iff re-encoding the whole word yields an all-zero
 * parity; d_info [rows, n - crc_length] (optional) receives the information bits. */
int sb_crc_check(const float* d_x, const uint32_t* d_gen_rows, int32_t n, int32_t crc_length, float* d_info,
                 uint8_t* d_valid, int64_t rows, void* stream);
/* TB5GScrambler.call (fec/scrambling.py:442-468): d_x [rows, n], d_seq [seq_rows, n] Gold sequence(s) (nr/utils.py:16-76);
 * binary != 0: |x - c|, else x * (1 - 2c); row r uses sequence r mod seq_rows. */
int sb_scramble(const float* d_x, const float* d_seq, int32_t binary, float* d_out, int64_t rows, int32_t n,
                int32_t seq_rows, void* stream);

/* ------------------------------------------------------------------------------------------------
 * OFDM, resource grid, channel estimation, MIMO equalisation (complex64 = interleaved float pairs)
 * ---------------------------------------------------------------------------------------------- */
/* OFDMModulator.call (ofdm/modulator.py:97-124): d_x [rows, num_symbols, fft_size] frequency-domain grid (DC centred)
 * -> d_out [rows, out_len]; symbol l starts at d_out_off[l] and carries d_cp[l] cyclic-prefix samples:
 * ifftshift, ifft * sqrt(N) (signal/utils.py:206-249), CP = last cp samples prepended. Any fft_size <= 8192.
 * shift = 0 skips the (i)fftshift: with cp = 0 the two functions are then signal.ifft / signal.fft (signal/utils.py:161-249). */
int sb_ofdm_modulate(const float* d_x, float* d_out, int64_t rows, int32_t num_symbols, int32_t fft_size,
                     const int32_t* d_cp, const int32_t* d_out_off, int32_t out_len, int32_t shift, void* stream);
/* OFDMDemodulator.call (ofdm/demodulator.py:162-203): d_x [rows, in_len] time samples -> d_out [rows, num_symbols,
 * fft_size]: CP removal, fft / sqrt(N), phase compensation exp(-j 2 pi k l_min / N), fftshift. */
int sb_ofdm_demodulate(const float* d_x, float* d_out, int64_t rows, int32_t num_symbols, int32_t fft_size,
                       const int32_t* d_cp, const int32_t* d_in_off, int32_t in_len, int32_t l_min, int32_t shift,
                       void* stream);
/* out[b, r, j] = in[b, (in_rows == 1 ? 0 : r), idx[r, j]] (0 where idx < 0); words = 1 (fp32), 2 (complex64 / fp64)
 * or 4 (complex128): a bit copy. cols_out == 0 is a no-op and the pointers may then be null.
 * Replaces the tf.gather re-indexing of RemoveNulledSubcarriers (ofdm/resource_grid.py:551), ResourceGridDemapper
 * (:466-520) and NearestNeighborInterpolator (ofdm/channel_estimation.py:409-435). */
int sb_gather_rows(const float* d_in, const int32_t* d_idx, float* d_out, int64_t batch, int32_t rows, int32_t cols_out,
                   int32_t in_rows, int32_t cols_in, int32_t words, void* stream);
/* ResourceGridMapper.call (ofdm/resource_grid.py:394-412): d_x [batch, num_streams, num_data], d_pilots [num_streams,
 * num_pilots], d_map [num_streams, grid_size] (>= 0 data index, -1 empty, <= -2 pilot index -(v+2)) -> d_out
 * [batch, num_streams, grid_size]. d_x may be null when num_data == 0 (every RE a pilot or nulled), d_pilots when
 * num_pilots == 0. */
int sb_rg_map(const float* d_x, const float* d_pilots, const int32_t* d_map, float* d_out, int64_t batch,
              int32_t num_streams, int32_t grid_size, int32_t num_data, int32_t num_pilots, void* stream);
/* Pilot gather (ofdm/channel_estimation.py:138-150) + LSChannelEstimator.estimate_at_pilot_locations (:257-285):
 * d_y [batch, grid_size] (effective subcarriers, flattened), d_pilot_ind / d_pilots [num_streams, num_pilots], d_no
 * [batch / no_inner] -> d_h [batch, num_streams, num_pilots] = y / p, d_err = no / |p|^2 (both 0 where p == 0). */
int sb_ls_at_pilots(const float* d_y, const int32_t* d_pilot_ind, const float* d_pilots, const float* d_no,
                    int64_t no_inner, float* d_h, float* d_err, int64_t batch, int32_t num_streams, int32_t num_pilots,
                    int32_t grid_size, void* stream);
/* LinearInterpolator._interpolate (ofdm/channel_estimation.py:657-734) with the index tables of :522-655:
 * d_h [batch, num_streams, num_pilots] -> d_out [batch, num_streams, num_symbols, num_subcarriers]; words = 2:
 * complex64 values (channel estimates), words = 1: fp32 values (error variances). time_avg: bit 0 = average the pilot
 * symbols over time (lin_time_avg); bit 1 = floor fp32 results at 0 (the err_var clipping of channel_estimation.py:171). */
int sb_interp_lin(const float* d_h, const int32_t* d_fx0, const int32_t* d_fx1, const int32_t* d_fy0,
                  const int32_t* d_fy1, const int32_t* d_ty0, const int32_t* d_ty1, const int32_t* d_npil,
                  int32_t time_avg, float* d_out, int64_t batch, int32_t num_streams, int32_t num_symbols,
                  int32_t num_subcarriers, int32_t num_pilots, int32_t words, void* stream);
/* ApplyOFDMChannel.call (channel/apply_ofdm_channel.py:70-80): y[b, r, re] = sum_t h[b, r, t, re] x[b, t, re] + w,
 * r over rx antennas, t over tx antennas, w ~ CN(0, no) if add_noise. */
int sb_apply_ofdm_channel(const float* d_x, const float* d_h, const float* d_no, int64_t no_inner, float* d_y,
                          int64_t batch, int32_t num_rx_ant_total, int32_t num_tx_ant_total, int32_t num_re,
                          int32_t add_noise, uint64_t seed, uint64_t offset, void* stream);
/* ApplyTimeChannel.call (channel/apply_time_channel.py:115-137): d_x [batch, num_tx_ant_total, num_time_samples], d_h
 * [batch, num_rx_ant_total, num_tx_ant_total, num_time_samples + l_tot - 1, l_tot] -> d_y [batch, num_rx_ant_total,
 * num_time_samples + l_tot - 1] = time-variant FIR of x (+ CN(0, no) noise if add_noise). */
int sb_apply_time_channel(const float* d_x, const float* d_h, const float* d_no, int64_t no_inner, float* d_y,
                          int64_t batch, int32_t num_rx_ant_total, int32_t num_tx_ant_total, int32_t num_time_samples,
                          int32_t l_tot, int32_t add_noise, uint64_t seed, uint64_t offset, void* stream);
/* TDL.__call__ (channel/tr38901/tdl.py:372-456): sum-of-sinusoids tap gains. d_doppler [batch] (radian Doppler),
 * d_theta [batch, paths, sinusoids], d_phi [batch, ant_pairs, paths, sinusoids], d_phi0 [batch] or NULL (NLoS models),
 * d_powers [paths] -> d_a [batch, ant_pairs, paths, time_steps] complex; ant_pairs = num_rx_ant * num_tx_ant, rx major. */
int sb_tdl_sos(const float* d_doppler, const float* d_theta, const float* d_phi, const float* d_phi0,
               const float* d_powers, float los_power, float los_aoa, float* d_a, int64_t batch, int32_t num_ant_pairs,
               int32_t num_paths, int32_t num_sinusoids, int32_t num_time_steps, float sampling_frequency, void* stream);
/* CDL.__call__ (channel/tr38901/cdl.py:258-332 and channel_coefficients.py:459-1030, no sub-clustering): cluster
 * coefficients of TR 38.901 (7.5-22), (7.5-28)..(7.5-30) summed over 20 rays. Draws: d_speed, d_v_phi, d_v_theta
 * [batch]; d_coupling [batch, 4, clusters, 20] normals whose per-cluster argsort permutes the arrival azimuth, departure
 * azimuth, arrival zenith and departure zenith of the rays (in that order); d_phases [batch, clusters, 20, 4] initial
 * phases. Per-instance tables over the rows c * 400 + zenith_index * 20 + azimuth_index (c in table order) plus one LoS
 * row at clusters * 400: d_rx_dir [rows, 3] arrival unit vectors, d_rx_field / d_tx_field [rows, 4] GCS fields (pol 1
 * theta, phi, pol 2 theta, phi), d_rx_phase [rows, num_rx_ant] / d_tx_phase [rows, num_tx_ant] complex antenna phases;
 * d_rx_pol / d_tx_pol [ant] polarization index 0 / 1; d_cluster_scale [clusters] = sqrt(P_c / 20) (times sqrt(1 / (K +
 * 1)) for LoS models); d_order [clusters]: table cluster of output cluster o (ascending delay); d_los_field [4] LoS gains
 * (rx pol major, times sqrt(K / (K + 1))) or NULL for NLoS models; xpr_scale = sqrt(1 / XPR); wavenumber = 2 pi / lambda.
 * -> d_a [batch, num_rx_ant, num_tx_ant, clusters, time_steps] complex, written once, no atomics. clusters <= 24. */
int sb_cdl_coefficients(const float* d_speed, const float* d_v_phi, const float* d_v_theta, const float* d_coupling,
                        const float* d_phases, const float* d_rx_dir, const float* d_rx_field, const float* d_rx_phase,
                        const int32_t* d_rx_pol, const float* d_tx_field, const float* d_tx_phase,
                        const int32_t* d_tx_pol, const float* d_cluster_scale, const int32_t* d_order,
                        const float* d_los_field, float xpr_scale, float wavenumber, float* d_a, int64_t batch,
                        int32_t num_clusters, int32_t num_rx_ant, int32_t num_tx_ant, int32_t num_time_steps,
                        float sampling_frequency, void* stream);
/* CIR -> channel conversion without eager tensor expressions (channel/utils.py:180-350), csrc/channel.cu.
 * sb_phase_table: d_e [n_tab, paths, cols] complex; mode 0: exp(-j 2 pi x_j tau[tab, p]) (x = subcarrier frequencies,
 *   cir_to_ofdm_channel :232-244); mode 1: sinc(x_j - tau[tab, p] * scale) (x = tap lags l, scale = bandwidth,
 *   cir_to_time_channel :318-338). n_tab = 1 when all links share the delays (every TDL model), else one table per link.
 * sb_cir_gram: d_g [n_tab, paths, paths] complex double = sum_j e[p, j] conj(e[q, j]), accumulated in double.
 * sb_cir_link_scale: normalisation of :246-251 / :341-348 per link (batch, rx, tx) from the taps d_a [batch, rx, rx_ant,
 *   tx, tx_ant, paths, time] and the Gram matrix (g_link_stride = 0: shared, else paths*paths): d_scale [batch*rx*tx] =
 *   1 / sqrt(link energy / (rx_ant * tx_ant * time * denom)), 0 only for a link of zero energy; denom = cols (OFDM: mean over
 *   subcarriers) or 1 (time channel: sum over taps). The quadratic form is evaluated in double; paths <= 96 as in sb_cir_apply.
 * sb_cir_apply: d_h [batch, rx, rx_ant, tx, tx_ant, time, cols] = scale[link] * sum_p a[..., p, t] e[tab, p, col]
 *   (d_scale may be NULL; e_link_stride = 0: shared table, else paths*cols). */
int sb_phase_table(const float* d_tau, const float* d_x, float scale, int32_t mode, float* d_e, int64_t n_tab,
                   int32_t num_paths, int32_t num_cols, void* stream);
int sb_cir_gram(const float* d_e, double* d_g, int64_t n_tab, int32_t num_paths, int32_t num_cols, void* stream);
int sb_cir_link_scale(const float* d_a, const double* d_g, int64_t g_link_stride, float* d_scale, int64_t batch,
                      int32_t num_rx, int32_t num_rx_ant, int32_t num_tx, int32_t num_tx_ant, int32_t num_paths,
                      int32_t num_time_steps, float denom, void* stream);
int sb_cir_apply(const float* d_a, const float* d_e, int64_t e_link_stride, const float* d_scale, float* d_h,
                 int64_t batch, int32_t num_rx, int32_t num_rx_ant, int32_t num_tx, int32_t num_tx_ant,
                 int32_t num_paths, int32_t num_time_steps, int32_t num_cols, void* stream);
/* TDL spatial correlation (channel/tr38901/tdl.py:466-490): d_in / d_out [batch, n, cols] complex (n = rx_ant * tx_ant
 * antenna pairs, rx antenna major; cols = paths * time steps), d_l [n, n] lower-triangular Cholesky factor of the
 * correlation matrix (for separate rx / tx matrices: kron(L_rx, conj(L_tx))): out[b, :, c] = L in[b, :, c]. */
int sb_spatial_corr(const float* d_in, const float* d_l, float* d_out, int64_t batch, int32_t n, int64_t cols,
                    void* stream);
/* Flat-fading MIMO channel (csrc/flat_fading.cu), complex64, M = num_rx_ant, K = num_tx_ant, num channel uses:
 * GenerateFlatFadingChannel / ApplyFlatFadingChannel / FlatFadingChannel and the KroneckerModel / PerColumnModel
 * products (channel/flat_fading_channel.py:11-246, channel/spatial_correlation.py:42-195) in one launch.
 *   h0: d_h_in [*, M, K] (h_in_stride 0: one matrix for every use, 1: one per use) or, d_h_in NULL, drawn from
 *       (seed_h, offset_h) with sb_awgn's counter convention over the flat [num, M, K] index (element i: Philox block
 *       i / 2, words (x, y) for even i, (z, w) for odd i), so the draw equals complex_normal([num, M, K]) bit for bit.
 *   h = L_rx h0 L_tx^H (tx factor applied first). d_l_tx [*, K, K] and d_l_rx [*, M, M] are lower-triangular factors
 *       (sb_chol_lower), either may be NULL, each with a stride of 0 (shared) or 1 (one set per use). per_column = 1
 *       takes d_l_rx as [*, K, M, M] and column k of h as L_rx[k] h0[:, k] (no tx factor).
 *   d_h_out [num, M, K]: h, written only if not NULL. d_x [*, K] (x_stride 0 or 1) and d_y [num, M]: y = h x, summed
 *       over k in order. d_no (needs d_x; NULL: no noise): y[i] += sqrt(d_no[i / no_inner]) n_i with n the unit
 *       complex noise of sb_awgn(seed_n, offset_n) over the flat [num, M] index, bit for bit.
 * No intermediate goes through global memory. Limits: M <= 128 with an rx factor, K <= 128 with a tx factor and
 * M K <= 16384 with either; without factors any M and K. Beyond them SB_EUNSUPPORTED with a message; malformed
 * arguments (strides outside {0, 1}, per_column without d_l_rx or with d_l_tx, neither d_h_out nor d_x, d_x without
 * d_y, d_no without d_x) return SB_EINVAL. All checks run before any device access; num = 0 then returns SB_OK. */
int sb_flat_fading(const float* d_h_in, int64_t h_in_stride, uint64_t seed_h, uint64_t offset_h, const float* d_l_tx,
                   int64_t l_tx_stride, const float* d_l_rx, int64_t l_rx_stride, int32_t per_column, float* d_h_out,
                   const float* d_x, int64_t x_stride, const float* d_no, int64_t no_inner, uint64_t seed_n,
                   uint64_t offset_n, float* d_y, int64_t num, int32_t num_rx_ant, int32_t num_tx_ant, void* stream);
/* Lower Cholesky factors L (L L^H = R) of count n x n complex matrices, d_r and d_l [count, n, n] (the strictly upper
 * triangle of L is 0), in fp32 by sb_dense::chol_lower, one thread per matrix in shared-memory scratch (n = 128: one
 * thread per CTA). Only the lower triangle of R is read. A non-positive pivot makes the rest of that matrix's factor
 * NaN; other matrices are unaffected and nothing synchronises. n <= 128 (SB_EUNSUPPORTED beyond). */
int sb_chol_lower(const float* d_r, float* d_l, int64_t count, int32_t n, void* stream);
/* PUSCHPrecoder.call (nr/pusch_precoder.py:75-95): d_x [batch, num_tx, num_layers, num_re] complex, d_w [num_tx,
 * num_ports, num_layers] complex -> d_y [batch, num_tx, num_ports, num_re], y = W x per resource element. */
int sb_pusch_precode(const float* d_x, const float* d_w, float* d_y, int64_t batch, int32_t num_tx, int32_t num_layers,
                     int32_t num_ports, int64_t num_re, void* stream);
/* PUSCHLSChannelEstimator.estimate_at_pilot_locations (nr/pusch_channel_estimation.py:117-169), the part after the LS
 * division (sb_ls_at_pilots): in-place CDM de-spreading of d_h [rows, num_pilots] complex (pilots ordered DMRS symbol
 * major): average over the two symbols of a double-symbol DMRS, then sum / 2 over groups of group_size = 2 *
 * num_cdm_groups_without_data adjacent pilots, written back to the group's non-zero entries; d_err_var [rows,
 * num_pilots] is scaled by 1/2 (and by another 1/2 for double-symbol DMRS). */
int sb_pusch_ls_combine(float* d_h, float* d_err_var, int64_t rows, int32_t num_pilots, int32_t pilots_per_dmrs_symbol,
                        int32_t dmrs_length, int32_t group_size, void* stream);
/* lmmse_equalizer (mimo/equalization.py:101-233, whiten_interference=True): d_y [num, M], d_h [num, M, K], d_s [num, M, M]
 * -> d_x_hat [num, K] complex, d_no_eff [num, K] real. 1 <= K <= 16, K <= M, and the per-vector scratch
 * 8 (M^2 + 2 M K + M + K^2) bytes must fit 200 KB: M <= 158 for K = 1, M <= 143 for K = 16. Shapes whose scratch
 * leaves room for fewer than 32 vectors per CTA run with 16 ... 1 threads per CTA (correct, not tuned for speed);
 * larger ones return SB_EUNSUPPORTED. */
int sb_lmmse_equalize(const float* d_y, const float* d_h, const float* d_s, float* d_x_hat, float* d_no_eff, int64_t num,
                      int32_t M, int32_t K, void* stream);
/* The reference's small dense helpers as callable kernels (complex64, one thread per matrix):
 *   mode 0  inv_cholesky(s)          utils/linalg.py:8-32         d_s [num, M, M] -> d_out0 = L^-1 [num, M, M]
 *   mode 1  whiten_channel(y, h, s)  mimo/utils.py:292-357        -> d_out0 = L^-1 y [num, M], d_out1 = L^-1 H [num, M, K]
 *   mode 2  lmmse_matrix(h, s)       mimo/equalization.py:11-99   -> d_out0 = G [num, K, M]; d_s == NULL: (H^H H + I)^-1 H^H
 *   mode 3  lmmse_equalizer(y, h, s, whiten_interference=False) :183-233 -> d_out0 = x_hat [num, K], d_out1 = no_eff (fp32)
 *   mode 4  zf_equalizer(y, h, s)    mimo/equalization.py:235-343 -> d_out0 = x_hat [num, K], d_out1 = no_eff [num, K] (fp32)
 *   mode 5  mf_equalizer(y, h, s)    mimo/equalization.py:345-466 -> d_out0 = x_hat [num, K], d_out1 = no_eff [num, K] (fp32)
 *   mode 6  matrix_pinv(h)           utils/linalg.py              -> d_out0 = (H^H H)^-1 H^H [num, K, M]
 * Modes 2 ... 6 read the lower triangle of S only. Modes 1, 3, 4, 5 need d_y, d_s and d_out1; malformed arguments return
 * SB_EINVAL. 1 <= K <= M (mode 0: K = M). The per-matrix scratch 8 (M^2 + 2 M K) bytes must fit the device's opt-in shared memory per
 * block (227 KB on H100: inv_cholesky up to M = 98, M <= 155 for K = 16); below 32 matrices per CTA the kernel runs
 * with 16 ... 1 threads per CTA (correct, not tuned for speed); larger shapes return SB_EUNSUPPORTED. */
int sb_mimo_linalg(int32_t mode, const float* d_y, const float* d_h, const float* d_s, float* d_out0, void* d_out1,
                   int64_t num, int32_t M, int32_t K, void* stream);
/* OFDMEqualizer.call with the LMMSE equaliser fused in (ofdm/equalization.py:109-275 + mimo/equalization.py:101-233):
 * d_y [batch, num_rx, num_rx_ant, num_symbols, num_subcarriers] (effective subcarriers), d_h_hat [batch, num_rx,
 * num_rx_ant, num_tx_streams, num_symbols, num_subcarriers], d_err_var addressed with h_ev_stride[6] (elements; 0 =
 * broadcast) over (batch, rx, ant, tx_stream, symbol, subcarrier), d_no with h_no_stride[3] over (batch, rx, ant);
 * d_desired [num_rx, streams_per_rx] / d_undesired [num_rx, interferers_per_rx]: tx-stream indices per receiver
 * (mimo/stream_management.py:200-246); d_out_stream [num_rx, streams_per_rx]: output stream row after the stream_ind
 * re-ordering; d_data_pos [num_tx_streams, num_symbols*num_subcarriers]: index among that stream's data symbols or -1.
 * Outputs d_x_hat / d_no_eff [batch, num_tx_streams, num_data]. 1 <= streams_per_rx <= min(16, num_rx_ant). Receivers
 * without interfering streams and streams_per_rx <= 4 run a register kernel with no limit on num_rx_ant; the others keep
 * 8 (M^2 + 2 M K + M + K^2) bytes of scratch per resource element (M = num_rx_ant, K = streams_per_rx) in shared memory,
 * which must fit 200 KB (M <= 143 for K = 16), with 16 ... 1 threads per CTA when fewer than 32 fit. */
int sb_ofdm_lmmse(const float* d_y, const float* d_h_hat, const float* d_err_var, const int64_t* h_ev_stride,
                  const float* d_no, const int64_t* h_no_stride, const int32_t* d_desired, const int32_t* d_undesired,
                  const int32_t* d_out_stream, const int32_t* d_data_pos, float* d_x_hat, float* d_no_eff, int64_t batch,
                  int32_t num_rx, int32_t num_rx_ant, int32_t num_tx_streams, int32_t num_symbols,
                  int32_t num_subcarriers, int32_t streams_per_rx, int32_t interferers_per_rx, int32_t num_data,
                  void* stream);
/* LMMSEEqualizer (whitened or not), ZFEqualizer and MFEqualizer (ofdm/equalization.py:277-462, mimo/equalization.py:
 * 101-466): sb_ofdm_lmmse's arguments, layouts and shared-memory limit with the equaliser chosen by `equalizer`:
 * 0 LMMSE (sb_ofdm_lmmse), 1 LMMSE with whiten_interference=False, 2 ZF, 3 MF. Receivers without interfering streams
 * and streams_per_rx <= 4 (equalizer 1: and num_rx_ant >= streams_per_rx + 2) run a register kernel (no limit on
 * num_rx_ant); all other cases run the shared-memory kernel and its scratch limit.
 * A bad equalizer, negative or zero sizes (batch may be 0) or, with batch > 0, a missing pointer return SB_EINVAL;
 * streams_per_rx outside 1 ... min(16, num_rx_ant) and scratch beyond 200 KB return SB_EUNSUPPORTED with a message.
 * All checks run before any device access. */
int sb_ofdm_equalize(int32_t equalizer, const float* d_y, const float* d_h_hat, const float* d_err_var,
                     const int64_t* h_ev_stride, const float* d_no, const int64_t* h_no_stride, const int32_t* d_desired,
                     const int32_t* d_undesired, const int32_t* d_out_stream, const int32_t* d_data_pos, float* d_x_hat,
                     float* d_no_eff, int64_t batch, int32_t num_rx, int32_t num_rx_ant, int32_t num_tx_streams,
                     int32_t num_symbols, int32_t num_subcarriers, int32_t streams_per_rx, int32_t interferers_per_rx,
                     int32_t num_data, void* stream);

/* MaximumLikelihoodDetector.call (mimo/detection.py:473-537, whiten_channel mimo/utils.py:292-357, SymbolLogits2LLRs.call
 * mapping.py:927-967), complex64: d_y [num, M], d_h [num, M, K], d_s [num, M, M], optional d_prior [num, K, num_points]
 * symbol logits (bit priors are converted by the caller, LLRs2SymbolLogits mapping.py:1045-1059), d_points [num_points]
 * complex (any constellation). method 0 app (logsumexp) / 1 maxlog (max); output 0 bit / 1 symbol; hard_out 0 / 1.
 * d_out: bit LLRs or hard bits [num, K, log2 num_points] (float), symbol logits [num, K, num_points] (float) or hard
 * symbol indices [num, K] (int32, first maximum). d_workspace: device memory of at least
 * sb_ml_workspace_bytes(num, K) bytes, 8-byte aligned (per-problem whitened triangular records and output positions;
 * SB_ENOMEM if it is missing or smaller).
 * Malformed arguments return SB_EINVAL; 1 <= K <= 8, num_points a power of two in 2 ... 1024, num_points^K <= 65536
 * and any M >= 1 (M < K allowed) whose whitening scratch 8 (M^2 + M K + M) bytes per problem fits 200 KB are
 * supported, larger configurations return SB_EUNSUPPORTED with a message. */
int sb_mimo_ml(const float* d_y, const float* d_h, const float* d_s, const float* d_prior, const float* d_points,
               void* d_out, void* d_workspace, size_t workspace_bytes, int64_t num, int32_t M, int32_t K,
               int32_t num_points, int32_t method, int32_t output, int32_t hard_out, void* stream);
/* Workspace bytes sb_mimo_ml / sb_ofdm_ml need for num_problems problems of K streams: 8 (K^2 + 2 K + 1) per problem
 * (sb_ofdm_ml: num_problems = batch * num_rx * num_symbols * num_subcarriers); 0 for K outside 1 ... 8. */
size_t sb_ml_workspace_bytes(int64_t num_problems, int32_t K);
/* OFDM MaximumLikelihoodDetector / MaximumLikelihoodDetectorWithPrior (ofdm/detection.py:448-738): sb_ofdm_lmmse's
 * inputs, strides, tables and broadcast rules (S = H_u H_u^H + diag(no) + diag(sum err_var) assembled per resource
 * element), then sb_mimo_ml's detector with K = streams_per_rx. d_prior (optional): symbol logits in the output layout
 * [batch, num_tx_streams, num_data, num_points]. d_out: [batch, num_tx_streams, num_data * log2 num_points] (bits),
 * [batch, num_tx_streams, num_data, num_points] (logits) or [batch, num_tx_streams, num_data] (int32 indices).
 * Workspace and limits as sb_mimo_ml with M = num_rx_ant. */
int sb_ofdm_ml(const float* d_y, const float* d_h_hat, const float* d_err_var, const int64_t* h_ev_stride,
               const float* d_no, const int64_t* h_no_stride, const int32_t* d_desired, const int32_t* d_undesired,
               const int32_t* d_out_stream, const int32_t* d_data_pos, const float* d_prior, const float* d_points,
               void* d_out, void* d_workspace, size_t workspace_bytes, int64_t batch, int32_t num_rx,
               int32_t num_rx_ant, int32_t num_tx_streams, int32_t num_symbols, int32_t num_subcarriers,
               int32_t streams_per_rx, int32_t interferers_per_rx, int32_t num_data, int32_t num_points, int32_t method,
               int32_t output, int32_t hard_out, void* stream);

/* KBestDetector.call (mimo/detection.py:539-1037, complex2real_channel mimo/utils.py:194-242, List2LLRSimple
 * mimo/utils.py:420-577, PAM2QAM mapping.py:1234-1320), complex64: d_y [num, M], d_h [num, M, K], d_s [num, M, M].
 * num_points = |C| of the transmitted constellation (m = log2 num_points output bits per symbol). real_rep 0: d_points
 * [num_points] complex (any constellation); real_rep 1 (QAM, m even): the real-valued representation, d_points
 * [2^(m/2)] real PAM levels by label. k: paths kept per layer (at most num_points^K are ever kept). output 0 bit /
 * 1 symbol (symbol needs hard_out = 1); d_out: LLRs or hard bits [num, K, m] (float) or symbol indices [num, K]
 * (int32). LLRs are clipped to +-llr_clip (INFINITY allowed). d_workspace: device memory of at least
 * sb_kbest_workspace_bytes(num, K, real_rep) bytes, 8-byte aligned (SB_ENOMEM if it is missing or smaller).
 * Malformed arguments return SB_EINVAL (K < 1, M < K, k < 1, num_points not a power of two >= 2, flags outside {0, 1},
 * real_rep with odd m, soft symbol output, llr_clip < 0 or NaN). Limits, counted in the detection domain (S = K or 2 K
 * layers of num_points or 2^(m/2) points): S <= 16, k <= 256, points <= 256, k * points <= 16384, and a whitening
 * scratch of 8 (M^2 + M K + M) (+ 8 (4 M K + 2 M) with real_rep) bytes per problem within 200 KB; beyond them
 * SB_EUNSUPPORTED with a message. */
int sb_mimo_kbest(const float* d_y, const float* d_h, const float* d_s, const float* d_points, void* d_out,
                  void* d_workspace, size_t workspace_bytes, int64_t num, int32_t M, int32_t K, int32_t num_points,
                  int32_t k, int32_t real_rep, int32_t output, int32_t hard_out, float llr_clip, void* stream);
/* Workspace bytes sb_mimo_kbest / sb_ofdm_kbest need for num_problems problems of K streams: with S = K << real_rep,
 * 8 (S^2 + S + 1) + 8 K + 4 S per problem (sb_ofdm_kbest: num_problems = batch * num_rx * num_symbols *
 * num_subcarriers); 0 for K << real_rep outside 1 ... 16 or real_rep outside {0, 1}. */
size_t sb_kbest_workspace_bytes(int64_t num_problems, int32_t K, int32_t real_rep);
/* K-Best detection per OFDM resource element: sb_ofdm_ml's inputs, strides, tables and output layouts (without priors
 * and soft symbols), then sb_mimo_kbest's detector with M = num_rx_ant and K = streams_per_rx. */
int sb_ofdm_kbest(const float* d_y, const float* d_h_hat, const float* d_err_var, const int64_t* h_ev_stride,
                  const float* d_no, const int64_t* h_no_stride, const int32_t* d_desired, const int32_t* d_undesired,
                  const int32_t* d_out_stream, const int32_t* d_data_pos, const float* d_points, void* d_out,
                  void* d_workspace, size_t workspace_bytes, int64_t batch, int32_t num_rx, int32_t num_rx_ant,
                  int32_t num_tx_streams, int32_t num_symbols, int32_t num_subcarriers, int32_t streams_per_rx,
                  int32_t interferers_per_rx, int32_t num_data, int32_t num_points, int32_t k, int32_t real_rep,
                  int32_t output, int32_t hard_out, float llr_clip, void* stream);

/* EPDetector.call (mimo/detection.py:1039-1312, complex2real_channel mimo/utils.py:194-242, SymbolLogits2LLRs
 * mapping.py:927-967, PAM2QAM mapping.py:1234-1316), complex64: d_y [num, M], d_h [num, M, K], d_s [num, M, M].
 * num_points = |C| of the transmitted QAM (m = log2 num_points, even); d_levels [2^(m/2)]: the real PAM levels by
 * label, scaled to energy 1/2. l >= 1 iterations, damping 0 <= beta <= 1. output 0 bit / 1 symbol; d_out: LLRs or hard
 * bits [num, K, m] (float; real PAM on the even bit positions), QAM logits [num, K, num_points] (float) or QAM indices
 * [num, K] (int32). One launch, no workspace. Malformed arguments return SB_EINVAL (M < 1, K < 1, num_points not a
 * power of two >= 2 or with odd m, l < 1, beta outside [0, 1] or NaN, flags outside {0, 1}). Limits: K <= 16,
 * num_points <= 256, and 8 (M^2 + M K + M + K^2 + K) + 4 (4 K^2 + 14 K) bytes of shared-memory scratch per problem
 * within 200 KB; beyond them SB_EUNSUPPORTED with a message. M < K is accepted. */
int sb_mimo_ep(const float* d_y, const float* d_h, const float* d_s, const float* d_levels, void* d_out, int64_t num,
               int32_t M, int32_t K, int32_t num_points, int32_t l, float beta, int32_t output, int32_t hard_out,
               void* stream);
/* EP per OFDM resource element: sb_ofdm_ml's inputs, strides, tables and output layouts (without priors), then
 * sb_mimo_ep's detector with M = num_rx_ant and K = streams_per_rx. */
int sb_ofdm_ep(const float* d_y, const float* d_h_hat, const float* d_err_var, const int64_t* h_ev_stride,
               const float* d_no, const int64_t* h_no_stride, const int32_t* d_desired, const int32_t* d_undesired,
               const int32_t* d_out_stream, const int32_t* d_data_pos, const float* d_levels, void* d_out,
               int64_t batch, int32_t num_rx, int32_t num_rx_ant, int32_t num_tx_streams, int32_t num_symbols,
               int32_t num_subcarriers, int32_t streams_per_rx, int32_t interferers_per_rx, int32_t num_data,
               int32_t num_points, int32_t l, float beta, int32_t output, int32_t hard_out, void* stream);

/* MMSEPICDetector.call (mimo/detection.py:1314-1643) with output "bit", complex64: d_y [num, M], d_h [num, M, K],
 * d_s [num, M, M], d_prior [num, K, m] a-priori bit LLRs (NULL: zero prior), d_points [num_points] complex (any
 * constellation, m = log2 num_points). num_iter >= 1 self-iterations, method 0 app / 1 maxlog demapping. d_out
 * [num, K, m]: extrinsic LLRs llr_d - llr_a of the last iteration, or their hard decisions (hard_out = 1). Symbol priors
 * and outputs are converted by the caller (SymbolLogits2LLRs, LLRs2SymbolLogits). One launch, no workspace. Malformed
 * arguments return SB_EINVAL (M < 1, K < 1, num_points not a power of two >= 2, num_iter < 1, method or hard_out outside
 * {0, 1}). Limits: K <= 16, num_points <= 1024, and 8 (M^2 + M K + M + 2 K^2 + 6 K) + 4 K m bytes of shared-memory
 * scratch per problem within 200 KB - 8 num_points; beyond them SB_EUNSUPPORTED with a message. M < K is accepted. */
int sb_mimo_mmse_pic(const float* d_y, const float* d_h, const float* d_s, const float* d_prior, const float* d_points,
                     float* d_out, int64_t num, int32_t M, int32_t K, int32_t num_points, int32_t num_iter,
                     int32_t method, int32_t hard_out, void* stream);
/* MMSE-PIC per OFDM resource element: sb_ofdm_ml's inputs, strides and tables, then sb_mimo_mmse_pic's detector with
 * M = num_rx_ant and K = streams_per_rx. d_prior (optional) and d_out: bit LLRs in the output layout
 * [batch, num_tx_streams, num_data * m]; a stream without data at an element has a zero prior there. */
int sb_ofdm_mmse_pic(const float* d_y, const float* d_h_hat, const float* d_err_var, const int64_t* h_ev_stride,
                     const float* d_no, const int64_t* h_no_stride, const int32_t* d_desired,
                     const int32_t* d_undesired, const int32_t* d_out_stream, const int32_t* d_data_pos,
                     const float* d_prior, const float* d_points, float* d_out, int64_t batch, int32_t num_rx,
                     int32_t num_rx_ant, int32_t num_tx_streams, int32_t num_symbols, int32_t num_subcarriers,
                     int32_t streams_per_rx, int32_t interferers_per_rx, int32_t num_data, int32_t num_points,
                     int32_t num_iter, int32_t method, int32_t hard_out, void* stream);

/* Transmit precoding (csrc/precoding.cu), complex64. kind 0: RZF, G = V D with V = H^H (H H^H + alpha I)^-1 computed
 * as the adjoint of cholesky_solve(chol(H H^H + alpha I), H); kind 1: CBF, V = H^H; kind 2 (OFDM only): identity. D
 * scales every column of V to unit norm, a zero column stays zero (mimo/precoding.py:12-245). alpha = 0 with K > M
 * gives a singular Gram matrix; the outputs are then not finite. Limits: K <= 16 streams, M <= 1024 transmit
 * antennas; beyond them SB_EUNSUPPORTED with a message. Malformed arguments return SB_EINVAL; all checks run before any
 * device access.
 * Dense problems: d_h [num, K, M]; d_alpha (RZF only; NULL: 0) one value (alpha_stride 0) or one per problem (1);
 * d_x [num, K] (needed for d_gx). Outputs, either may be NULL but not both: d_g [num, M, K], d_gx = G x [num, M]. */
int sb_mimo_precode(const float* d_h, const float* d_alpha, int64_t alpha_stride, const float* d_x, float* d_g,
                    float* d_gx, int64_t num, int32_t K, int32_t M, int32_t kind, void* stream);
/* RZFPrecoder / RZFPrecodedChannel / CBFPrecodedChannel / EyePrecodedChannel (ofdm/precoding.py:15-566) per resource
 * element, K = num_streams_per_tx, M = num_tx_ant. d_h_hat [batch, num_rx, num_rx_ant, num_tx, M, S, fft_size] is the
 * channel the precoder is computed from: stream k of transmitter j uses row k % num_rx_ant of the channel to receiver
 * d_precoding_ind[j, k / num_rx_ant] (d_precoding_ind [num_tx, K / num_rx_ant], StreamManagement.precoding_ind).
 * K must equal num_rx_per_tx * num_rx_ant (SB_EINVAL otherwise). d_alpha (RZF; NULL: 0) with element strides
 * h_alpha_stride[4] over (batch, tx, symbol, subcarrier), d_tx_power (NULL: 1) with h_tx_power_stride[5] over
 * (batch, tx, stream, symbol, subcarrier); a stride of 0 broadcasts. sqrt(tx_power) scales column k of G.
 * Outputs, either may be NULL but not both: d_x_precoded = G x [batch, num_tx, M, S, fft_size] from d_x
 * [batch, num_tx, K, S, fft_size]; d_h_eff [batch, num_rx, num_rx_ant, num_tx, K, S, num_effective_subcarriers] =
 * H_ij G_j for every receiver i and transmitter j, computed from d_h (same layout as d_h_hat, may be the same
 * pointer); d_sc_pos [fft_size] gives each subcarrier's column in h_eff, -1 for a nulled one. */
int sb_ofdm_precode(const float* d_h_hat, const float* d_h, const int32_t* d_precoding_ind, const float* d_x,
                    const float* d_alpha, const int64_t* h_alpha_stride, const float* d_tx_power,
                    const int64_t* h_tx_power_stride, const int32_t* d_sc_pos, float* d_x_precoded, float* d_h_eff,
                    int64_t batch, int32_t num_rx, int32_t num_rx_ant, int32_t num_tx, int32_t num_tx_ant,
                    int32_t num_streams_per_tx, int32_t num_symbols, int32_t fft_size,
                    int32_t num_effective_subcarriers, int32_t kind, void* stream);

/* Fused receive front-end (csrc/frontend.cu): LS estimation at the pilots (+ PUSCH CDM de-spreading) + nearest /
 * linear interpolation + OFDM equaliser glue + LMMSE equalisation + square-QAM demapping in ONE launch, for receivers
 * without interfering streams and 1..4 streams (ofdm/channel_estimation.py:138-285, 364-734, ofdm/equalization.py:126-275,
 * mimo/equalization.py:101-233, mapping.py:664-691, 927-967). The estimator is linear in the received pilots, so the host
 * passes it as tables over a LIST of num_re resource elements (normally the data-carrying ones; pilot-only symbols need
 * not be listed): h_hat[ant, q](re) = sum_i t_w[q, i, re] * y[ant, t_idx[q, i, re]]  (term-major [num_tx_streams,
 * num_terms <= 16, num_re]; t_idx = position in the FULL grid, -1 ends the list), err_var[ant, q](re) = no[ant] * E[q, re],
 * d_e_sum[re] = sum_q max(E[q, re], 0).
 *   d_y [batch, num_rx, num_rx_ant, grid_size] full resource grid (num_ofdm_symbols * fft_size), d_re_full[num_re]:
 *   full-grid position of every listed RE; d_data_pos [num_tx_streams, num_re]; d_no / h_no_stride, d_desired,
 *   d_out_stream as sb_ofdm_lmmse; h_lev_re / h_lev_im: HOST arrays of the 2^bits_per_dim PAM levels by label (they
 *   travel as kernel parameters).
 *   Outputs: d_llr [batch, num_tx_streams, num_data * 2 * bits_per_dim] (method 0 app / 1 maxlog, levels as sb_demap_qam)
 *   and / or d_x_hat, d_no_eff [batch, num_tx_streams, num_data]; either may be NULL. */
int sb_ofdm_frontend(const float* d_y, const float* d_no, const int64_t* h_no_stride, const int32_t* d_desired,
                     const int32_t* d_out_stream, const int32_t* d_data_pos, const int32_t* d_re_full,
                     const int32_t* d_t_idx, const float* d_t_w, const float* d_e_sum, const float* h_lev_re,
                     const float* h_lev_im, float* d_llr, float* d_x_hat, float* d_no_eff, int64_t batch, int32_t num_rx,
                     int32_t num_rx_ant, int32_t num_tx_streams, int32_t num_re, int32_t grid_size, int32_t streams_per_rx,
                     int32_t num_terms, int32_t num_data, int32_t bits_per_dim, int32_t method, int32_t hard_out,
                     void* stream);

/* ------------------------------------------------------------------------------------------------
 * Convolutional codes, rate 1/conv_n (csrc/conv.cu)
 * replaces ConvEncoder.call                     fec/conv/encoding.py:204-291
 *          ViterbiDecoder.call / _update_fwd   fec/conv/decoding.py:236-453
 *          BCJRDecoder.call / _update_fwd/_bwd  fec/conv/decoding.py:694-943
 * Trellis: constraint length K, ns = 2^(K-1) states, the newest register bit is the state's MSB. The decoders take the
 * reference's Trellis tables (fec/conv/utils.py:148-190) as host arrays [ns, 2] int32: h_from_nodes,
 * h_op_by_tonode, h_ip_by_tonode; their order is the order in which the Viterbi decoder breaks ties. Tables that are
 * not those of a rate-1/conv_n shift register return SB_EINVAL. Limits: 2 <= ns <= 256 (K <= 9), conv_n <= 8; beyond
 * them SB_EUNSUPPORTED with a message. Any k >= 1 and any batch; codeword bits num_syms * conv_n < 2^31. All checks run
 * before any device access.
 * ---------------------------------------------------------------------------------------------- */
/* ConvEncoder: d_u [batch, k] bits (0 / 1 as float), d_x [batch, T * conv_n] with T = k + (terminate ? K - 1 : 0),
 * the conv_n bits of step t adjacent. h_gen_poly [conv_n]: polynomial j as an integer whose MSB (bit K - 1) is the
 * first character of the reference's bit string. rsc = 1: polynomial 0 is the feedback polynomial (its MSB must be
 * 1) and the termination inputs are the feedback bits (encoding.py:262-285). */
int sb_conv_encode(const float* d_u, float* d_x, int64_t batch, int32_t k, const int32_t* h_gen_poly, int32_t conv_n,
                   int32_t constraint_length, int32_t rsc, int32_t terminate, void* stream);
/* ViterbiDecoder: d_llr [batch, num_syms * conv_n] logits (Sionna's sign). method 0 "soft_llr" (branch metric
 * sum_j llr_j (1 - 2 b_j) in j order), 1 "hard" (Manhattan distance of int_mod_2 of the input). Path metrics start at
 * 0 for state 0 and 2^20 elsewhere and are never renormalised; ties go to the first predecessor. The traceback starts
 * from state 0 (terminate = 1) or the first state with the least metric. return_info_bits = 1: d_out [batch, k] input
 * bits of the first k steps (1 <= k <= num_syms); 0: d_out [batch, num_syms * conv_n] the re-encoded survivor.
 * d_workspace: sb_viterbi_workspace_bytes(batch, num_syms, ns) bytes (may be 0 and NULL; SB_ENOMEM if short). */
int sb_viterbi_decode(const float* d_llr, float* d_out, int64_t batch, int32_t num_syms, int32_t k, int32_t method,
                      int32_t terminate, int32_t return_info_bits, const int32_t* h_from_nodes,
                      const int32_t* h_op_by_tonode, const int32_t* h_ip_by_tonode, int32_t ns, int32_t conv_n,
                      void* d_workspace, size_t workspace_bytes, void* stream);
/* Device bytes of one decision bit per state and step when they do not fit in shared memory, else 0. */
size_t sb_viterbi_workspace_bytes(int64_t batch, int32_t num_syms, int32_t ns);
/* BCJRDecoder: d_llr_ch [batch, num_syms * conv_n] and optional d_llr_a [batch, num_syms] (NULL: 0) logits. algorithm
 * 0 "map", 1 "log", 2 "maxlog". "map" and "log" are the same function and both run in the log domain with the exact
 * max* (the reference's probability-domain "map" overflows fp32 once |0.5 sum llr| > 88). The backward recursion starts
 * uniform unless terminate = 1. d_out [batch, num_out] (1 <= num_out <= num_syms): the APP LLRs of the first num_out
 * steps' input bits (a turbo decoder takes all num_syms), or llr > 0 as 0 / 1 with hard_out = 1.
 * d_workspace: sb_bcjr_workspace_bytes(batch, num_syms, ns) bytes (may be 0 and NULL; SB_ENOMEM if short). */
int sb_bcjr_decode(const float* d_llr_ch, const float* d_llr_a, float* d_out, int64_t batch, int32_t num_syms,
                   int32_t num_out, int32_t algorithm, int32_t terminate, int32_t hard_out, const int32_t* h_from_nodes,
                   const int32_t* h_op_by_tonode, const int32_t* h_ip_by_tonode, int32_t ns, int32_t conv_n,
                   void* d_workspace, size_t workspace_bytes, void* stream);
/* Device bytes of the forward metrics (ns floats per step) when they do not fit in shared memory, else 0. */
size_t sb_bcjr_workspace_bytes(int64_t batch, int32_t num_syms, int32_t ns);

/* ------------------------------------------------------------------------------------------------
 * Turbo codes: two rate-1/2 RSC component codes joined by an interleaver (csrc/conv.cu)
 * replaces TurboDecoder.call / _convenc_cws      fec/turbo/decoding.py:271-312, 357-435
 *          BCJRDecoder (the component decoder)   fec/conv/decoding.py:694-943
 * The encoder composes sb_gather_rows and sb_conv_encode; only the decoder has a kernel of its own.
 * ---------------------------------------------------------------------------------------------- */
typedef struct sb_turbo_perm sb_turbo_perm;
/* The interleaver pi (Turbo3GPPInterleaver / RandomInterleaver, fec/interleaving.py:197-745): h_perm [k], decoder 2
 * sees u[pi(i)] at step i. Returns SB_EINVAL unless h_perm is a permutation of 0 ... k - 1; checked on the host
 * before any device access. The table is copied to a device by the first decode there. */
int sb_turbo_perm_create(sb_turbo_perm** out, const int32_t* h_perm, int32_t k);
void sb_turbo_perm_destroy(sb_turbo_perm* p);
/* TurboDecoder: d_llr [batch, 2, 2 T] logits (Sionna's sign) of the two component codewords, T = k + (terminate ?
 * K - 1 : 0) steps of conv_n = 2 bits each (systematic, parity), punctured positions 0; decoder 2's systematic LLRs
 * are decoder 1's through pi. Trellis tables and algorithm as sb_bcjr_decode; both component codes share them. Runs
 * num_iter iterations of decoder 1 then decoder 2 in one launch, exchanging extrinsic LLRs clipped to +-20 (prior 0 on
 * the termination steps). d_out [batch, k]: decoder 2's APP LLRs deinterleaved, or llr > 0 as 0 / 1 with hard_out = 1;
 * num_iter = 0 gives zeros. Limits: ns <= 256; conv_n other than 2 is SB_EUNSUPPORTED. A missing handle or one of
 * another length is SB_EINVAL. d_workspace: sb_turbo_workspace_bytes(batch, k, terminate, ns) bytes (may be 0 and
 * NULL; SB_ENOMEM if short). All checks run before any device access. */
int sb_turbo_decode(const float* d_llr, const sb_turbo_perm* perm, float* d_out, int64_t batch, int32_t k,
                    int32_t num_iter, int32_t algorithm, int32_t terminate, int32_t hard_out,
                    const int32_t* h_from_nodes, const int32_t* h_op_by_tonode, const int32_t* h_ip_by_tonode,
                    int32_t ns, int32_t conv_n, void* d_workspace, size_t workspace_bytes, void* stream);
/* Device bytes of the forward metrics (ns floats per step) and the extrinsic LLRs (k floats per codeword), each when it
 * does not fit in shared memory; 0 when both do. */
size_t sb_turbo_workspace_bytes(int64_t batch, int32_t k, int32_t terminate, int32_t ns);

/* ------------------------------------------------------------------------------------------------
 * Binary linear block codes (csrc/linear_codes.cu)
 * replaces LinearEncoder.call                    fec/linear/encoding.py:122-140
 *          OSDecoder.call / _find_mrb / _find_min_dist   fec/linear/decoding.py:237-478
 * ---------------------------------------------------------------------------------------------- */
/* c = u G mod 2. d_u [batch, k] and d_c [batch, n] of one dtype: 0 float32, 1 float64, 2 int32, 3 int64; an input
 * element contributes bit (long long)u & 1. d_gen_rows: G as k bit-packed rows of ceil(n / 32) words, bit b of word w
 * = column 32 w + b. Any 1 <= k <= n. batch = 0 is SB_OK with NULL pointers. */
int sb_gf2_encode(const void* d_u, void* d_c, int32_t dtype, int64_t batch, int32_t k, int32_t n,
                  const uint32_t* d_gen_rows, void* stream);
typedef struct sb_osd_code sb_osd_code;
/* h_gm [k, n] (uint8, 0 / 1): the generator matrix, checked on the host to be binary (SB_EINVAL) and of full rank
 * (SB_EINVAL); n > 1024 is SB_EUNSUPPORTED. The generator is copied to a device by the first decode there. */
int sb_osd_code_create(sb_osd_code** out, const uint8_t* h_gm, int32_t k, int32_t n);
void sb_osd_code_destroy(sb_osd_code* p);
/* Ordered statistics decoding of order t (t > k acts as t = k, i.e. exact ML): d_llr [batch, n] logits
 * log p(1) / p(0), clipped to +-100; d_out [batch, n] the hard decisions (0.0 / 1.0) of the best candidate by the
 * discrepancy sum over mismatched positions of |llr| (equal to the reference's metric's order). Ties keep the first
 * candidate in (order, itertools.combinations rank over the most reliable basis in reliability order). More than
 * 2^62 candidates, or tables that exceed shared memory, is SB_EUNSUPPORTED. All checks run before any device
 * access; batch = 0 is SB_OK with NULL pointers. */
int sb_osd_decode(const sb_osd_code* code, const float* d_llr, float* d_out, int64_t batch, int32_t t, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SIONNA_B200_H */
