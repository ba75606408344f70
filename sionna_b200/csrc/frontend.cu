// frontend.cu -- fused OFDM receive front-end for sm_90a (SURVEY.md section 8 row f1): from the received resource grid
// to bit LLRs in ONE launch. Replaces the chain (paths under /root/reference/src/sionna/phy/)
//   RemoveNulledSubcarriers                     ofdm/resource_grid.py:551
//   LSChannelEstimator / PUSCHLSChannelEstimator ofdm/channel_estimation.py:138-173, 257-285, nr/pusch_channel_estimation.py:117-169
//   Nearest-neighbour / linear interpolation    ofdm/channel_estimation.py:364-435, 479-734
//   OFDMEqualizer glue + lmmse_equalizer        ofdm/equalization.py:126-275, mimo/equalization.py:101-233
//   Demapper (square QAM, app / maxlog)         mapping.py:664-691, 927-967
// for receivers without interfering streams (diagonal noise-plus-estimation-error covariance) and up to 4 streams.
//
// Why this fuses cleanly. LS estimation (y_p / p), CDM de-spreading, nearest-neighbour and (time-averaged) linear
// interpolation are all LINEAR in the received pilot symbols, and the error variance they propagate is the noise power
// times a constant. So for stream q and resource element r
//     h_hat[ant, q](r) = sum_{i < NT} W[q, r, i] * y[ant, P[q, r, i]],      err_var[ant, q](r) = no[ant] * E[q, r]
// with host-built tables (P: pilot RE of the full grid, W: complex weight = interpolation weight / pilot, E >= 0). The
// kernel never materialises h_hat (512 B per RE for 4 x 16) or err_var: a thread owns one RE, walks the antennas once
// (y coalesced over the subcarriers; the pilot REs it gathers are shared by the whole frame and stay in L1), builds
// B = H_w^H H_w and z = H_w^H y_w in registers, solves (lmmse_diag.cuh), demaps (demap_qam.cuh) and writes the LLRs in
// the layout the decoder reads. HBM traffic per RE: y (8 B per antenna) + LLRs - against 692 B of SURVEY 8(d).
//
// Work decomposition. The host lists only the data-carrying REs (pilot-only OFDM symbols are not walked). A CTA owns a
// tile of 128 listed REs of one receiver and loops over a slice of the batch: the table words of its REs (term-major in
// HBM, so the staging loads are coalesced) are copied once into per-thread columns of shared memory and reused for every
// frame and antenna chunk. The kernel is a long straight-line program per RE (K x K solve, 2 * 2^H exponentials), so the
// instruction stream is kept small on purpose: demapping method is a template argument, the per-stream epilogue is a
// rolled loop, the underflow fallback of the demapper is out of line, and the PAM levels are kernel parameters
// (constant-bank operands, no registers).
#include <algorithm>
#include "sb_common.h"
#include "lmmse_diag.cuh"
#include "demap_qam.cuh"

namespace {

struct FrontParams {
    const float2* y;          // [B, RX, ANT, GRID] full grid (OFDM symbols x fft_size)
    const float* no;          // addressed with no_stride over (b, rx, ant)
    long long no_stride[3];
    const int* des;           // [RX, K] tx-stream index of every desired stream
    const int* out_ts;        // [RX, K] output row (tx * streams_per_tx + stream) after the stream re-ordering
    const int* data_pos;      // [TXS, SF] index among that stream's data symbols or -1
    const int* re_full;       // [SF] position of the listed RE in the full grid
    const int* t_idx;         // [TXS, NT, SF] pilot position in the full grid, -1 = unused term (term-major)
    const float2* t_w;        // [TXS, NT, SF]
    const float* e_sum;       // [SF] sum over ALL streams of the (floored) error-variance factor
    float* llr;               // [B, TXS, ND * 2H]
    float2* xh;               // optional [B, TXS, ND]
    float* ne;                // optional [B, TXS, ND]
    long long B;
    int RX, ANT, TXS, SF, ND, NT, GRID, hard_out;
    int tiles, nbg;           // RE tiles of 128; number of batch slices (grid = tiles * RX * nbg)
    float lev[2][32];         // real / imaginary PAM levels by label
};

constexpr int kAntChunk = 4;
constexpr int kTile = 128;

template <int D>
struct ParamLev {                                         // level t of dimension D straight from the constant bank
    const FrontParams& p;
    __device__ __forceinline__ float operator()(int t) const { return p.lev[D][t]; }
};

template <int K, int H, int METHOD>
__global__ void __launch_bounds__(kTile) ofdm_frontend_kernel(const __grid_constant__ FrontParams p) {
    using namespace sb_lmmse;
    constexpr int M = 2 * H;
    extern __shared__ __align__(8) unsigned char front_smem[];
    float2* s_w = reinterpret_cast<float2*>(front_smem);                       // [K][NT][128] this thread's column only
    int* s_idx = reinterpret_cast<int*>(front_smem + sizeof(float2) * K * p.NT * kTile);
    const int tid = threadIdx.x;
    const int tile = blockIdx.x % p.tiles;
    const int rx = (blockIdx.x / p.tiles) % p.RX;
    const int g = blockIdx.x / (p.tiles * p.RX);
    const int re = tile * kTile + tid;
    if (re >= p.SF) return;                                                    // no barriers below
    const long long SF = p.SF;
    int dp[K];
    bool any = false;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        dp[k] = p.data_pos[(size_t)p.out_ts[rx * K + k] * SF + re];
        any = any || dp[k] >= 0;
    }
    if (!any) return;
#pragma unroll
    for (int k = 0; k < K; ++k) {
        const long long tb = (long long)p.des[rx * K + k] * p.NT * SF + re;
        for (int t = 0; t < p.NT; ++t) {
            s_idx[(k * p.NT + t) * kTile + tid] = p.t_idx[tb + t * SF];
            s_w[(k * p.NT + t) * kTile + tid] = p.t_w[tb + t * SF];
        }
    }
    const int rf = p.re_full[re];
    const float es = p.e_sum[re];
    for (long long b = g; b < p.B; b += p.nbg) {
        float2 Bm[K * (K + 1) / 2], z[K];
        lmmse_diag_clear<K>(Bm, z);
        const float2* yb = p.y + (b * p.RX + rx) * (long long)p.ANT * p.GRID;
        const float* nb = p.no + b * p.no_stride[0] + rx * p.no_stride[1];
#pragma unroll 1
        for (int m0 = 0; m0 < p.ANT; m0 += kAntChunk) {
            const float2* yp[kAntChunk];
            float w[kAntChunk];
            float2 h[kAntChunk][K];
#pragma unroll
            for (int c = 0; c < kAntChunk; ++c) {
                const int m = min(m0 + c, p.ANT - 1);                        // tail lanes repeat the last antenna (w = 0)
                yp[c] = yb + (long long)m * p.GRID;
                const float nn = nb[m * p.no_stride[2]];
                // whitening by 1 / sqrt(no + sum_q err_var_q), err_var_q = no * E_q  (ofdm/equalization.py:205-218)
                w[c] = (m0 + c < p.ANT) ? rsqrtf(nn + nn * es) : 0.f;       // MUFU.RSQ, <= 2 ulp
#pragma unroll
                for (int k = 0; k < K; ++k) h[c][k] = make_float2(0.f, 0.f);
            }
            // channel estimates of this antenna chunk: the table words are read once per chunk
#pragma unroll
            for (int k = 0; k < K; ++k) {
#pragma unroll 1
                for (int t = 0; t < p.NT; ++t) {
                    const int pi = s_idx[(k * p.NT + t) * kTile + tid];
                    if (pi < 0) break;
                    const float2 wt = s_w[(k * p.NT + t) * kTile + tid];
#pragma unroll
                    for (int c = 0; c < kAntChunk; ++c) {
                        const float2 yv = yp[c][pi];
                        h[c][k].x = fmaf(wt.x, yv.x, fmaf(-wt.y, yv.y, h[c][k].x));
                        h[c][k].y = fmaf(wt.x, yv.y, fmaf(wt.y, yv.x, h[c][k].y));
                    }
                }
            }
#pragma unroll
            for (int c = 0; c < kAntChunk; ++c) {
                float2 yw = yp[c][rf];
                yw = make_float2(yw.x * w[c], yw.y * w[c]);
                float2 hw[K];
#pragma unroll
                for (int k = 0; k < K; ++k) hw[k] = make_float2(h[c][k].x * w[c], h[c][k].y * w[c]);
#pragma unroll
                for (int a = 0; a < K; ++a) {
                    z[a] = cadd(z[a], cmulc(yw, hw[a]));                       // conj(H_w[m, a]) * y_w[m]
#pragma unroll
                    for (int q = 0; q <= a; ++q) Bm[a * (a + 1) / 2 + q] = cadd(Bm[a * (a + 1) / 2 + q], cmulc(hw[q], hw[a]));
                }
            }
        }
        float2 xo[K];
        float no_e[K];
        lmmse_diag_solve<K>(Bm, z, xo, no_e);
#pragma unroll 1
        for (int k = 0; k < K; ++k) {                                          // rolled: ONE copy of the demapper code
            float2 x = xo[0];
            float nk = no_e[0];
            int d = dp[0];
#pragma unroll
            for (int j = 1; j < K; ++j)
                if (k == j) { x = xo[j]; nk = no_e[j]; d = dp[j]; }
            if (d < 0) continue;
            const long long o = (b * p.TXS + p.out_ts[rx * K + k]) * (long long)p.ND + d;
            if (p.xh) { p.xh[o] = x; p.ne[o] = nk; }
            if (p.llr) {
                const float inv_n0 = __fdiv_rn(1.0f, fmaxf(nk, 1.17549435e-38f));   // mapping.py:653, 672-681
                float o_re[H], o_im[H];
                demap_qam_dim<METHOD, H>(x.x, inv_n0, ParamLev<0>{p}, &p.lev[0][0], p.hard_out, o_re);
                demap_qam_dim<METHOD, H>(x.y, inv_n0, ParamLev<1>{p}, &p.lev[1][0], p.hard_out, o_im);
                float* lp = p.llr + o * M;
#pragma unroll
                for (int u = 0; u < H; ++u) { lp[2 * u] = o_re[u]; lp[2 * u + 1] = o_im[u]; }
            }
        }
    }
}

}  // namespace

extern "C" int sb_ofdm_frontend(const float* d_y, const float* d_no, const int64_t* h_no_stride, const int32_t* d_desired,
                                const int32_t* d_out_stream, const int32_t* d_data_pos, const int32_t* d_re_full,
                                const int32_t* d_t_idx, const float* d_t_w, const float* d_e_sum, const float* h_lev_re,
                                const float* h_lev_im, float* d_llr, float* d_x_hat, float* d_no_eff, int64_t batch,
                                int32_t num_rx, int32_t num_rx_ant, int32_t num_tx_streams, int32_t num_re,
                                int32_t grid_size, int32_t streams_per_rx, int32_t num_terms, int32_t num_data,
                                int32_t bits_per_dim, int32_t method, int32_t hard_out, void* stream) {
    if (batch == 0) return SB_OK;
    SB_CHECK_ARG(d_y && d_no && h_no_stride && d_desired && d_out_stream && d_data_pos && d_re_full && d_t_idx && d_t_w &&
                     d_e_sum && (d_llr || (d_x_hat && d_no_eff)) && (!d_llr || (h_lev_re && h_lev_im)),
                 "sb_ofdm_frontend: null pointer");
    SB_CHECK_ARG(batch > 0 && num_rx > 0 && num_rx_ant > 0 && num_tx_streams > 0 && num_re > 0 && grid_size > 0 &&
                     num_terms >= 1 && num_terms <= 16 && num_data > 0 && (method == 0 || method == 1),
                 "sb_ofdm_frontend: bad sizes");
    SB_CHECK_ARG(streams_per_rx >= 1 && streams_per_rx <= 4, "sb_ofdm_frontend: 1..4 streams per receiver");
    SB_CHECK_ARG(!d_llr || (bits_per_dim >= 1 && bits_per_dim <= 5), "sb_ofdm_frontend: square QAM up to 1024 points");
    SB_CHECK_ARG((d_x_hat == nullptr) == (d_no_eff == nullptr), "sb_ofdm_frontend: x_hat and no_eff go together");
    FrontParams p{};
    p.y = (const float2*)d_y; p.no = d_no;
    for (int i = 0; i < 3; ++i) p.no_stride[i] = h_no_stride[i];
    p.des = d_desired; p.out_ts = d_out_stream; p.data_pos = d_data_pos; p.re_full = d_re_full; p.t_idx = d_t_idx;
    p.t_w = (const float2*)d_t_w; p.e_sum = d_e_sum; p.llr = d_llr;
    p.xh = (float2*)d_x_hat; p.ne = d_no_eff; p.B = batch; p.RX = num_rx; p.ANT = num_rx_ant; p.TXS = num_tx_streams;
    p.SF = num_re; p.ND = num_data; p.NT = num_terms; p.GRID = grid_size; p.hard_out = hard_out;
    const int h = d_llr ? bits_per_dim : 1;
    if (d_llr)
        for (int t = 0; t < (1 << h); ++t) { p.lev[0][t] = h_lev_re[t]; p.lev[1][t] = h_lev_im[t]; }
    p.tiles = (p.SF + kTile - 1) / kTile;
    const long long per_slice = (long long)p.tiles * p.RX;
    p.nbg = (int)std::max<long long>(1, std::min<long long>(p.B, ((long long)sb_num_sms() * 8 + per_slice - 1) / per_slice));
    const long long grid = per_slice * p.nbg;
    const size_t smem = (sizeof(float2) + sizeof(int)) * (size_t)streams_per_rx * p.NT * kTile;
    const int rc = grid > 0x7fffffffLL ? SB_EUNSUPPORTED : sb_dispatch<1, 4>(streams_per_rx, [&](auto K) {
        return sb_dispatch<1, 5>(h, [&](auto H) {
            return sb_dispatch<0, 1>(method, [&](auto METHOD) {
                auto kern = ofdm_frontend_kernel<K, H, METHOD>;
                if (smem > 48 * 1024 &&
                    cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
                    return SB_EUNSUPPORTED;
                kern<<<(unsigned)grid, kTile, smem, (cudaStream_t)stream>>>(p);
                return SB_OK;
            });
        });
    });
    if (rc) { sb_set_error("sb_ofdm_frontend: unsupported configuration"); return rc; }
    SB_LAUNCH_CHECK();
    return SB_OK;
}
