// channel.cu -- on-device channel generation and application for sm_90a (SURVEY.md section 8 row f3): the TDL taps,
// everything the CIR -> channel conversion needs so that no step of it runs as an eager tensor expression, and the
// channel applied to a signal. Replaces (paths under /root/reference/src/sionna/phy/):
//   sb_tdl_sos            TDL.__call__ sum of sinusoids      channel/tr38901/tdl.py:372-456
//   sb_phase_table        exp(-j 2 pi f tau) of cir_to_ofdm_channel   channel/utils.py:232-244
//                         sinc(l - tau W)    of cir_to_time_channel   channel/utils.py:318-338
//   sb_cir_gram           (no counterpart: Gram matrix of the table, used to normalise without a second pass over h)
//   sb_cir_link_scale     normalisation factor of channel/utils.py:246-251 (OFDM) and :341-348 (time)
//   sb_cir_apply          h = sum_p a_p e_p (channel/utils.py:240-244, 336-338), per-link tables and scaling folded in
//   sb_spatial_corr       TDL._apply_correlation (channel/tr38901/tdl.py:466-490): v' = L v per (batch, path, time step)
//   sb_apply_ofdm_channel ApplyOFDMChannel.call   channel/apply_ofdm_channel.py:70-80
//   sb_apply_time_channel ApplyTimeChannel.call   channel/apply_time_channel.py:115-137
//
// Normalisation without touching h twice. The reference computes c = sqrt(mean |h|^2) over (rx ant, tx ant, time,
// frequency) per link from the finished tensor and divides. Because h[f] = sum_p a_p e[p, f],
//     sum_f |h[f]|^2 = sum_{p,q} a_p conj(a_q) G[p, q],   G[p, q] = sum_f e[p, f] conj(e[q, f]),
// so the link energy follows from the P path gains and the P x P Gram matrix of the table (P <= 24 for every TDL
// model): sb_cir_link_scale evaluates that quadratic form (P^2 MACs per (antenna pair, time step) instead of reading
// F * 8 bytes) and sb_cir_apply writes the already scaled h exactly once. Every reduction runs in a fixed order
// (no atomics): results are reproducible bit for bit from run to run.
#include "sb_common.h"
#include "rng.cuh"

namespace {

// e[tab, p, j]: mode 0: exp(-j 2 pi x_j tau[tab, p]); mode 1: sinc(x_j - tau[tab, p] * scale) (+ 0 j).
// The phase is reduced in double precision (f tau reaches a few turns) and evaluated with sincospi.
__global__ void phase_table_kernel(const float* __restrict__ tau, const float* __restrict__ x, float2* __restrict__ e,
                                   long long n_tab, int P, int F, float scale, int mode) {
    const long long total = n_tab * P * (long long)F;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const int j = (int)(i % F);
        const long long tp = i / F;
        const double t = (double)tau[tp];
        if (mode == 0) {
            double turns = (double)x[j] * t;                     // f * tau
            turns -= rint(turns);
            double s, c;
            sincospi(-2.0 * turns, &s, &c);
            e[i] = make_float2((float)c, (float)s);
        } else {
            const double u = (double)x[j] - t * (double)scale;   // l - tau W
            double v = 1.0;
            if (u != 0.0) v = sinpi(u) / (3.141592653589793 * u);
            e[i] = make_float2((float)v, 0.f);
        }
    }
}

// G[tab, p, q] = sum_j e[tab, p, j] conj(e[tab, q, j]) in double (every fp32 x fp32 product is exact there); one warp per
// (tab, p, q), lanes stride j, fixed shuffle tree.
__global__ void cir_gram_kernel(const float2* __restrict__ e, double2* __restrict__ g, long long n_tab, int P, int F) {
    const int lane = threadIdx.x & 31;
    const long long warps = ((long long)gridDim.x * blockDim.x) >> 5;
    const long long total = n_tab * P * (long long)P;
    for (long long w = (((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5); w < total; w += warps) {
        const int q = (int)(w % P);
        const int p = (int)((w / P) % P);
        const long long tab = w / ((long long)P * P);
        const float2* ep = e + (tab * P + p) * (long long)F;
        const float2* eq = e + (tab * P + q) * (long long)F;
        double re = 0.0, im = 0.0;
        for (int j = lane; j < F; j += 32) {
            const float2 a = ep[j], b = eq[j];
            re += (double)a.x * b.x + (double)a.y * b.y;
            im += (double)a.y * b.x - (double)a.x * b.y;
        }
        for (int o = 16; o > 0; o >>= 1) {
            re += __shfl_down_sync(0xffffffffu, re, o);
            im += __shfl_down_sync(0xffffffffu, im, o);
        }
        if (lane == 0) g[w] = make_double2(re, im);
    }
}

// Tap layout a[b, rx, ra, tx, ta, p, t]; a "link" is (b, rx, tx), its rows are the RA * TA antenna pairs.
struct CirDims { long long B; int RX, RA, TX, TA, P, T; };

// scale[link] = 1 / sqrt( (sum over the link's antenna pairs and time steps of a^H G a) / (RA * TA * T * denom) ), 0 if
// the energy is 0. One CTA per link: thread k takes (pair, t) items k, k + blockDim, ... in order; fixed tree afterwards.
// Everything in double: on a nearly flat channel (delays close against 1 / bandwidth) G is almost rank one, and on a link
// in a deep fade the diagonal and the off-diagonal terms cancel to a small fraction of either; in fp32 that left
// errors of up to a few percent in the factor and could even drive the energy of a non-zero link to <= 0. In double
// the taps' fp32 products are exact and the rounding of the sum stays ~1e-16 of the terms.
__global__ void cir_link_scale_kernel(const float2* __restrict__ a, const double2* __restrict__ g, long long g_link_stride,
                                      float* __restrict__ scale, CirDims d, double denom) {
    extern __shared__ double2 s_g[];                             // P x P
    __shared__ double s_part[32];
    const long long links = d.B * d.RX * d.TX;
    for (long long link = blockIdx.x; link < links; link += gridDim.x) {
        const int tx = (int)(link % d.TX);
        const int rx = (int)((link / d.TX) % d.RX);
        const long long b = link / ((long long)d.TX * d.RX);
        const double2* gp = g + link * g_link_stride;
        __syncthreads();
        for (int i = threadIdx.x; i < d.P * d.P; i += blockDim.x) s_g[i] = gp[i];
        __syncthreads();
        const int items = d.RA * d.TA * d.T;
        double acc = 0.0;
        for (int it = threadIdx.x; it < items; it += blockDim.x) {
            const int t = it % d.T;
            const int pair = it / d.T;
            const int ta = pair % d.TA, ra = pair / d.TA;
            const long long row = (((b * d.RX + rx) * d.RA + ra) * d.TX + tx) * d.TA + ta;
            const float2* ap = a + row * (long long)d.P * d.T + t;
            double e = 0.0;
            for (int p = 0; p < d.P; ++p) {
                const float2 x = ap[(size_t)p * d.T];
                // diagonal term + 2 Re of the strictly lower triangle (G is Hermitian)
                e += ((double)x.x * x.x + (double)x.y * x.y) * s_g[p * d.P + p].x;
                double s = 0.0;
                for (int q = 0; q < p; ++q) {
                    const float2 y = ap[(size_t)q * d.T];
                    const double2 gq = s_g[p * d.P + q];            // sum_f e_p conj(e_q)
                    // terms (p, q) and (q, p) together: 2 Re( a_p conj(a_q) G[p, q] ); a_p conj(a_q) is exact in double
                    const double cr = (double)x.x * y.x + (double)x.y * y.y, ci = (double)x.y * y.x - (double)x.x * y.y;
                    s += cr * gq.x - ci * gq.y;
                }
                e += 2.0 * s;
            }
            acc += e;
        }
        for (int o = 16; o > 0; o >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, o);
        if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
        __syncthreads();
        if (threadIdx.x == 0) {
            double tot = 0.0;
            for (int w = 0; w < (int)(blockDim.x >> 5); ++w) tot += s_part[w];
            const double mean = tot / ((double)items * denom);
            scale[link] = mean > 0.0 ? (float)(1.0 / sqrt(mean)) : 0.f;
        }
    }
}

// h[row, t, j] = scale[link(row)] * sum_p a[row, p, t] e[tab(row), p, j]
// A CTA owns a TILE_T x TILE_F tile of one antenna-pair row: the P x TILE_T taps and the P x TILE_F table entries are
// staged in shared memory once, every thread accumulates RT x RJ outputs in registers (per path: RT + RJ shared loads
// feed RT * RJ complex multiply-adds), so the kernel is bound by the FP32 pipe and by the single write of h instead of
// by 2 * P loads per output. Two shapes: wide rows (OFDM: F = 76 ... 4096 subcarriers, few time steps) and narrow rows
// (time channel: l_tot ~ 20 taps, thousands of time steps).
template <int TILE_T, int RT, int TILE_F, int RJ>
__global__ void __launch_bounds__((TILE_T / RT) * (TILE_F / RJ))
cir_apply_kernel(const float2* __restrict__ a, const float2* __restrict__ e, long long e_link_stride,
                 const float* __restrict__ scale, float2* __restrict__ h, CirDims d, int F, int tiles_t, int tiles_f) {
    extern __shared__ float2 s_cir[];
    constexpr int NTJ = TILE_F / RJ;                             // threads along the columns
    float2* s_a = s_cir;                                          // [P][TILE_T]
    float2* s_e = s_cir + (size_t)d.P * TILE_T;                   // [P][TILE_F]
    const int tj = threadIdx.x % NTJ, tt = threadIdx.x / NTJ;
    const long long R = d.B * d.RX * d.RA * d.TX * d.TA;
    const long long n_tiles = R * tiles_t * tiles_f;
    for (long long tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int ft = (int)(tile % tiles_f);
        const int tq = (int)((tile / tiles_f) % tiles_t);
        const long long r = tile / ((long long)tiles_f * tiles_t);
        const int tx = (int)((r / d.TA) % d.TX);
        const long long link = (r / ((long long)d.TA * d.TX * d.RA)) * d.TX + tx;   // (b * RX + rx) * TX + tx
        const float sc = scale ? scale[link] : 1.f;
        const float2* ap = a + r * (long long)d.P * d.T;
        const float2* ep = e + link * e_link_stride;
        const int t0 = tq * TILE_T, j0 = ft * TILE_F;
        __syncthreads();
        for (int i = threadIdx.x; i < d.P * TILE_T; i += blockDim.x) {
            const int p = i / TILE_T, t = t0 + i % TILE_T;
            s_a[i] = t < d.T ? ap[(size_t)p * d.T + t] : make_float2(0.f, 0.f);
        }
        for (int i = threadIdx.x; i < d.P * TILE_F; i += blockDim.x) {
            const int p = i / TILE_F, j = j0 + i % TILE_F;
            s_e[i] = j < F ? ep[(size_t)p * F + j] : make_float2(0.f, 0.f);
        }
        __syncthreads();
        float2 acc[RT][RJ];
#pragma unroll
        for (int u = 0; u < RT; ++u)
#pragma unroll
            for (int v = 0; v < RJ; ++v) acc[u][v] = make_float2(0.f, 0.f);
        for (int p = 0; p < d.P; ++p) {
            float2 av[RT], ev[RJ];
#pragma unroll
            for (int u = 0; u < RT; ++u) av[u] = s_a[p * TILE_T + tt * RT + u];
#pragma unroll
            for (int v = 0; v < RJ; ++v) ev[v] = s_e[p * TILE_F + tj + v * NTJ];
#pragma unroll
            for (int u = 0; u < RT; ++u)
#pragma unroll
                for (int v = 0; v < RJ; ++v) {
                    // explicit FMAs (the library is built with -fmad=false for the bit-exact decoder kernels)
                    acc[u][v].x = fmaf(av[u].x, ev[v].x, fmaf(-av[u].y, ev[v].y, acc[u][v].x));
                    acc[u][v].y = fmaf(av[u].x, ev[v].y, fmaf(av[u].y, ev[v].x, acc[u][v].y));
                }
        }
#pragma unroll
        for (int u = 0; u < RT; ++u) {
            const int t = t0 + tt * RT + u;
            if (t >= d.T) continue;
            float2* hp = h + (r * d.T + t) * (long long)F;
#pragma unroll
            for (int v = 0; v < RJ; ++v) {
                const int j = j0 + tj + v * NTJ;
                if (j < F) hp[j] = make_float2(acc[u][v].x * sc, acc[u][v].y * sc);
            }
        }
    }
}

template <int TILE_T, int RT, int TILE_F, int RJ>
int launch_cir_apply(const float2* a, const float2* e, long long e_link_stride, const float* scale, float2* h, const CirDims& d,
                     int F, cudaStream_t stream) {
    auto kern = cir_apply_kernel<TILE_T, RT, TILE_F, RJ>;
    const size_t smem = sizeof(float2) * (size_t)d.P * (TILE_T + TILE_F);
    SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int tiles_t = (d.T + TILE_T - 1) / TILE_T, tiles_f = (F + TILE_F - 1) / TILE_F;
    const long long R = d.B * d.RX * d.RA * d.TX * d.TA;
    kern<<<sb_grid(R * tiles_t * tiles_f, 1, 16), (TILE_T / RT) * (TILE_F / RJ), smem, stream>>>(a, e, e_link_stride, scale, h, d, F,
                                                                                         tiles_t, tiles_f);
    return SB_OK;
}

// out[b, i, c] = sum_j L[i, j] in[b, j, c]: i, j over the n antenna pairs (rx ant major), c over the (path, time) columns.
__global__ void spatial_corr_kernel(const float2* __restrict__ in, const float2* __restrict__ l, float2* __restrict__ out,
                                    long long B, int n, long long cols) {
    extern __shared__ float2 s_l[];                              // n x n
    for (int i = threadIdx.x; i < n * n; i += blockDim.x) s_l[i] = l[i];
    __syncthreads();
    const long long total = B * cols;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
        const long long b = i / cols, c = i - b * cols;
        const float2* ip = in + b * n * cols + c;
        float2* op = out + b * n * cols + c;
        for (int r = 0; r < n; ++r) {
            float2 acc = make_float2(0.f, 0.f);
            for (int j = 0; j <= r; ++j) {                         // L is lower triangular (Cholesky factor)
                const float2 v = cmul(s_l[r * n + j], ip[(size_t)j * cols]);
                acc.x += v.x;
                acc.y += v.y;
            }
            op[(size_t)r * cols] = acc;
        }
    }
}

// TDL tap gains by the sum-of-sinusoids model: for link b, antenna pair a (rx-major), path p, time step t
//   a = sqrt(P_p / Ns) sum_n exp(j (w_b t/fs cos(2 pi (n+1)/Ns + theta[b,p,n]) + phi[b,a,p,n]))
//       (+ sqrt(P_los) exp(j (w_b t/fs cos(aoa) + phi0[b])) on path 0 of the LoS models)
// One thread per (b, a, p) row. Time is processed in chunks of 16 steps held in registers: per sinusoid one cos for the
// angular rate, one sincos for the phasor at the chunk start and one for the per-step rotation, then 16 complex
// multiplications (the recurrence is re-anchored every chunk, so its rounding error stays below 1e-6).
constexpr int kSosChunk = 16;
__device__ __forceinline__ void sos_accumulate(float2* acc, float rate, float phase, int t0) {
    float s0, c0, sd, cd;
    sincosf(rate * (float)t0 + phase, &s0, &c0);
    sincosf(rate, &sd, &cd);
    float2 z = make_float2(c0, s0);
    const float2 step = make_float2(cd, sd);
#pragma unroll
    for (int i = 0; i < kSosChunk; ++i) {
        acc[i].x += z.x;
        acc[i].y += z.y;
        z = cmul(z, step);
    }
}
__global__ void tdl_sos_kernel(const float* __restrict__ doppler, const float* __restrict__ theta,
                               const float* __restrict__ phi, const float* __restrict__ phi0,
                               const float* __restrict__ powers, float los_power, float los_aoa, float2* __restrict__ out,
                               long long B, int A, int P, int Ns, int T, float fs) {
    const long long rows = B * A * P;                            // (b, a, p)
    for (long long row = (long long)blockIdx.x * blockDim.x + threadIdx.x; row < rows; row += (long long)gridDim.x * blockDim.x) {
        const int p = (int)(row % P);
        const long long b = row / ((long long)P * A);
        const float wd = doppler[b] / fs;                        // radians per time step at cos = 1
        const float* th = theta + (b * P + p) * (long long)Ns;
        const float* ph = phi + row * (long long)Ns;
        const float amp = sqrtf(powers[p]) * (1.0f / sqrtf((float)Ns));
        const bool los = phi0 != nullptr && p == 0;
        const float la = los ? sqrtf(los_power) : 0.f;
        for (int t0 = 0; t0 < T; t0 += kSosChunk) {
            float2 acc[kSosChunk];
#pragma unroll
            for (int i = 0; i < kSosChunk; ++i) acc[i] = make_float2(0.f, 0.f);
            for (int n = 0; n < Ns; ++n) {
                const float alpha = 6.283185307179586f / (float)Ns * (float)(n + 1) + th[n];
                sos_accumulate(acc, wd * cosf(alpha), ph[n], t0);
            }
            float2 spec[kSosChunk];
#pragma unroll
            for (int i = 0; i < kSosChunk; ++i) spec[i] = make_float2(0.f, 0.f);
            if (los) sos_accumulate(spec, wd * cosf(los_aoa), phi0[b], t0);
#pragma unroll
            for (int i = 0; i < kSosChunk; ++i)
                if (t0 + i < T) out[row * T + t0 + i] = make_float2(acc[i].x * amp + la * spec[i].x, acc[i].y * amp + la * spec[i].y);
        }
    }
}

// CDL cluster coefficients (TR 38.901 (7.5-22), (7.5-28)..(7.5-30) without sub-clustering):
//   a[b, u, v, o, t] = sum_r g_r[pol(u), pol(v)] A_rx[rx_r, u] A_tx[tx_r, v] exp(j w_r t)   (+ the LoS ray on o = 0)
// for output cluster o = table cluster c = order[o]. Ray r of cluster c takes the arrival angles (zenith index
// perm_zoa[r], azimuth index perm_aoa[r]) and the departure angles likewise, perm = argsort of the coupling normals; rx_r
// and tx_r are the rows c * 400 + zenith * 20 + azimuth of the per-instance tables. g_r = F_rx^T M_r F_tx scaled by
// sqrt(P_c / 20) (and sqrt(1 / (K + 1))), M_r = [[e^{j p0}, x e^{j p1}], [x e^{j p2}, e^{j p3}]], x = sqrt(1 / XPR);
// w_r = k (r_rx . v) / fs is the Doppler phase per sample with the arrival unit vector r_rx.
// A CTA owns one batch element and a tile of up to kCdlTile time steps:
//   1. ranks the 4 x C x 20 coupling normals (comparison counts, ties broken by index as a stable argsort does);
//   2. builds the per-ray record (table rows, 4 polarization gains, Doppler rate) in shared memory;
//   3. evaluates the C x 20 (+ 1) Doppler phasors of the tile once, for every antenna pair;
//   4. thread = (antenna pair, output cluster): the 20 (21) ray coefficients in registers, one complex MAC per ray and
//      time step; the tile goes through shared memory so that the stores are contiguous runs of the
//      [batch, rx ant, tx ant, cluster, time] output, which is written exactly once.
// Shared-memory arrays are indexed with the cluster innermost: adjacent lanes read adjacent words.
constexpr int kCdlRays = 20;
constexpr int kCdlTile = 16;
constexpr int kCdlThreads = 256;
constexpr int kCdlMaxClusters = 24;
struct CdlArgs {
    const float *speed, *v_phi, *v_theta, *coupling, *phases, *rx_dir, *rx_field, *tx_field, *cluster_scale, *los_field;
    const float2 *rx_phase, *tx_phase;
    const int *rx_pol, *tx_pol, *order;
    float xpr_scale, wavenumber, fs;
    float2* out;
    long long B;
    int C, NR, NT, T;
};

__global__ void __launch_bounds__(kCdlThreads) cdl_kernel(CdlArgs p) {
    extern __shared__ float2 s_cdl[];
    const int C = p.C, CR = C * kCdlRays;
    float2* s_dop = s_cdl;                                          // [20][tile][C] + LoS [tile]
    float2* s_out = s_dop + (size_t)(CR + 1) * kCdlTile;            // [threads][tile + 1]
    float2* s_g = s_out + (size_t)kCdlThreads * (kCdlTile + 1);     // [20][4][C] + LoS [4]
    float* s_w = (float*)(s_g + (size_t)4 * CR + 4);                // [20][C] + LoS
    int* s_rx = (int*)(s_w + CR + 1);                               // [20][C]
    int* s_tx = s_rx + CR;                                          // [20][C]
    unsigned char* s_perm = (unsigned char*)(s_tx + CR);            // [4][C][20]
    const bool los = p.los_field != nullptr;
    const int tiles = (p.T + kCdlTile - 1) / kCdlTile;
    const int pairs = p.NR * p.NT, items = pairs * C;
    for (long long blk = blockIdx.x; blk < p.B * tiles; blk += gridDim.x) {
        const long long b = blk / tiles;
        const int t0 = (int)(blk % tiles) * kCdlTile;
        const int nt = min(kCdlTile, p.T - t0);
        __syncthreads();
        for (int i = threadIdx.x; i < 4 * CR; i += blockDim.x) {
            const float* x = p.coupling + (b * 4 * C + i / kCdlRays) * kCdlRays;
            const int r = i % kCdlRays;
            const float v = x[r];
            int rank = 0;
            for (int j = 0; j < kCdlRays; ++j) rank += (x[j] < v) || (x[j] == v && j < r);
            s_perm[i - r + rank] = (unsigned char)r;
        }
        __syncthreads();
        const float sp = p.speed[b], vph = p.v_phi[b], vth = p.v_theta[b];
        const float vx = sp * cosf(vph) * sinf(vth), vy = sp * sinf(vph) * sinf(vth), vz = sp * cosf(vth);
        const float kw = p.wavenumber / p.fs;
        for (int i = threadIdx.x; i < CR + 1; i += blockDim.x) {
            if (i == CR) {                                          // the LoS ray: fixed gains, LoS arrival direction
                if (los) {
                    const float* d = p.rx_dir + (size_t)CR * kCdlRays * 3;
                    s_w[CR] = kw * (d[0] * vx + d[1] * vy + d[2] * vz);
                    for (int k = 0; k < 4; ++k) s_g[4 * CR + k] = make_float2(p.los_field[k], 0.f);
                }
                continue;
            }
            const int c = i / kCdlRays, r = i % kCdlRays;
            const int ia = s_perm[(0 * C + c) * kCdlRays + r], id = s_perm[(1 * C + c) * kCdlRays + r];
            const int iz = s_perm[(2 * C + c) * kCdlRays + r], izd = s_perm[(3 * C + c) * kCdlRays + r];
            const int rx = (c * kCdlRays + iz) * kCdlRays + ia, tx = (c * kCdlRays + izd) * kCdlRays + id;
            const int k = r * C + c;
            s_rx[k] = rx;
            s_tx[k] = tx;
            const float* d = p.rx_dir + (size_t)rx * 3;
            s_w[k] = kw * (d[0] * vx + d[1] * vy + d[2] * vz);
            const float* ph = p.phases + ((b * C + c) * kCdlRays + r) * 4;
            float2 e[4];
            for (int q = 0; q < 4; ++q) sincosf(ph[q], &e[q].y, &e[q].x);
            const float xs = p.xpr_scale, sc = p.cluster_scale[c];
            const float* fr = p.rx_field + (size_t)rx * 4;
            const float* ft = p.tx_field + (size_t)tx * 4;
            for (int pr = 0; pr < 2; ++pr)
                for (int pt = 0; pt < 2; ++pt) {
                    const float t_th = ft[2 * pt], t_ph = ft[2 * pt + 1];
                    // M F_tx, then F_rx^T (M F_tx)
                    const float2 m0 = make_float2(e[0].x * t_th + xs * e[1].x * t_ph, e[0].y * t_th + xs * e[1].y * t_ph);
                    const float2 m1 = make_float2(xs * e[2].x * t_th + e[3].x * t_ph, xs * e[2].y * t_th + e[3].y * t_ph);
                    const float r_th = fr[2 * pr], r_ph = fr[2 * pr + 1];
                    s_g[(r * 4 + pr * 2 + pt) * C + c] = make_float2(sc * (r_th * m0.x + r_ph * m1.x), sc * (r_th * m0.y + r_ph * m1.y));
                }
        }
        __syncthreads();
        for (int i = threadIdx.x; i < (CR + 1) * kCdlTile; i += blockDim.x) {
            const int tt = i / (CR + 1), k = i % (CR + 1);         // k = r * C + c, or CR for the LoS ray
            if (k == CR && !los) continue;
            float s, co;
            sincosf(s_w[k] * (float)(t0 + tt), &s, &co);
            const int r = k / C, c = k % C;
            s_dop[k == CR ? (size_t)CR * kCdlTile + tt : ((size_t)r * kCdlTile + tt) * C + c] = make_float2(co, s);
        }
        __syncthreads();
        for (int base = 0; base < items; base += kCdlThreads) {
            const int item = base + threadIdx.x;
            if (item < items) {
                const int o = item % C, pair = item / C;
                const int c = p.order[o], u = pair / p.NT, v = pair % p.NT;
                const int pq = p.rx_pol[u] * 2 + p.tx_pol[v];
                float2 coef[kCdlRays + 1];
#pragma unroll
                for (int r = 0; r < kCdlRays; ++r) {
                    const int k = r * C + c;
                    const float2 g = s_g[(r * 4 + pq) * C + c];
                    const float2 ar = __ldg(p.rx_phase + (size_t)s_rx[k] * p.NR + u);
                    const float2 at = __ldg(p.tx_phase + (size_t)s_tx[k] * p.NT + v);
                    coef[r] = cmul(cmul(g, ar), at);
                }
                const bool los_here = los && o == 0;
                coef[kCdlRays] = make_float2(0.f, 0.f);
                if (los_here) {
                    const size_t row = (size_t)C * kCdlRays * kCdlRays;
                    coef[kCdlRays] = cmul(cmul(s_g[4 * CR + pq], __ldg(p.rx_phase + row * p.NR + u)),
                                          __ldg(p.tx_phase + row * p.NT + v));
                }
                for (int tt = 0; tt < nt; ++tt) {
                    float2 acc = make_float2(0.f, 0.f);
#pragma unroll
                    for (int r = 0; r < kCdlRays; ++r) {
                        const float2 z = s_dop[((size_t)r * kCdlTile + tt) * C + c];
                        acc.x += coef[r].x * z.x - coef[r].y * z.y;
                        acc.y += coef[r].x * z.y + coef[r].y * z.x;
                    }
                    if (los_here) {
                        const float2 z = s_dop[(size_t)CR * kCdlTile + tt];
                        acc.x += coef[kCdlRays].x * z.x - coef[kCdlRays].y * z.y;
                        acc.y += coef[kCdlRays].x * z.y + coef[kCdlRays].y * z.x;
                    }
                    s_out[threadIdx.x * (kCdlTile + 1) + tt] = acc;
                }
            }
            __syncthreads();
            const int n_items = min(kCdlThreads, items - base);
            float2* op = p.out + ((b * items + base) * (long long)p.T + t0);
            for (int i = threadIdx.x; i < n_items * nt; i += blockDim.x) {
                const int li = i / nt, tt = i % nt;
                op[(size_t)li * p.T + tt] = s_out[li * (kCdlTile + 1) + tt];
            }
            __syncthreads();
        }
    }
}

static size_t cdl_smem_bytes(int C) {
    const size_t cr = (size_t)C * kCdlRays;
    return sizeof(float2) * ((cr + 1) * kCdlTile + (size_t)kCdlThreads * (kCdlTile + 1) + 4 * cr + 4) +
           sizeof(float) * (cr + 1) + 2 * sizeof(int) * cr + 4 * cr;
}

// ApplyOFDMChannel: y[b, r, re] = sum_t h[b, r, t, re] * x[b, t, re] + sqrt(no) CN(0,1)   (r = rx*ant, t = tx*ant)
__global__ void apply_ofdm_channel_kernel(const float2* __restrict__ x, const float2* __restrict__ h,
                                          const float* __restrict__ no, long long no_inner, float2* __restrict__ y,
                                          long long B, int R, int Tt, int RE, int add_noise, unsigned long long seed,
                                          unsigned long long offset) {
    const long long rows = B * R;
    for (long long row = (long long)blockIdx.x * blockDim.y + threadIdx.y; row < rows; row += (long long)gridDim.x * blockDim.y) {
        const long long b = row / R;
        const float2* hp = h + row * (long long)Tt * RE;
        const float2* xp = x + b * (long long)Tt * RE;
        const long long obase = row * (long long)RE;
        const bool row_no = add_noise && (no_inner % RE) == 0;      // one noise power per row (the usual case)
        const float sd_row = row_no ? sqrtf(no[obase / no_inner]) * 0.70710678118654752f : 0.f;
        for (int re = threadIdx.x; re < RE; re += blockDim.x) {
            float2 acc = make_float2(0.f, 0.f);
            for (int t = 0; t < Tt; ++t) acc = cadd(acc, cmul(hp[(size_t)t * RE + re], xp[(size_t)t * RE + re]));
            if (add_noise) {
                const unsigned long long i = (unsigned long long)(obase + re);    // same Philox counter as the flat index
                uint4 rr = philox4x32_10(seed, offset, i);
                float2 g = box_muller(rr.x, rr.y);
                float sd = row_no ? sd_row : sqrtf(no[i / (unsigned long long)no_inner]) * 0.70710678118654752f;
                acc.x += g.x * sd;
                acc.y += g.y * sd;
            }
            y[obase + re] = acc;
        }
    }
}

// ApplyTimeChannel (channel/apply_time_channel.py:115-137): time-variant FIR filtering
//   y[b, r, n] = sum_t sum_l h[b, r, t, n, l] x[b, t, n - l]   (x = 0 outside [0, N)),  n in [0, N + L - 1)
// r = (rx, rx_ant), t = (tx, tx_ant). A CTA row is (b, r); threads walk the output samples.
__global__ void apply_time_channel_kernel(const float2* __restrict__ x, const float2* __restrict__ h,
                                          const float* __restrict__ no, long long no_inner, float2* __restrict__ y,
                                          long long B, int R, int Tt, int N, int L, int add_noise, unsigned long long seed,
                                          unsigned long long offset) {
    const int NO = N + L - 1;
    const long long rows = B * R;
    for (long long row = (long long)blockIdx.x * blockDim.y + threadIdx.y; row < rows; row += (long long)gridDim.x * blockDim.y) {
        const long long b = row / R;
        const long long obase = row * (long long)NO;
        for (int n = threadIdx.x; n < NO; n += blockDim.x) {
            float2 acc = make_float2(0.f, 0.f);
            for (int t = 0; t < Tt; ++t) {
                const float2* hp = h + ((row * Tt + t) * (long long)NO + n) * L;
                const float2* xp = x + (b * Tt + t) * (long long)N;
                const int l0 = n - (N - 1) > 0 ? n - (N - 1) : 0;     // n - l <= N - 1
                const int l1 = n < L - 1 ? n : L - 1;                  // n - l >= 0
                for (int l = l0; l <= l1; ++l) acc = cadd(acc, cmul(hp[l], xp[n - l]));
            }
            if (add_noise) {
                const unsigned long long i = (unsigned long long)(obase + n);
                uint4 rr = philox4x32_10(seed, offset, i);
                float2 g = box_muller(rr.x, rr.y);
                float sd = sqrtf(no[i / (unsigned long long)no_inner]) * 0.70710678118654752f;
                acc.x += g.x * sd;
                acc.y += g.y * sd;
            }
            y[obase + n] = acc;
        }
    }
}

}  // namespace

extern "C" int sb_tdl_sos(const float* d_doppler, const float* d_theta, const float* d_phi, const float* d_phi0,
                          const float* d_powers, float los_power, float los_aoa, float* d_a, int64_t batch,
                          int32_t num_ant_pairs, int32_t num_paths, int32_t num_sinusoids, int32_t num_time_steps,
                          float sampling_frequency, void* stream) {
    if (batch == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_doppler && d_theta && d_phi && d_powers && d_a && num_ant_pairs > 0 && num_paths > 0 &&
                     num_sinusoids > 0 && num_time_steps > 0 && sampling_frequency > 0.f, "sb_tdl_sos: bad arguments");
    tdl_sos_kernel<<<sb_grid(batch * num_ant_pairs * num_paths, 128, 16), 128, 0, (cudaStream_t)stream>>>(
        d_doppler, d_theta, d_phi, d_phi0, d_powers, los_power, los_aoa, (float2*)d_a, batch, num_ant_pairs, num_paths,
        num_sinusoids, num_time_steps, sampling_frequency);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_cdl_coefficients(const float* d_speed, const float* d_v_phi, const float* d_v_theta,
                                   const float* d_coupling, const float* d_phases, const float* d_rx_dir,
                                   const float* d_rx_field, const float* d_rx_phase, const int32_t* d_rx_pol,
                                   const float* d_tx_field, const float* d_tx_phase, const int32_t* d_tx_pol,
                                   const float* d_cluster_scale, const int32_t* d_order, const float* d_los_field,
                                   float xpr_scale, float wavenumber, float* d_a, int64_t batch, int32_t num_clusters,
                                   int32_t num_rx_ant, int32_t num_tx_ant, int32_t num_time_steps,
                                   float sampling_frequency, void* stream) {
    if (batch == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_speed && d_v_phi && d_v_theta && d_coupling && d_phases && d_rx_dir && d_rx_field && d_rx_phase &&
                     d_rx_pol && d_tx_field && d_tx_phase && d_tx_pol && d_cluster_scale && d_order && d_a && batch > 0 &&
                     num_clusters > 0 && num_clusters <= kCdlMaxClusters && num_rx_ant > 0 && num_tx_ant > 0 &&
                     num_time_steps > 0 && sampling_frequency > 0.f && xpr_scale >= 0.f,
                 "sb_cdl_coefficients: bad arguments (1 <= num_clusters <= 24)");
    SB_CHECK_ARG((long long)num_rx_ant * num_tx_ant * num_clusters <= INT32_MAX,
                 "sb_cdl_coefficients: too many antenna pairs");
    CdlArgs p{d_speed, d_v_phi, d_v_theta, d_coupling, d_phases, d_rx_dir, d_rx_field, d_tx_field, d_cluster_scale,
              d_los_field, (const float2*)d_rx_phase, (const float2*)d_tx_phase, d_rx_pol, d_tx_pol, d_order, xpr_scale,
              wavenumber, sampling_frequency, (float2*)d_a, batch, num_clusters, num_rx_ant, num_tx_ant, num_time_steps};
    const size_t smem = cdl_smem_bytes(num_clusters);
    SB_CUDA(cudaFuncSetAttribute(cdl_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const long long ctas = batch * ((num_time_steps + kCdlTile - 1) / kCdlTile);
    cdl_kernel<<<sb_grid(ctas, 1, 16), kCdlThreads, smem, (cudaStream_t)stream>>>(p);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_phase_table(const float* d_tau, const float* d_x, float scale, int32_t mode, float* d_e, int64_t n_tab,
                              int32_t num_paths, int32_t num_cols, void* stream) {
    if (n_tab == 0) return SB_OK;
    SB_CHECK_ARG(d_tau && d_x && d_e && n_tab > 0 && num_paths > 0 && num_cols > 0 && (mode == 0 || mode == 1),
                 "sb_phase_table: bad arguments");
    const long long total = n_tab * num_paths * (long long)num_cols;
    phase_table_kernel<<<sb_grid(total, 256, 16), 256, 0, (cudaStream_t)stream>>>(d_tau, d_x, (float2*)d_e, n_tab,
                                                                                       num_paths, num_cols, scale, mode);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_cir_gram(const float* d_e, double* d_g, int64_t n_tab, int32_t num_paths, int32_t num_cols, void* stream) {
    if (n_tab == 0) return SB_OK;
    SB_CHECK_ARG(d_e && d_g && n_tab > 0 && num_paths > 0 && num_cols > 0, "sb_cir_gram: bad arguments");
    const long long warps = n_tab * num_paths * (long long)num_paths;
    cir_gram_kernel<<<sb_grid(warps, 8, 16), 256, 0, (cudaStream_t)stream>>>((const float2*)d_e, (double2*)d_g, n_tab,
                                                                                num_paths, num_cols);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

constexpr int kMaxCirPaths = 96;                   // sb_cir_apply and sb_cir_link_scale

static int check_dims(int64_t batch, int32_t rx, int32_t ra, int32_t tx, int32_t ta, int32_t p, int32_t t) {
    return batch > 0 && rx > 0 && ra > 0 && tx > 0 && ta > 0 && p > 0 && t > 0;
}

extern "C" int sb_cir_link_scale(const float* d_a, const double* d_g, int64_t g_link_stride, float* d_scale, int64_t batch,
                                 int32_t num_rx, int32_t num_rx_ant, int32_t num_tx, int32_t num_tx_ant, int32_t num_paths,
                                 int32_t num_time_steps, float denom, void* stream) {
    if (batch == 0) return SB_OK;
    SB_CHECK_ARG(d_a && d_g && d_scale && check_dims(batch, num_rx, num_rx_ant, num_tx, num_tx_ant, num_paths, num_time_steps) &&
                     g_link_stride >= 0 && denom > 0.f, "sb_cir_link_scale: bad arguments");
    SB_CHECK_ARG(num_paths <= kMaxCirPaths, "sb_cir_link_scale: more than 96 paths are not supported");
    CirDims d{batch, num_rx, num_rx_ant, num_tx, num_tx_ant, num_paths, num_time_steps};
    const long long links = batch * num_rx * (long long)num_tx;
    const size_t smem = sizeof(double2) * (size_t)num_paths * num_paths;     // 96 paths: 144 KB, opt-in above 48 KB
    if (smem > 48 * 1024)
        SB_CUDA(cudaFuncSetAttribute(cir_link_scale_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cir_link_scale_kernel<<<sb_grid(links, 1, 16), 256, smem, (cudaStream_t)stream>>>((const float2*)d_a, (const double2*)d_g,
                                                                                g_link_stride, d_scale, d, (double)denom);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_cir_apply(const float* d_a, const float* d_e, int64_t e_link_stride, const float* d_scale, float* d_h,
                            int64_t batch, int32_t num_rx, int32_t num_rx_ant, int32_t num_tx, int32_t num_tx_ant,
                            int32_t num_paths, int32_t num_time_steps, int32_t num_cols, void* stream) {
    if (batch == 0) return SB_OK;
    SB_CHECK_ARG(d_a && d_e && d_h && check_dims(batch, num_rx, num_rx_ant, num_tx, num_tx_ant, num_paths, num_time_steps) &&
                     num_cols > 0 && e_link_stride >= 0, "sb_cir_apply: bad arguments");
    CirDims d{batch, num_rx, num_rx_ant, num_tx, num_tx_ant, num_paths, num_time_steps};
    SB_CHECK_ARG(num_paths <= kMaxCirPaths, "sb_cir_apply: more than 96 paths are not supported");
    int rc;
    if (num_cols > 48)          // OFDM-like: wide rows
        rc = launch_cir_apply<16, 2, 256, 8>((const float2*)d_a, (const float2*)d_e, e_link_stride, d_scale, (float2*)d_h, d,
                                             num_cols, (cudaStream_t)stream);
    else                        // time-channel-like: a few taps, many time steps
        rc = launch_cir_apply<128, 8, 32, 2>((const float2*)d_a, (const float2*)d_e, e_link_stride, d_scale, (float2*)d_h, d,
                                             num_cols, (cudaStream_t)stream);
    if (rc) return rc;
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_spatial_corr(const float* d_in, const float* d_l, float* d_out, int64_t batch, int32_t n, int64_t cols,
                               void* stream) {
    if (batch == 0) return SB_OK;
    SB_CHECK_ARG(d_in && d_l && d_out && d_in != d_out && batch > 0 && n > 0 && n <= 128 && cols > 0,
                 "sb_spatial_corr: bad arguments (n <= 128, out of place)");
    const long long total = batch * cols;
    const size_t smem = sizeof(float2) * (size_t)n * n;
    if (smem > 48 * 1024) SB_CUDA(cudaFuncSetAttribute(spatial_corr_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    spatial_corr_kernel<<<sb_grid(total, 128, 16), 128, smem, (cudaStream_t)stream>>>((const float2*)d_in, (const float2*)d_l,
                                                                                          (float2*)d_out, batch, n, cols);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_apply_ofdm_channel(const float* d_x, const float* d_h, const float* d_no, int64_t no_inner, float* d_y,
                                     int64_t batch, int32_t num_rx_ant_total, int32_t num_tx_ant_total, int32_t num_re,
                                     int32_t add_noise, uint64_t seed, uint64_t offset, void* stream) {
    if (batch == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_x && d_h && d_y && batch >= 0 && num_rx_ant_total > 0 && num_tx_ant_total > 0 && num_re > 0 &&
                     (!add_noise || (d_no && no_inner >= 1)), "sb_apply_ofdm_channel: bad arguments");
    long long total = batch * num_rx_ant_total * (long long)num_re;
    if (total == 0) return SB_OK;
    const RowLaunch rl = row_launch(batch * num_rx_ant_total, num_re);
    apply_ofdm_channel_kernel<<<rl.grid, rl.block, 0, (cudaStream_t)stream>>>(
        (const float2*)d_x, (const float2*)d_h, d_no, no_inner > 0 ? no_inner : 1, (float2*)d_y, batch, num_rx_ant_total,
        num_tx_ant_total, num_re, add_noise, seed, offset);
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_apply_time_channel(const float* d_x, const float* d_h, const float* d_no, int64_t no_inner, float* d_y,
                                     int64_t batch, int32_t num_rx_ant_total, int32_t num_tx_ant_total,
                                     int32_t num_time_samples, int32_t l_tot, int32_t add_noise, uint64_t seed,
                                     uint64_t offset, void* stream) {
    if (batch == 0) return SB_OK;                         // empty batch: nothing to do, pointers may be null
    SB_CHECK_ARG(d_x && d_h && d_y && num_rx_ant_total > 0 && num_tx_ant_total > 0 && num_time_samples > 0 && l_tot > 0 &&
                     (!add_noise || (d_no && no_inner >= 1)), "sb_apply_time_channel: bad arguments");
    const RowLaunch rl = row_launch(batch * num_rx_ant_total, num_time_samples + l_tot - 1);
    apply_time_channel_kernel<<<rl.grid, rl.block, 0, (cudaStream_t)stream>>>(
        (const float2*)d_x, (const float2*)d_h, d_no, no_inner > 0 ? no_inner : 1, (float2*)d_y, batch, num_rx_ant_total,
        num_tx_ant_total, num_time_samples, l_tot, add_noise, seed, offset);
    SB_LAUNCH_CHECK();
    return SB_OK;
}
