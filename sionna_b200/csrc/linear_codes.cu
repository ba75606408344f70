// linear_codes.cu -- binary linear block codes: generator-matrix encoding (fec/linear/encoding.py:10-140) and ordered
// statistics decoding (fec/linear/decoding.py:14-478), DESIGN §3.13.
//
// Bit packing. A row of m bits is ceil(m / 32) 32-bit words; bit b of word w is column 32 w + b.
//
// Encoder. c = u G over GF(2): a CTA owns a tile of kEncRows codewords x 32 output words. It packs the codewords'
// information bits into shared memory kEncChunk bits at a time (one __ballot_sync per 32 bits), and every thread XORs
// the generator words of its output column selected by those bits into kEncRows / 8 accumulators. Rows of any width.
//
// OSD. One CTA per codeword (grid-stride over the batch):
//   1. |l| of the clipped LLRs is sorted descending by a bitonic sort of (~bits(|l|), index) keys, so equal |l| keep
//      the lower index first (stable).
//   2. The generator, held column-major by the code handle, is gathered into the sorted column order as bit-packed
//      rows in shared memory (one __ballot_sync per row word), then reduced column by column: a column becomes a pivot
//      iff some not yet pivoted row has a 1 there, and the lowest such row is XORed into every other row with a 1.
//      This keeps exactly the columns independent of those before them (the greedy basis), which is the set the
//      reference's row-wise pivot rule selects (tests/test_oracle_linear_codes.py).
//   3. Each row is compacted in place to its parity part P[i] (bits at the non-pivot columns, in sorted order).
//   4. A candidate flips the hard decisions at MRB positions e_1 < ... < e_t' (in reliability order) and re-encodes; its
//      discrepancy D = sum of |l| over the flipped positions + sum of |l| over the set bits of the parity residual
//      r = (p0 ^ hd_par) ^ P[e_1] ^ ... ^ P[e_t']. D orders candidates exactly as the reference's sum of softplus does.
//      The parity sum reads one 256-entry table per residual byte.
//   5. Order t' candidates are ranked in itertools.combinations order; each thread takes a contiguous range of ranks,
//      unranks its first one and then steps the last index, one row XOR per candidate. A prefix whose flipped sum
//      already exceeds the thread's best D is skipped: none of its candidates can win or tie.
//   6. The minimum of (D, order, rank) over the CTA wins, so ties keep the first candidate in enumeration order. Every
//      candidate's D is summed in a fixed order, so the output depends on nothing but the codeword's LLRs.
#include "sb_common.h"
#include <math.h>
#include <stdint.h>
#include <vector>

struct sb_osd_code {
    int k = 0, n = 0, wk = 0;
    std::vector<uint32_t> h;   // column-major: n columns of wk words, bit b of word q = G[32 q + b][column]
    mutable DeviceTables tables;   // device copies of h
};

namespace {

constexpr int kEncRows = 64;            // codewords per encoder CTA
constexpr int kEncChunk = 256;          // information bits packed per pass
constexpr int kOsdThreads = 256;
constexpr int kOsdMaxN = 1024;
constexpr int kOsdMaxOrder = 64;
constexpr float kLlrMax = 100.f;
constexpr unsigned kFull = 0xffffffffu;

template <typename T>
__device__ __forceinline__ unsigned bit_of(T v) { return (unsigned)((long long)v & 1); }

template <typename T>
__global__ void __launch_bounds__(256) gf2_encode_kernel(const T* __restrict__ u, T* __restrict__ c,
                                                         const uint32_t* __restrict__ g, long long batch, int k, int n,
                                                         int wn) {
    __shared__ uint32_t sU[kEncRows][kEncChunk / 32];
    __shared__ uint32_t sOut[kEncRows][33];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    constexpr int R = kEncRows / 8;                                    // codewords per thread
    const int w = blockIdx.x * 32 + lane;                              // output word of this thread
    for (long long tile = blockIdx.y; tile * kEncRows < batch; tile += gridDim.y) {
        const long long row0 = tile * kEncRows;
        uint32_t acc[R];
#pragma unroll
        for (int r = 0; r < R; ++r) acc[r] = 0u;
        for (int i0 = 0; i0 < k; i0 += kEncChunk) {
            __syncthreads();
            for (int r = warp; r < kEncRows; r += 8) {                 // pack: warp per codeword, one ballot per word
                const long long row = row0 + r;
                for (int q = 0; q < kEncChunk / 32; ++q) {
                    const int i = i0 + 32 * q + lane;
                    const unsigned b = (row < batch && i < k) ? bit_of(u[row * k + i]) : 0u;
                    const unsigned word = __ballot_sync(kFull, b);
                    if (lane == 0) sU[r][q] = word;
                }
            }
            __syncthreads();
            if (w < wn) {
                const int iend = min(kEncChunk, k - i0);
                for (int i = 0; i < iend; ++i) {
                    const uint32_t gw = __ldg(g + (size_t)(i0 + i) * wn + w);
#pragma unroll
                    for (int r = 0; r < R; ++r)
                        acc[r] ^= gw & (0u - ((sU[warp * R + r][i >> 5] >> (i & 31)) & 1u));
                }
            }
        }
#pragma unroll
        for (int r = 0; r < R; ++r) sOut[warp * R + r][lane] = acc[r];
        __syncthreads();
        const int col0 = blockIdx.x * 1024;
        const int cols = min(1024, n - col0);
        for (int e = threadIdx.x; e < kEncRows * cols; e += blockDim.x) {   // coalesced bit expansion
            const int r = e / cols, j = e - r * cols;
            const long long row = row0 + r;
            if (row < batch) c[row * n + col0 + j] = (T)((sOut[r][j >> 5] >> (j & 31)) & 1u);
        }
    }
}

// Shared-memory layout of the OSD kernel; every region is 8-byte aligned.
struct OsdLayout {
    int np, s, nbytes;
    size_t binom, lut, m, lsort, idx, a, row_of, mrb_pos, par_pos, flag, piv, total;
};

__host__ __device__ inline size_t al8(size_t x) { return (x + 7) & ~(size_t)7; }

__host__ __device__ inline OsdLayout osd_layout(int k, int n, int t, int wp) {
    OsdLayout L;
    L.np = 1;
    while (L.np < n) L.np <<= 1;
    const int wn = (n + 31) / 32;
    L.s = wn > wp ? wn : wp;
    if (!(L.s & 1)) L.s += 1;                                           // odd row stride: rows hit distinct banks
    L.nbytes = (n - k + 7) / 8;
    size_t o = 0;
    L.binom = o; o = al8(o + sizeof(unsigned long long) * (size_t)(k + 1) * (t + 1));
    const size_t lut = sizeof(float) * 256 * (size_t)L.nbytes, keys = sizeof(unsigned long long) * L.np;
    L.lut = o;   o = al8(o + (lut > keys ? lut : keys));
    L.m = o;     o = al8(o + sizeof(uint32_t) * (size_t)k * L.s);
    L.lsort = o; o = al8(o + sizeof(float) * n);
    L.idx = o;   o = al8(o + sizeof(int) * n);
    L.a = o;     o = al8(o + sizeof(float) * n);
    L.row_of = o; o = al8(o + sizeof(int) * k);
    L.mrb_pos = o; o = al8(o + sizeof(int) * k);
    L.par_pos = o; o = al8(o + sizeof(int) * (n - k + 1));
    L.flag = o;  o = al8(o + sizeof(unsigned char) * k * 2);           // row has the column's bit | row is pivoted
    L.piv = o;   o = al8(o + 64 * sizeof(uint32_t) + 8 * 32);           // pivot slots, residual words, reduction
    L.total = o;
    return L;
}

// First combination of rank r among the C(k, tt) combinations of 0 ... k - 1 in lexicographic order.
__device__ void unrank(unsigned long long r, int k, int tt, const unsigned long long* binom, int t1, int* e) {
    int x = 0;
    for (int i = 0; i < tt; ++i) {
        for (;; ++x) {
            const unsigned long long c = binom[(size_t)(k - 1 - x) * t1 + (tt - 1 - i)];
            if (r < c) break;
            r -= c;
        }
        e[i] = x++;
    }
}

template <int WP>
struct Residual {
    uint32_t w[WP];
};

template <int WP>
__device__ __forceinline__ float parity_sum(const Residual<WP>& r, const uint32_t* p, const float* lut, int nbytes,
                                            float d) {
#pragma unroll
    for (int w = 0; w < WP; ++w) {
        const uint32_t x = r.w[w] ^ p[w];
#pragma unroll
        for (int q = 0; q < 4; ++q)
            if (4 * w + q < nbytes) d += lut[(4 * w + q) * 256 + ((x >> (8 * q)) & 255u)];
    }
    return d;
}

template <int WP>
__global__ void __launch_bounds__(kOsdThreads) osd_kernel(const float* __restrict__ llr, float* __restrict__ out,
                                                          const uint32_t* __restrict__ gT, long long batch, int k,
                                                          int n, int t) {
    extern __shared__ __align__(16) unsigned char smem[];
    const OsdLayout L = osd_layout(k, n, t, WP);
    auto* sBinom = (unsigned long long*)(smem + L.binom);
    auto* sKey = (unsigned long long*)(smem + L.lut);                  // the sort keys share the table region
    auto* sLut = (float*)(smem + L.lut);
    auto* sM = (uint32_t*)(smem + L.m);
    auto* sL = (float*)(smem + L.lsort);
    auto* sIdx = (int*)(smem + L.idx);
    auto* sA = (float*)(smem + L.a);
    auto* sRowOf = (int*)(smem + L.row_of);
    auto* sMrbPos = (int*)(smem + L.mrb_pos);
    auto* sParPos = (int*)(smem + L.par_pos);
    auto* sFlag = (unsigned char*)(smem + L.flag);
    auto* sPivoted = sFlag + k;
    auto* sPiv = (int*)(smem + L.piv);                                  // [2] pivot slots, [2] winner (order, flag)
    auto* sRes = (uint32_t*)(smem + L.piv) + 32;                        // [32] residual words
    auto* sRedD = (float*)(smem + L.piv + 64 * sizeof(uint32_t));       // [8] per-warp best D
    auto* sRedO = (int*)(sRedD + 8);                                    // [8] per-warp best order
    auto* sRedR = (unsigned long long*)(sRedO + 8);                     // [8] per-warp best rank
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
    const int wk = (k + 31) / 32, wn = (n + 31) / 32, m = n - k, S = L.s, t1 = t + 1;

    for (int i = tid; i <= k; i += blockDim.x) {                        // C(i, j), exact while it fits 64 bits
        unsigned __int128 c = 1;
        sBinom[(size_t)i * t1] = 1;
        for (int j = 1; j <= t; ++j) {
            c = j > i ? 0 : c * (unsigned)(i - j + 1) / (unsigned)j;
            sBinom[(size_t)i * t1 + j] = (unsigned long long)c;
        }
    }

    for (long long cw = blockIdx.x; cw < batch; cw += gridDim.x) {
        const float* l = llr + cw * n;
        __syncthreads();
        for (int i = tid; i < L.np; i += blockDim.x) {
            unsigned long long key = ~0ull;
            if (i < n) {
                const float v = fminf(fmaxf(l[i], -kLlrMax), kLlrMax);
                sL[i] = v;
                key = ((unsigned long long)(~__float_as_uint(fabsf(v))) << 32) | (unsigned)i;
            }
            sKey[i] = key;
        }
        for (int size = 2; size <= L.np; size <<= 1) {                 // bitonic sort, ascending keys
            for (int stride = size >> 1; stride > 0; stride >>= 1) {
                __syncthreads();
                for (int i = tid; i < L.np / 2; i += blockDim.x) {
                    const int lo = 2 * i - (i & (stride - 1)), hi = lo + stride;
                    const bool up = (lo & size) == 0;
                    const unsigned long long a = sKey[lo], b = sKey[hi];
                    if ((a > b) == up) { sKey[lo] = b; sKey[hi] = a; }
                }
            }
        }
        __syncthreads();
        for (int j = tid; j < n; j += blockDim.x) {
            const int c = (int)(sKey[j] & 0xffffffffu);
            sIdx[j] = c;
            sA[j] = fabsf(sL[c]);
        }
        for (int i = tid; i < k; i += blockDim.x) sPivoted[i] = 0;
        if (tid < 2) sPiv[tid] = INT_MAX;
        __syncthreads();
        for (int w = warp; w < wn; w += nw) {                           // gather the generator in sorted column order
            const int j = 32 * w + lane;
            const uint32_t* col = j < n ? gT + (size_t)sIdx[j] * wk : nullptr;
            for (int q = 0; q < wk; ++q) {
                const uint32_t cw32 = col ? __ldg(col + q) : 0u;
                const int rows = min(32, k - 32 * q);
                uint32_t mine = 0;
                for (int b = 0; b < rows; ++b) {
                    const uint32_t word = __ballot_sync(kFull, (cw32 >> b) & 1u);
                    if (lane == b) mine = word;
                }
                if (lane < rows) sM[(size_t)(32 * q + lane) * S + w] = mine;
            }
        }
        __syncthreads();

        int rank = 0, npar = 0;
        for (int j = 0; j < n; ++j) {                                   // greedy basis, reduced row echelon form
            if (rank == k) {
                if (tid == 0) sParPos[npar] = j;
                ++npar;
                continue;
            }
            int* slot = sPiv + (j & 1);
            for (int r = tid; r < k; r += blockDim.x) {
                const unsigned b = (sM[(size_t)r * S + (j >> 5)] >> (j & 31)) & 1u;
                sFlag[r] = (unsigned char)b;
                if (b && !sPivoted[r]) atomicMin(slot, r);
            }
            __syncthreads();
            const int p = *slot;
            if (tid == 0) sPiv[(j + 1) & 1] = INT_MAX;
            if (p != INT_MAX) {
                for (int e = tid; e < k * wn; e += blockDim.x) {
                    const int r = e / wn, w = e - r * wn;
                    if (sFlag[r] && r != p) sM[(size_t)r * S + w] ^= sM[(size_t)p * S + w];
                }
                if (tid == 0) { sPivoted[p] = 1; sRowOf[rank] = p; sMrbPos[rank] = j; }
                ++rank;
            } else {
                if (tid == 0) sParPos[npar] = j;
                ++npar;
            }
            __syncthreads();
        }
        __syncthreads();                                                // parity positions written after rank == k
        for (int r = warp; r < k; r += nw) {                            // compact each row to its parity part
            uint32_t* row = sM + (size_t)r * S;
            uint32_t word = 0;
            if (lane < WP) {
                for (int b = 0; b < 32; ++b) {
                    const int q = 32 * lane + b;
                    if (q < m) word |= ((row[sParPos[q] >> 5] >> (sParPos[q] & 31)) & 1u) << b;
                }
            }
            __syncwarp();
            if (lane < WP) row[lane] = word;
            __syncwarp();
        }
        if (tid < 32) sRes[tid] = 0u;
        __syncthreads();
        {                                                               // residual of the order-0 word: p0 ^ hd_par
            Residual<WP> acc;
#pragma unroll
            for (int w = 0; w < WP; ++w) acc.w[w] = 0u;
            for (int i = tid; i < k; i += blockDim.x)
                if (sL[sIdx[sMrbPos[i]]] > 0.f) {
                    const uint32_t* p = sM + (size_t)sRowOf[i] * S;
#pragma unroll
                    for (int w = 0; w < WP; ++w) acc.w[w] ^= p[w];
                }
            for (int q = tid; q < m; q += blockDim.x)
                if (sL[sIdx[sParPos[q]]] > 0.f) atomicXor(sRes + (q >> 5), 1u << (q & 31));
#pragma unroll
            for (int w = 0; w < WP; ++w)
                if (acc.w[w]) atomicXor(sRes + w, acc.w[w]);
        }
        for (int e = tid; e < 256 * L.nbytes; e += blockDim.x) {        // per-byte parity weight tables
            const int byte = e >> 8, v = e & 255;
            float s = 0.f;
            for (int b = 0; b < 8; ++b)
                if (((v >> b) & 1) && 8 * byte + b < m) s += sA[sParPos[8 * byte + b]];
            sLut[e] = s;
        }
        __syncthreads();

        Residual<WP> r0;
#pragma unroll
        for (int w = 0; w < WP; ++w) r0.w[w] = sRes[w];
        float bestD;
        {
            uint32_t zero[WP];
#pragma unroll
            for (int w = 0; w < WP; ++w) zero[w] = 0u;
            bestD = parity_sum<WP>(r0, zero, sLut, L.nbytes, 0.f);
        }
        int bestO = 0;
        unsigned long long bestR = 0;
        int e[kOsdMaxOrder];
        for (int tt = 1; tt <= t; ++tt) {
            const unsigned long long total = sBinom[(size_t)k * t1 + tt];
            const unsigned long long per = (total + blockDim.x - 1) / blockDim.x;
            unsigned long long rk = per * tid;
            const unsigned long long end = min(total, rk + per);
            if (rk >= end) continue;
            unrank(rk, k, tt, sBinom, t1, e);
            Residual<WP> pr;
            float pre = 0.f;
            int last = e[tt - 1];
            auto load_prefix = [&]() {
                pr = r0;
                pre = 0.f;
                for (int i = 0; i < tt - 1; ++i) {
                    const uint32_t* p = sM + (size_t)sRowOf[e[i]] * S;
#pragma unroll
                    for (int w = 0; w < WP; ++w) pr.w[w] ^= p[w];
                    pre += sA[sMrbPos[e[i]]];
                }
                last = e[tt - 1];
            };
            auto next_prefix = [&]() {
                int i = tt - 2;
                while (i >= 0 && e[i] == k - tt + i) --i;
                ++e[i];
                for (int j = i + 1; j < tt; ++j) e[j] = e[j - 1] + 1;
                load_prefix();
            };
            load_prefix();
            while (rk < end) {
                if (pre > bestD) {                                      // every candidate of this prefix is worse
                    rk += (unsigned long long)(k - last);
                    if (rk >= end) break;
                    next_prefix();
                    continue;
                }
                const float d = parity_sum<WP>(pr, sM + (size_t)sRowOf[last] * S, sLut, L.nbytes,
                                               pre + sA[sMrbPos[last]]);
                if (d < bestD) { bestD = d; bestO = tt; bestR = rk; }
                ++rk;
                if (++last == k && rk < end) next_prefix();
            }
        }
        // (D, order, rank) minimum over the CTA
        for (int off = 16; off > 0; off >>= 1) {
            const float d2 = __shfl_down_sync(kFull, bestD, off);
            const int o2 = __shfl_down_sync(kFull, bestO, off);
            const unsigned long long r2 = __shfl_down_sync(kFull, bestR, off);
            if (d2 < bestD || (d2 == bestD && (o2 < bestO || (o2 == bestO && r2 < bestR)))) {
                bestD = d2; bestO = o2; bestR = r2;
            }
        }
        if (lane == 0) { sRedD[warp] = bestD; sRedO[warp] = bestO; sRedR[warp] = bestR; }
        __syncthreads();
        if (tid == 0) {
            for (int w = 1; w < nw; ++w) {
                const float d2 = sRedD[w];
                const int o2 = sRedO[w];
                const unsigned long long r2 = sRedR[w];
                if (d2 < bestD || (d2 == bestD && (o2 < bestO || (o2 == bestO && r2 < bestR)))) {
                    bestD = d2; bestO = o2; bestR = r2;
                }
            }
            for (int i = 0; i < k; ++i) sFlag[i] = 0;
            if (bestO > 0) {
                unrank(bestR, k, bestO, sBinom, t1, e);
                for (int i = 0; i < bestO; ++i) {
                    sFlag[e[i]] = 1;
                    const uint32_t* p = sM + (size_t)sRowOf[e[i]] * S;
                    for (int w = 0; w < WP; ++w) sRes[w] ^= p[w];
                }
            }
        }
        __syncthreads();
        float* o = out + cw * n;
        for (int i = tid; i < k; i += blockDim.x) {
            const int c = sIdx[sMrbPos[i]];
            o[c] = (float)((sL[c] > 0.f) ^ sFlag[i]);
        }
        for (int q = tid; q < m; q += blockDim.x) {
            const int c = sIdx[sParPos[q]];
            o[c] = (float)((sL[c] > 0.f) ^ ((sRes[q >> 5] >> (q & 31)) & 1u));
        }
    }
}

int osd_wp_bucket(int m) {
    const int words = (m + 31) / 32;
    int wp = 1;
    while (wp < words) wp <<= 1;
    return wp;
}

// Number of candidates of orders 1 ... t, or 0 when it exceeds 2^62.
unsigned long long osd_candidates(int k, int t) {
    unsigned long long sum = 0;
    unsigned __int128 c = 1;
    for (int j = 1; j <= t; ++j) {
        c = c * (unsigned)(k - j + 1) / (unsigned)j;
        if (c > ((unsigned __int128)1 << 62)) return 0;
        sum += (unsigned long long)c;
        if (sum > (1ull << 62)) return 0;
    }
    return sum;
}

}  // namespace

extern "C" int sb_gf2_encode(const void* d_u, void* d_c, int32_t dtype, int64_t batch, int32_t k, int32_t n,
                             const uint32_t* d_gen_rows, void* stream) {
    SB_CHECK_ARG(k >= 1 && n >= k && batch >= 0, "sb_gf2_encode: bad shape (1 <= k <= n, batch >= 0)");
    SB_CHECK_ARG(dtype >= 0 && dtype <= 3, "sb_gf2_encode: dtype = %d, supported are 0 float32, 1 float64, 2 int32, "
                 "3 int64", dtype);
    if (batch == 0) return SB_OK;
    SB_CHECK_ARG(d_u && d_c && d_gen_rows, "sb_gf2_encode: missing input, output or generator rows");
    const int wn = (n + 31) / 32;
    const dim3 grid((unsigned)((wn + 31) / 32),
                    (unsigned)std::min<long long>((batch + kEncRows - 1) / kEncRows, 65535));
    cudaStream_t st = (cudaStream_t)stream;
    switch (dtype) {
        case 0: gf2_encode_kernel<float><<<grid, 256, 0, st>>>((const float*)d_u, (float*)d_c, d_gen_rows, batch, k, n, wn); break;
        case 1: gf2_encode_kernel<double><<<grid, 256, 0, st>>>((const double*)d_u, (double*)d_c, d_gen_rows, batch, k, n, wn); break;
        case 2: gf2_encode_kernel<int32_t><<<grid, 256, 0, st>>>((const int32_t*)d_u, (int32_t*)d_c, d_gen_rows, batch, k, n, wn); break;
        default: gf2_encode_kernel<int64_t><<<grid, 256, 0, st>>>((const int64_t*)d_u, (int64_t*)d_c, d_gen_rows, batch, k, n, wn); break;
    }
    SB_LAUNCH_CHECK();
    return SB_OK;
}

extern "C" int sb_osd_code_create(sb_osd_code** out, const uint8_t* h_gm, int32_t k, int32_t n) {
    const char* who = "sb_osd_code_create";
    SB_CHECK_ARG(out && h_gm && k >= 1 && n >= k, "%s: bad arguments (out and h_gm given, 1 <= k <= n)", who);
    if (n > kOsdMaxN) {
        sb_set_error("%s: n = %d, supported are n <= %d", who, n, kOsdMaxN);
        return SB_EUNSUPPORTED;
    }
    const int wk = (k + 31) / 32, wn = (n + 31) / 32;
    std::vector<uint32_t> rows((size_t)k * wn, 0u);
    for (int r = 0; r < k; ++r)
        for (int c = 0; c < n; ++c) {
            const uint8_t v = h_gm[(size_t)r * n + c];
            SB_CHECK_ARG(v <= 1, "%s: h_gm[%d, %d] = %d is not binary", who, r, c, (int)v);
            if (v) rows[(size_t)r * wn + c / 32] |= 1u << (c & 31);
        }
    std::vector<uint32_t> ech(rows);                                    // rank over GF(2)
    int rank = 0;
    for (int c = 0; c < n && rank < k; ++c) {
        int p = -1;
        for (int r = rank; r < k && p < 0; ++r)
            if ((ech[(size_t)r * wn + c / 32] >> (c & 31)) & 1u) p = r;
        if (p < 0) continue;
        for (int w = 0; w < wn; ++w) std::swap(ech[(size_t)p * wn + w], ech[(size_t)rank * wn + w]);
        for (int r = 0; r < k; ++r)
            if (r != rank && ((ech[(size_t)r * wn + c / 32] >> (c & 31)) & 1u))
                for (int w = 0; w < wn; ++w) ech[(size_t)r * wn + w] ^= ech[(size_t)rank * wn + w];
        ++rank;
    }
    SB_CHECK_ARG(rank == k, "%s: the generator matrix is not full rank (rank %d < k = %d)", who, rank, k);
    auto* p = new sb_osd_code();
    p->k = k;
    p->n = n;
    p->wk = wk;
    p->h.assign((size_t)n * wk, 0u);
    for (int r = 0; r < k; ++r)
        for (int c = 0; c < n; ++c)
            if (h_gm[(size_t)r * n + c]) p->h[(size_t)c * wk + r / 32] |= 1u << (r & 31);
    p->tables.set(p->h);
    *out = p;
    return SB_OK;
}

extern "C" void sb_osd_code_destroy(sb_osd_code* p) { delete p; }

extern "C" int sb_osd_decode(const sb_osd_code* code, const float* d_llr, float* d_out, int64_t batch, int32_t t,
                             void* stream) {
    const char* who = "sb_osd_decode";
    SB_CHECK_ARG(code && batch >= 0 && t >= 0, "%s: bad arguments (code given, batch >= 0, t >= 0)", who);
    const int k = code->k, n = code->n;
    const int tt = std::min(t, k);
    if (tt > kOsdMaxOrder || (tt > 0 && osd_candidates(k, tt) == 0)) {
        sb_set_error("%s: order %d over k = %d needs more than 2^62 candidates (or order > %d)", who, tt, k,
                     kOsdMaxOrder);
        return SB_EUNSUPPORTED;
    }
    const int wp = osd_wp_bucket(n - k);
    const size_t smem = osd_layout(k, n, tt, wp).total;
    if (smem > 227 * 1024) {
        sb_set_error("%s: k = %d, n = %d, t = %d needs %zu bytes of shared memory, at most %d are available", who, k, n,
                     tt, smem, 227 * 1024);
        return SB_EUNSUPPORTED;
    }
    if (batch == 0) return SB_OK;
    SB_CHECK_ARG(d_llr && d_out, "%s: missing input or output", who);
    const DeviceTables::Copy* d = nullptr;
    const int rc = code->tables.get(&d);
    if (rc) return rc;
    const int grid = sb_grid(batch, 1, 16);
    return sb_dispatch<0, 5>(__builtin_ctz((unsigned)wp), [&](auto LW) {
        auto kern = osd_kernel<(1 << LW)>;
        if (smem > 48 * 1024) SB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        kern<<<grid, kOsdThreads, smem, (cudaStream_t)stream>>>(d_llr, d_out, d->at<uint32_t>(0), batch, k, n, tt);
        SB_LAUNCH_CHECK();
        return SB_OK;
    });
}
