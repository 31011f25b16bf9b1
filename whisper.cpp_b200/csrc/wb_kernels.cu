// wb_kernels.cu -- the bandwidth-bound kernels of the encode/decode path (everything that is not a wgmma GEMM).
// Each kernel cites the reference lines whose arithmetic it reproduces.
#include <cmath>
#include <mutex>
#include <vector>
#include "wb_kernels.cuh"
#include "wb_common.h"
#include "wb_dev.cuh"

namespace wb {

// =====================================================================================================================
//  small utilities
// =====================================================================================================================
// warp_sum / warp_max / block_sum / block_max / gelu_ref_f16 / mma wrappers: wb_dev.cuh

// =====================================================================================================================
//  conversions / re-layout
// =====================================================================================================================
__global__ void k_f32_to_f16(const float * __restrict__ s, __half * __restrict__ d, int64_t n) {
    int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t) gridDim.x * blockDim.x;
    for (; i < n; i += stride) d[i] = __float2half_rn(s[i]);
}
__global__ void k_f16_to_f32(const __half * __restrict__ s, float * __restrict__ d, int64_t n) {
    int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t) gridDim.x * blockDim.x;
    for (; i < n; i += stride) d[i] = __half2float(s[i]);
}
static inline int grid_for(int64_t n, int tpb) { int64_t b = (n + tpb - 1) / tpb; return (int) (b < 132 * 16 ? (b > 0 ? b : 1) : 132 * 16); }
void f32_to_f16(const float * src, __half * dst, int64_t n, cudaStream_t st) {
    if (n <= 0) return;
    k_f32_to_f16<<<grid_for(n, 256), 256, 0, st>>>(src, dst, n); count_launch();
}
void f16_to_f32(const __half * src, float * dst, int64_t n, cudaStream_t st) {
    if (n <= 0) return;
    k_f16_to_f32<<<grid_for(n, 256), 256, 0, st>>>(src, dst, n); count_launch();
}

// one thread per 32-block: gather the unaligned file block with byte loads, scatter to the planar arrays
template <int WT>
__global__ void k_repack32(const uint8_t * __restrict__ src, uint8_t * __restrict__ qs, uint32_t * __restrict__ qh,
                           __half * __restrict__ d, __half * __restrict__ m, int64_t nblk) {
    constexpr int BS = (WT == WT_Q4_0) ? 18 : (WT == WT_Q5_0 ? 22 : (WT == WT_Q4_1 ? 20 : (WT == WT_Q5_1 ? 24 : 34)));
    constexpr int QS = (WT == WT_Q8_0) ? 32 : 16;
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nblk) return;
    const uint8_t * b = src + i * BS;
    d[i] = __ushort_as_half((unsigned short) ((uint16_t) b[0] | ((uint16_t) b[1] << 8)));
    int off = 2;
    if (wt_has_min(WT)) { m[i] = __ushort_as_half((unsigned short) ((uint16_t) b[2] | ((uint16_t) b[3] << 8))); off = 4; }
    if (wt_has_qh(WT)) { qh[i] = (uint32_t) b[off] | ((uint32_t) b[off + 1] << 8) | ((uint32_t) b[off + 2] << 16) | ((uint32_t) b[off + 3] << 24); off += 4; }
    for (int j = 0; j < QS; ++j) qs[i * QS + j] = b[off + j];
}
bool repack_block32_into(int wtype, const uint8_t * src, const QMat & dst, int rows, int K, cudaStream_t st) {
    const int64_t nblk = (int64_t) rows * (K / 32);
    if (nblk == 0) return true;
    const int blocks = (int) ((nblk + 255) / 256);
    uint8_t * qs = const_cast<uint8_t *>(dst.qs); uint32_t * qh = const_cast<uint32_t *>(dst.qh); __half * d = const_cast<__half *>(dst.d);
    __half * m = const_cast<__half *>(dst.m);
    switch (wtype) {
        case WT_Q4_0: k_repack32<WT_Q4_0><<<blocks, 256, 0, st>>>(src, qs, qh, d, m, nblk); break;
        case WT_Q4_1: k_repack32<WT_Q4_1><<<blocks, 256, 0, st>>>(src, qs, qh, d, m, nblk); break;
        case WT_Q5_0: k_repack32<WT_Q5_0><<<blocks, 256, 0, st>>>(src, qs, qh, d, m, nblk); break;
        case WT_Q5_1: k_repack32<WT_Q5_1><<<blocks, 256, 0, st>>>(src, qs, qh, d, m, nblk); break;
        case WT_Q8_0: k_repack32<WT_Q8_0><<<blocks, 256, 0, st>>>(src, qs, qh, d, m, nblk); break;
        default: set_error("repack_block32: bad type %d", wtype); return false;
    }
    count_launch();
    return cudaGetLastError() == cudaSuccess;
}
bool repack_block32(int wtype, const uint8_t * src, uint8_t * dst, int N, int K, QMat * out, cudaStream_t st) {
    const int64_t nblk = (int64_t) N * (K / 32);
    out->type = wtype; out->N = N; out->K = K; out->base = nullptr;
    out->qs = dst;
    uint8_t * p = dst + nblk * wt_qs_bytes(wtype);
    out->qh = nullptr; out->m = nullptr;
    if (wt_has_qh(wtype)) { out->qh = reinterpret_cast<uint32_t *>(p); p += nblk * 4; }
    if (wt_has_min(wtype)) { out->m = reinterpret_cast<__half *>(p); p += nblk * 2; }
    out->d = reinterpret_cast<__half *>(p);
    return repack_block32_into(wtype, src, *out, N, K, st);
}

// tile-major records (wb_quant.cuh): one thread per (tile, record, lane)
template <int WT>
__global__ void k_repack_tm(const uint8_t * __restrict__ src, uint8_t * __restrict__ dst, int rows, int K, int64_t n_threads) {
    constexpr int BS = (WT == WT_Q4_0) ? 18 : (WT == WT_Q5_0 ? 22 : (WT == WT_Q4_1 ? 20 : (WT == WT_Q5_1 ? 24 : (WT == WT_Q8_0 ? 34 : 0))));
    const int REC = wt_tm_rec_bytes(WT), nrec = K / wt_tm_rec_k(WT);
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_threads) return;
    const int lane = (int) (i & 31), g = lane >> 2, c = lane & 3;
    const int64_t rb = i >> 5;
    const int b = (int) (rb % nrec);
    const int64_t tile = rb / nrec;
    uint8_t * rec = dst + (tile * nrec + b) * REC;
    const int64_t r0 = tile * 16 + g, r1 = r0 + 8;
    if (WT == WT_F16) {
        const __half * h = reinterpret_cast<const __half *>(src);
        uint32_t w[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int64_t r = (k & 1) ? r1 : r0;
            const int col = b * 16 + 2 * c + ((k >> 1) ? 8 : 0);
            const unsigned short lo = r < rows ? __half_as_ushort(h[r * K + col]) : 0, hi = r < rows ? __half_as_ushort(h[r * K + col + 1]) : 0;
            w[k] = (uint32_t) lo | ((uint32_t) hi << 16);
        }
        reinterpret_cast<uint4 *>(rec)[lane] = make_uint4(w[0], w[1], w[2], w[3]);
        return;
    }
    const uint8_t * b0 = src + (r0 * nrec + b) * BS, * b1 = src + (r1 * nrec + b) * BS;
    const int qoff = (WT == WT_Q5_0) ? 6 : (WT == WT_Q4_1 ? 4 : (WT == WT_Q5_1 ? 8 : 2));
    auto word = [&](const uint8_t * blk, int64_t r, int wi) -> uint32_t {
        if (r >= rows) return 0u;
        const uint8_t * q = blk + qoff + 4 * wi;
        return (uint32_t) q[0] | ((uint32_t) q[1] << 8) | ((uint32_t) q[2] << 16) | ((uint32_t) q[3] << 24);
    };
    if (WT == WT_Q8_0) reinterpret_cast<uint4 *>(rec)[lane] = make_uint4(word(b0, r0, c), word(b1, r1, c), word(b0, r0, 4 + c), word(b1, r1, 4 + c));
    else               reinterpret_cast<uint2 *>(rec)[lane] = make_uint2(word(b0, r0, c), word(b1, r1, c));
    if (c == 0) {                                                // lanes 0,4,..: the per-row fields of rows g and g+8
        auto d16 = [&](const uint8_t * blk, int64_t r) -> uint32_t { return r < rows ? ((uint32_t) blk[0] | ((uint32_t) blk[1] << 8)) : 0u; };
        if (wt_has_min(WT)) {                                    // Q4_1 / Q5_1: file block d, m, (qh), qs
            auto m16 = [&](const uint8_t * blk, int64_t r) -> uint32_t { return r < rows ? ((uint32_t) blk[2] | ((uint32_t) blk[3] << 8)) : 0u; };
            if (WT == WT_Q5_1) {
                auto h32 = [&](const uint8_t * blk, int64_t r) -> uint32_t { return r < rows ? ((uint32_t) blk[4] | ((uint32_t) blk[5] << 8) | ((uint32_t) blk[6] << 16) | ((uint32_t) blk[7] << 24)) : 0u; };
                reinterpret_cast<uint2 *>(rec + wt_tm_qs_bytes(WT))[g] = make_uint2(h32(b0, r0), h32(b1, r1));
            }
            reinterpret_cast<uint2 *>(rec + wt_tm_d_off(WT))[g] = make_uint2(d16(b0, r0) | (d16(b1, r1) << 16), m16(b0, r0) | (m16(b1, r1) << 16));
        } else if (WT == WT_Q5_0) {
            auto h32 = [&](const uint8_t * blk, int64_t r) -> uint32_t { return r < rows ? ((uint32_t) blk[2] | ((uint32_t) blk[3] << 8) | ((uint32_t) blk[4] << 16) | ((uint32_t) blk[5] << 24)) : 0u; };
            reinterpret_cast<uint2 *>(rec + wt_tm_qs_bytes(WT))[g] = make_uint2(h32(b0, r0), h32(b1, r1));
            reinterpret_cast<uint32_t *>(rec + wt_tm_d_off(WT))[g] = d16(b0, r0) | (d16(b1, r1) << 16);
        } else {
            reinterpret_cast<uint32_t *>(rec + wt_tm_d_off(WT))[g] = d16(b0, r0) | (d16(b1, r1) << 16);
        }
    }
}
// K-quant tile-major records (wb_quant.cuh): one thread per (tile, 32-value sub-block, lane); the lanes of sub-block 0 also copy
// the header (8 bytes each)
template <int WT>
__global__ void k_repack_tm_kq(const uint8_t * __restrict__ src, uint8_t * __restrict__ dst, int rows, int K, int64_t n_threads) {
    constexpr int BLK = (WT == WT_Q4_K) ? 144 : 176, QOFF = (WT == WT_Q4_K) ? 16 : 48;
    const int REC = wt_tm_rec_bytes(WT), nsub = K / 32, nsb = K / 256;
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_threads) return;
    const int lane = (int) (i & 31), g = lane >> 2, c = lane & 3;
    const int64_t rb = i >> 5;
    const int b = (int) (rb % nsub), sb = b >> 3, j = b & 7;
    const int64_t tile = rb / nsub;
    uint8_t * sbp = dst + (tile * nsb + sb) * REC;
    uint8_t * rec = sbp + wt_tm_sub_off(WT, j);
    const int64_t r0 = tile * 16 + g, r1 = r0 + 8;
    auto blk = [&](int64_t r) { return src + (r * nsb + sb) * BLK; };
    // bytes 4c .. 4c+3 of the row's 32 values in the Q4_0 order: byte i = q[i] | q[i + 16] << 4
    auto word = [&](int64_t r) -> uint32_t {
        if (r >= rows) return 0u;
        const uint8_t * q = blk(r) + QOFF + 32 * (j >> 1);
        const int sh = 4 * (j & 1);
        uint32_t w = 0;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int e = 4 * c + k;
            w |= ((uint32_t) (((q[e] >> sh) & 0xF) | (((q[e + 16] >> sh) & 0xF) << 4))) << (8 * k);
        }
        return w;
    };
    reinterpret_cast<uint2 *>(rec)[lane] = make_uint2(word(r0), word(r1));
    if (WT == WT_Q5_K && c == 0) {                               // fifth bits: bit e of the word = bit j of qh[e]
        auto hbits = [&](int64_t r) -> uint32_t {
            if (r >= rows) return 0u;
            const uint8_t * qh = blk(r) + 16;
            uint32_t h = 0;
            for (int e = 0; e < 32; ++e) h |= (uint32_t) ((qh[e] >> j) & 1) << e;
            return h;
        };
        reinterpret_cast<uint2 *>(rec + wt_tm_qs_bytes(WT))[g] = make_uint2(hbits(r0), hbits(r1));
    }
    if (j == 0) {                                                // header: 16 bytes (d, dmin, scales) of each of the 16 rows
        static_assert(WT_TM_KQ_HDR_ROW == 16, "two lanes per header row");
        const int64_t r = tile * 16 + (lane >> 1);
        uint32_t w[2] = { 0u, 0u };
        if (r < rows) memcpy(w, blk(r) + 8 * (lane & 1), 8);
        reinterpret_cast<uint2 *>(sbp)[lane] = make_uint2(w[0], w[1]);
    }
}

// Q3_K tile-major records (wb_quant.cuh): one thread per (tile, 32-value sub-block, lane); the lanes of sub-block 0 also write the
// header (scale words lane and lane + 32, d words of lanes 0 .. 7)
__global__ void k_repack_tm_q3k(const uint8_t * __restrict__ src, uint8_t * __restrict__ dst, int rows, int K, int64_t n_threads) {
    constexpr int BLK = 110;
    const int REC = wt_tm_rec_bytes(WT_Q3_K), nsub = K / 32, nsb = K / 256;
    const int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_threads) return;
    const int lane = (int) (i & 31), g = lane >> 2, c = lane & 3;
    const int64_t rb = i >> 5;
    const int b = (int) (rb % nsub), sb = b >> 3, j = b & 7;
    const int64_t tile = rb / nsub;
    uint8_t * sbp = dst + (tile * nsb + sb) * REC;
    uint8_t * rec = sbp + wt_tm_sub_off(WT_Q3_K, j);
    const int64_t r0 = tile * 16 + g, r1 = r0 + 8;
    auto blk = [&](int64_t r) { return src + (r * nsb + sb) * BLK; };
    // stored values q + 4 of values 32 j + v .. + 3 of row r; rows >= N: 0 (their scales are 0)
    auto uval4 = [&](int64_t r, int v) -> uint32_t { return r < rows ? __vadd4(q3k_q4(blk(r), 32 * j + v), 0x04040404u) : 0u; };
    // the lane's A registers: r = 0 / 1 rows g / g + 8 values 4c .., r = 2 / 3 values 16 + 4c ..
    const uint32_t u[4] = { uval4(r0, 4 * c), uval4(r1, 4 * c), uval4(r0, 16 + 4 * c), uval4(r1, 16 + 4 * c) };
    uint32_t lw = 0;
#pragma unroll
    for (int r = 0; r < 4; ++r) lw |= (u[r] & 0x03030303u) << (2 * r);
    reinterpret_cast<uint32_t *>(rec)[lane] = lw;
    if (c == 0) {                                                // high bits of the 32 values of rows g, g + 8 (bit v = value v)
        auto hbits = [&](int64_t r) -> uint32_t {
            uint32_t h = 0;
            for (int v = 0; v < 32; v += 4) h |= spread_bit2(uval4(r, v)) << v;
            return h;
        };
        reinterpret_cast<uint2 *>(rec + wt_tm_qs_bytes(WT_Q3_K))[g] = make_uint2(hbits(r0), hbits(r1));
    }
    if (j == 0) {                                                // header
        auto sc = [&](int64_t r, int is) -> uint32_t { return r < rows ? (uint32_t) (q3k_scale(blk(r), is) & 0xff) : 0u; };
#pragma unroll
        for (int k = 0; k < 2; ++k) {
            const int w = lane + 32 * k, jj = w >> 3, gg = w & 7;
            const int64_t ra = tile * 16 + gg, rb8 = ra + 8;
            reinterpret_cast<uint32_t *>(sbp)[w] = sc(ra, 2 * jj) | (sc(ra, 2 * jj + 1) << 8) | (sc(rb8, 2 * jj) << 16) | (sc(rb8, 2 * jj + 1) << 24);
        }
        if (lane < 8) {
            const int64_t ra = tile * 16 + lane, rb8 = ra + 8;
            reinterpret_cast<uint32_t *>(sbp + WT_TM_Q3K_D_OFF)[lane] = (ra < rows ? q3k_dbits(blk(ra)) : 0u) | ((rb8 < rows ? q3k_dbits(blk(rb8)) : 0u) << 16);
        }
    }
}

bool repack_tile_major(int wtype, const uint8_t * src, const QMat & dst, int row_off, int rows, cudaStream_t st) {
    if (dst.layout != 1 || (row_off & 15)) { set_error("repack_tile_major: bad destination"); return false; }
    const int K = dst.K, nrec = K / wt_tm_rec_k(wtype);
    if (wt_is_kquant(wtype)) {
        const int64_t n_threads = (int64_t) ((rows + 15) / 16) * (K / 32) * 32;
        if (n_threads == 0) return true;
        uint8_t * out = const_cast<uint8_t *>(reinterpret_cast<const uint8_t *>(dst.base)) + (size_t) (row_off / 16) * nrec * wt_tm_rec_bytes(wtype);
        const unsigned blocks = (unsigned) ((n_threads + 255) / 256);
        switch (wtype) {
            case WT_Q4_K: k_repack_tm_kq<WT_Q4_K><<<blocks, 256, 0, st>>>(src, out, rows, K, n_threads); break;
            case WT_Q5_K: k_repack_tm_kq<WT_Q5_K><<<blocks, 256, 0, st>>>(src, out, rows, K, n_threads); break;
            case WT_Q3_K: k_repack_tm_q3k<<<blocks, 256, 0, st>>>(src, out, rows, K, n_threads); break;
        }
        count_launch();
        return cudaGetLastError() == cudaSuccess;
    }
    const int64_t tiles = (rows + 15) / 16, n_threads = tiles * nrec * 32;
    if (n_threads == 0) return true;
    uint8_t * out = const_cast<uint8_t *>(reinterpret_cast<const uint8_t *>(dst.base)) + (size_t) (row_off / 16) * nrec * wt_tm_rec_bytes(wtype);
    const unsigned blocks = (unsigned) ((n_threads + 255) / 256);
    switch (wtype) {
        case WT_F16:  k_repack_tm<WT_F16><<<blocks, 256, 0, st>>>(src, out, rows, K, n_threads); break;
        case WT_Q4_0: k_repack_tm<WT_Q4_0><<<blocks, 256, 0, st>>>(src, out, rows, K, n_threads); break;
        case WT_Q5_0: k_repack_tm<WT_Q5_0><<<blocks, 256, 0, st>>>(src, out, rows, K, n_threads); break;
        case WT_Q4_1: k_repack_tm<WT_Q4_1><<<blocks, 256, 0, st>>>(src, out, rows, K, n_threads); break;
        case WT_Q5_1: k_repack_tm<WT_Q5_1><<<blocks, 256, 0, st>>>(src, out, rows, K, n_threads); break;
        case WT_Q8_0: k_repack_tm<WT_Q8_0><<<blocks, 256, 0, st>>>(src, out, rows, K, n_threads); break;
        default: set_error("repack_tile_major: bad type %d", wtype); return false;
    }
    count_launch();
    return cudaGetLastError() == cudaSuccess;
}

// =====================================================================================================================
//  log-mel spectrogram  (src/whisper.cpp:3005-3272)
// =====================================================================================================================
// Hann window and the 400-entry sin/cos table are evaluated on the HOST with the reference's own expressions
// (whisper.cpp:3023-3039) so they are bit-identical to the tables the CPU path uses; [0,400)=hann [400,800)=cos [800,1200)=sin
__constant__ float c_mel_tab[1200];

static void mel_tables_upload() {
    static std::mutex mu; static bool done[64] = { false };
    int dev = 0; cudaGetDevice(&dev);
    std::lock_guard<std::mutex> lk(mu);
    if (dev < 64 && done[dev]) return;
    std::vector<float> t(1200);
    for (int i = 0; i < 400; ++i) {
        t[i] = (float) (0.5 * (1.0 - cosf((float) ((2.0 * M_PI * i) / 400))));
        const double theta = (2 * M_PI * i) / 400;
        t[400 + i] = cosf((float) theta);
        t[800 + i] = sinf((float) theta);
    }
    cudaMemcpyToSymbol(c_mel_tab, t.data(), 1200 * sizeof(float));
    if (dev < 64) done[dev] = true;
}

__device__ __forceinline__ int float_order_key(float f) { int i = __float_as_int(f); return i >= 0 ? i : i ^ 0x7FFFFFFF; }
__device__ __forceinline__ float float_from_key(int k)  { return __int_as_float(k >= 0 ? k : k ^ 0x7FFFFFFF); }

__global__ void k_mel_init(int * gmax_key) { *gmax_key = float_order_key(-1e20f); }

// one block per frame
__global__ void __launch_bounds__(256)
k_mel_frames(const float * __restrict__ pcm, int N, const float * __restrict__ filt, int n_mel,
             float * __restrict__ mel, int n_len, int * __restrict__ gmax_key) {
    __shared__ float x[400];
    __shared__ float P[204];
    __shared__ float red[32];
    __shared__ float tc[400], ts[400];                          // twiddles in shared memory: the DFT indexes them divergently,
    const int i   = blockIdx.x;                                  // which a __constant__ array would serialise 32-way
    const int tid = threadIdx.x;
    const int n_eff  = N + 200;                               // samples handed to the worker: n_samples + stage_2_pad
    const int n_comp = min(n_eff / 160 + 1, n_len);           // frames that are really transformed (whisper.cpp:3125)
    if (i >= n_comp) {                                        // whisper.cpp:3168-3174
        for (int j = tid; j < n_mel; j += blockDim.x) mel[(int64_t) j * n_len + i] = -10.0f;
        if (tid == 0) atomicMax(gmax_key, float_order_key(-10.0f));
        return;
    }
    for (int j = tid; j < 400; j += blockDim.x) { tc[j] = c_mel_tab[400 + j]; ts[j] = c_mel_tab[800 + j]; }
    const int offset   = i * 160;
    const int n_reflect = min(200, max(0, N - 1));
    const int lim = min(400, n_eff - offset);
    for (int j = tid; j < 400; j += blockDim.x) {
        float s = 0.0f;
        if (j < lim) {
            const int idx = offset + j;                       // index into the padded signal
            if (idx < 200) { const int r = idx - (200 - n_reflect); s = (r >= 0) ? pcm[n_reflect - r] : 0.0f; }
            else if (idx < 200 + N) s = pcm[idx - 200];
            s = c_mel_tab[j] * s;
        }
        x[j] = s;
    }
    __syncthreads();
    if (tid < 201) {                                          // direct 400-point DFT bin `tid`
        float re = 0.0f, im = 0.0f;
        int idx = 0;
        for (int n = 0; n < 400; ++n) {
            const float v = x[n];
            re += v * tc[idx];
            im -= v * ts[idx];
            idx += tid; if (idx >= 400) idx -= 400;
        }
        P[tid] = re * re + im * im;
    }
    __syncthreads();
    float lmax = -1e20f;
    for (int j = tid; j < n_mel; j += blockDim.x) {
        const float * f = filt + (int64_t) j * 201;
        double sum = 0.0;
        int k = 0;
        for (; k < 201 - 3; k += 4) {                         // same grouping as whisper.cpp:3152-3158 (float inside, double outside)
            const float part = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(P[k], f[k]), __fmul_rn(P[k+1], f[k+1])), __fmul_rn(P[k+2], f[k+2])), __fmul_rn(P[k+3], f[k+3]));
            sum += part;
        }
        for (; k < 201; ++k) sum += __fmul_rn(P[k], f[k]);
        sum = log10(fmax(sum, 1e-10));
        const float v = (float) sum;
        mel[(int64_t) j * n_len + i] = v;
        lmax = fmaxf(lmax, v);
    }
    lmax = block_max(lmax, red);
    if (tid == 0) atomicMax(gmax_key, float_order_key(lmax));
}

__global__ void k_mel_norm(float * __restrict__ mel, int64_t n, const int * __restrict__ gmax_key) {
    const double mmax = (double) float_from_key(*gmax_key) - 8.0;     // whisper.cpp:3240-3256
    int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    const int64_t stride = (int64_t) gridDim.x * blockDim.x;
    for (; i < n; i += stride) {
        float v = mel[i];
        if ((double) v < mmax) v = (float) mmax;
        mel[i] = (float) (((double) v + 4.0) / 4.0);
    }
}

void mel_spectrogram(const float * pcm, int n_samples, const float * filters, int n_mel, float * mel, int n_len,
                     float * gmax_scratch, cudaStream_t st) {
    mel_tables_upload();
    int * key = reinterpret_cast<int *>(gmax_scratch);
    k_mel_init<<<1, 1, 0, st>>>(key);
    k_mel_frames<<<n_len, 256, 0, st>>>(pcm, n_samples, filters, n_mel, mel, n_len, key);
    const int64_t n = (int64_t) n_mel * n_len;
    k_mel_norm<<<grid_for(n, 256), 256, 0, st>>>(mel, n, key);
    count_launch(3);
}

__global__ void k_mel_window(const float * __restrict__ mel, int n_len, int n_mel, int seek, int n_frames, __half * __restrict__ out) {
    // out[r][j], r in [0, n_frames+2): tile transpose through shared memory (mel is mel-major, out is time-major)
    __shared__ float tile[32][33];
    const int t0 = blockIdx.x * 32, j0 = blockIdx.y * 32;
    for (int dj = threadIdx.y; dj < 32; dj += blockDim.y) {
        const int j = j0 + dj, t = t0 + threadIdx.x;
        float v = 0.0f;
        if (j < n_mel && t < n_frames && seek + t < n_len && seek + t >= 0) v = mel[(int64_t) j * n_len + seek + t];
        tile[dj][threadIdx.x] = v;
    }
    __syncthreads();
    for (int dt = threadIdx.y; dt < 32; dt += blockDim.y) {
        const int t = t0 + dt, j = j0 + threadIdx.x;
        if (t < n_frames && j < n_mel) out[(int64_t) (t + 1) * n_mel + j] = __float2half_rn(tile[threadIdx.x][dt]);
    }
}
__global__ void k_zero_rows2(__half * out, int n_mel, int n_frames) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j < n_mel) { out[j] = __float2half(0.0f); out[(int64_t) (n_frames + 1) * n_mel + j] = __float2half(0.0f); }
}
void mel_window_f16(const float * mel, int n_len, int n_mel, int seek, int n_frames, __half * out, cudaStream_t st) {
    dim3 grid((n_frames + 31) / 32, (n_mel + 31) / 32), block(32, 8);
    k_mel_window<<<grid, block, 0, st>>>(mel, n_len, n_mel, seek, n_frames, out);
    k_zero_rows2<<<(n_mel + 127) / 128, 128, 0, st>>>(out, n_mel, n_frames);
    count_launch(2);
}

// =====================================================================================================================
//  LayerNorm: two-pass statistics, then (x-mean)*rstd*w + b   (ggml-cpu/ops.cpp:3698-3765; whisper.cpp:2108-2115)
// =====================================================================================================================
__global__ void __launch_bounds__(256)
k_layernorm(const float * __restrict__ x, const float * __restrict__ w, const float * __restrict__ b, float eps,
            int rows, int d, __half * __restrict__ o16, float * __restrict__ o32) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= rows) return;
    const float * xr = x + (int64_t) warp * d;
    float s = 0.0f;
    for (int i = lane; i < d; i += 32) s += xr[i];
    const float mean = warp_sum(s) / d;
    float v = 0.0f;
    for (int i = lane; i < d; i += 32) { const float t = xr[i] - mean; v += t * t; }
    const float var = warp_sum(v) / d;
    const float rstd = 1.0f / sqrtf(var + eps);
    for (int i = lane; i < d; i += 32) {
        const float y = __fadd_rn(__fmul_rn(__fmul_rn(xr[i] - mean, rstd), w[i]), b[i]);
        if (o16) o16[(int64_t) warp * d + i] = __float2half_rn(y);
        if (o32) o32[(int64_t) warp * d + i] = y;
    }
}
void layernorm(const float * x, const float * w, const float * b, float eps, int rows, int d, __half * o16, float * o32, cudaStream_t st) {
    if (rows <= 0) return;
    const int blocks = (rows * 32 + 255) / 256;
    k_layernorm<<<blocks, 256, 0, st>>>(x, w, b, eps, rows, d, o16, o32); count_launch();
}

// =====================================================================================================================
//  row softmax for the unfused attention path (scores are already scaled)
// =====================================================================================================================
__global__ void __launch_bounds__(256)
k_softmax_rows(const float * __restrict__ s, __half * __restrict__ p, int64_t rows, int cols) {
    const int64_t row = ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    const float * sr = s + row * cols;
    float m = -INFINITY;
    for (int i = lane; i < cols; i += 32) m = fmaxf(m, sr[i]);
    m = warp_max(m);
    float sum = 0.0f;
    for (int i = lane; i < cols; i += 32) sum += expf(sr[i] - m);
    sum = warp_sum(sum);
    const float inv = 1.0f / sum;
    for (int i = lane; i < cols; i += 32) p[row * cols + i] = __float2half_rn(expf(sr[i] - m) * inv);
}
void softmax_rows_f16(const float * s, __half * p, int64_t rows, int cols, cudaStream_t st) {
    if (rows <= 0) return;
    const int64_t blocks = (rows * 32 + 255) / 256;
    k_softmax_rows<<<(unsigned) blocks, 256, 0, st>>>(s, p, rows, cols); count_launch();
}

// =====================================================================================================================
//  decoder: token + position embedding (get_rows on the quantised table is an exact f32 dequantisation,
//  ggml-cpu/ops.cpp:4850 -> ggml-quants.c dequantize_row_*)
// =====================================================================================================================
__device__ __forceinline__ float dequant_elem_tm(const QMat & W, int64_t row, int e) {     // tile-major records (wb_quant.cuh)
    const int REC = wt_tm_rec_bytes(W.type), rk = wt_tm_rec_k(W.type), nrec = W.K / rk;
    const int rr = (int) (row & 15), g = rr & 7, up = rr >> 3, i = e % rk;
    const uint8_t * rec = reinterpret_cast<const uint8_t *>(W.base) + ((row >> 4) * nrec + e / rk) * REC;
    if (W.type == WT_Q3_K) {                                     // dequantize_row_q3_K: (d * sc) * q, each product rounded
        const int j = i >> 5, l = i & 31, hf = l >> 4, c = (l & 15) >> 2, k = l & 3, r = up + 2 * hf, lane = g * 4 + c;
        const int sc = (int) reinterpret_cast<const int8_t *>(rec)[4 * (j * 8 + g) + 2 * up + hf];
        const uint32_t dw = reinterpret_cast<const uint32_t *>(rec + WT_TM_Q3K_D_OFF)[g];
        const float d = __half2float(__ushort_as_half((unsigned short) (up ? (dw >> 16) : (dw & 0xffffu))));
        const uint8_t * sub = rec + wt_tm_sub_off(W.type, j);
        const int lo = (int) ((reinterpret_cast<const uint32_t *>(sub)[lane] >> (8 * k + 2 * r)) & 3u);
        const int hb = (int) ((reinterpret_cast<const uint32_t *>(sub + wt_tm_qs_bytes(W.type))[g * 2 + up] >> l) & 1u);
        const int q = (lo | (hb << 2)) - 4;
        return __fmul_rn(__fmul_rn(d, (float) sc), (float) q);
    }
    if (wt_is_kquant(W.type)) {                                  // dequantize_row_q4_K / _q5_K: (d * sc) * q - dmin * m, each product rounded
        const uint8_t * hdr = rec + WT_TM_KQ_HDR_ROW * rr;
        const int j = i >> 5, l = i & 31, c = (l & 15) >> 2;
        int sc, mn; kq_scale_min(j, hdr + 4, sc, mn);
        const float d = __half2float(*reinterpret_cast<const __half *>(hdr)), dmin = __half2float(*reinterpret_cast<const __half *>(hdr + 2));
        const uint8_t * sub = rec + wt_tm_sub_off(W.type, j);
        const uint32_t w = reinterpret_cast<const uint32_t *>(sub)[(g * 4 + c) * 2 + up];
        int q = (int) ((w >> (8 * (l & 3) + 4 * (l >> 4))) & 0xFu);
        if (W.type == WT_Q5_K) q |= (int) ((reinterpret_cast<const uint32_t *>(sub + wt_tm_qs_bytes(W.type))[g * 2 + up] >> l) & 1u) << 4;
        return __fsub_rn(__fmul_rn(__fmul_rn(d, (float) sc), (float) q), __fmul_rn(dmin, (float) mn));
    }
    if (W.type == WT_F16) {
        const int c = (i & 7) >> 1, k = up + ((i >> 3) << 1);
        const uint32_t w = reinterpret_cast<const uint32_t *>(rec)[(g * 4 + c) * 4 + k];
        return __half2float(__ushort_as_half((unsigned short) ((i & 1) ? (w >> 16) : (w & 0xffffu))));
    }
    if (wt_has_min(W.type)) {                                    // dequantize_row_q4_1 / _q5_1: q * d + m
        const uint2 dm = reinterpret_cast<const uint2 *>(rec + wt_tm_d_off(W.type))[g];
        const float d = __half2float(__ushort_as_half((unsigned short) (up ? (dm.x >> 16) : (dm.x & 0xffffu))));
        const float m = __half2float(__ushort_as_half((unsigned short) (up ? (dm.y >> 16) : (dm.y & 0xffffu))));
        const int c = (i & 15) >> 2;
        const uint32_t w = reinterpret_cast<const uint32_t *>(rec)[(g * 4 + c) * 2 + up];
        int q = (int) ((w >> (8 * (i & 3) + 4 * (i >> 4))) & 0xFu);
        if (W.type == WT_Q5_1) q |= (int) ((reinterpret_cast<const uint32_t *>(rec + wt_tm_qs_bytes(W.type))[g * 2 + up] >> i) & 1u) << 4;
        return __fadd_rn(__fmul_rn((float) q, d), m);
    }
    const uint32_t dd = reinterpret_cast<const uint32_t *>(rec + wt_tm_d_off(W.type))[g];
    const float d = __half2float(__ushort_as_half((unsigned short) (up ? (dd >> 16) : (dd & 0xffffu))));
    if (W.type == WT_Q8_0) {
        const int c = (i & 15) >> 2, k = up + ((i >> 4) << 1);
        const uint32_t w = reinterpret_cast<const uint32_t *>(rec)[(g * 4 + c) * 4 + k];
        return d * (float) (int8_t) ((w >> (8 * (i & 3))) & 0xffu);
    }
    const int c = (i & 15) >> 2;
    const uint32_t w = reinterpret_cast<const uint32_t *>(rec)[(g * 4 + c) * 2 + up];
    int q = (int) ((w >> (8 * (i & 3) + 4 * (i >> 4))) & 0xFu);
    if (W.type == WT_Q5_0) { const uint32_t qh = reinterpret_cast<const uint32_t *>(rec + wt_tm_qs_bytes(W.type))[g * 2 + up]; q |= (int) ((qh >> i) & 1u) << 4; return d * (float) (q - 16); }
    return d * (float) (q - 8);
}
__device__ __forceinline__ float dequant_elem(const QMat & W, int64_t row, int e) {
    const int K = W.K;
    if (W.layout == 1) return dequant_elem_tm(W, row, e);
    switch (W.type) {
        case WT_F16: return __half2float(reinterpret_cast<const __half *>(W.base)[row * K + e]);
        case WT_Q4_0: { const int64_t b = row * (K >> 5) + (e >> 5); const int i = e & 31;
                        const uint8_t q = W.qs[b * 16 + (i & 15)]; const int v = (i < 16 ? (q & 0xF) : (q >> 4)) - 8;
                        return (float) v * __half2float(W.d[b]); }
        case WT_Q5_0: { const int64_t b = row * (K >> 5) + (e >> 5); const int i = e & 31;
                        const uint8_t q = W.qs[b * 16 + (i & 15)]; const uint32_t h = (W.qh[b] >> i) & 1u;
                        const int v = (int) ((i < 16 ? (q & 0xF) : (q >> 4)) | (h << 4)) - 16;
                        return (float) v * __half2float(W.d[b]); }
        case WT_Q4_1: case WT_Q5_1: {
                        const int64_t b = row * (K >> 5) + (e >> 5); const int i = e & 31;
                        const uint8_t q = W.qs[b * 16 + (i & 15)];
                        int v = i < 16 ? (q & 0xF) : (q >> 4);
                        if (W.type == WT_Q5_1) v |= (int) ((W.qh[b] >> i) & 1u) << 4;
                        return __fadd_rn(__fmul_rn((float) v, __half2float(W.d[b])), __half2float(W.m[b])); }
        case WT_Q8_0: { const int64_t b = row * (K >> 5) + (e >> 5);
                        return (float) reinterpret_cast<const int8_t *>(W.qs)[b * 32 + (e & 31)] * __half2float(W.d[b]); }
        case WT_Q4_K: case WT_Q5_K: {
            const int BLK = W.type == WT_Q4_K ? 144 : 176;
            const uint8_t * blk = reinterpret_cast<const uint8_t *>(W.base) + (row * (K >> 8) + (e >> 8)) * BLK;
            const int j = (e & 255) >> 5, l = e & 31;
            int sc, mn; kq_scale_min(j, blk + 4, sc, mn);
            const float d = __half2float(*reinterpret_cast<const __half *>(blk)), dmin = __half2float(*reinterpret_cast<const __half *>(blk + 2));
            const uint8_t * qs = blk + 16 + (W.type == WT_Q5_K ? 32 : 0) + 32 * (j >> 1);
            int q = (qs[l] >> (4 * (j & 1))) & 0xF;
            if (W.type == WT_Q5_K) q |= ((blk[16 + l] >> j) & 1) << 4;
            return d * sc * q - dmin * mn;
        }
        case WT_Q3_K:
            return q3k_elem(reinterpret_cast<const uint8_t *>(W.base) + (row * (K >> 8) + (e >> 8)) * 110, e & 255);
    }
    return 0.0f;
}
__global__ void k_dec_embed(const QMat te, const float * __restrict__ pe, const int * __restrict__ tok, const int * __restrict__ pos,
                            int d, float * __restrict__ x) {
    const int t = blockIdx.x;
    const int token = tok[t], p = pos[t];
    for (int e = threadIdx.x; e < d; e += blockDim.x)
        x[(int64_t) t * d + e] = dequant_elem(te, token, e) + pe[(int64_t) p * d + e];
}
void dec_embed(const QMat & te, const float * pe, const int * tokens, const int * pos, int n_tok, int d, float * x, cudaStream_t st) {
    k_dec_embed<<<n_tok, 256, 0, st>>>(te, pe, tokens, pos, d, x); count_launch();
}
__global__ void k_tok_resolve(int * __restrict__ tok, const SampOut * __restrict__ samp, int n_tok) {
    const int t = threadIdx.x;
    if (t < n_tok && tok[t] < 0) tok[t] = samp[-1 - tok[t]].id;
}
void tok_resolve(int * tokens, const SampOut * samp, int n_tok, cudaStream_t st) {
    k_tok_resolve<<<1, 64 * ((n_tok + 63) / 64), 0, st>>>(tokens, samp, n_tok); count_launch();
}
__global__ void k_dequant_rows(const QMat W, float * __restrict__ out) {
    const int64_t n = (int64_t) W.N * W.K;
    for (int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x * blockDim.x)
        out[i] = dequant_elem(W, i / W.K, (int) (i % W.K));
}
void dequant_rows_f32(const QMat & W, float * out, cudaStream_t st) {
    k_dequant_rows<<<1024, 256, 0, st>>>(W, out); count_launch();
}

// =====================================================================================================================
//  GEMV for the decode step: y[t][n] = act((W[n,:] . x[t,:] + bias[n]) * scale[n]) + res[t][n]
//
//  Reference arithmetic (ggml-cpu/ggml-cpu.c:1181-1357): activations are quantised per 32 values to Q8_0
//  (quantize_row_q8_0, AVX2 form ggml-cpu/arch/x86/quants.c: d = amax/127 stored as f16, q = rint(x*127/amax)) or per 256
//  values to Q8_K for K-quants (ggml-quants.c:2768-2805); the dot product is integer inside a block and
//  sum_b (d_w*d_x) * sumi outside (ggml-cpu/quants.c:365-406, 696-769).  This kernel does the same with __dp4a, so it
//  differs from the reference only in f32 summation order.  F16 weights: x rounded to f16, products accumulated in f32.
//  LayerNorm of x (when requested) is fused in front: every CTA recomputes it from the f32 residual stream.
// =====================================================================================================================
struct GemvK {
    QMat W; const float * x; int n_tok;
    const float * ln_w, * ln_b; float eps;
    const float * bias, * scale; int act; const float * res; float * out;
    __half * k_cache, * v_cache; const int * cells; int kv_d;
};

// quantize_row_q8_K (ggml-quants.c:2768-2805) of super-block sb of one activation row (layout: act_tok_stride), by one warp: per 256
// values iscale = -127/max (signed max-magnitude), q = min(127, nearest(iscale*x)), d = 1/iscale, and the sums of the eight 32-value
// sub-blocks.  xval(i): value i of the row.
template <class F>
__device__ __forceinline__ void q8k_quant_sb(F xval, uint8_t * tp, int K, int sb, int lane) {
    int8_t * xq = reinterpret_cast<int8_t *>(tp);
    float * xd = reinterpret_cast<float *>(tp + K);
    int *   bs = reinterpret_cast<int *>(tp + K + (K / 256) * 4);
    float v[8]; float amax = 0.0f, mx = 0.0f;
#pragma unroll
    for (int j = 0; j < 8; ++j) { v[j] = xval(sb * 256 + j * 32 + lane); const float av = fabsf(v[j]); if (av > amax) { amax = av; mx = v[j]; } }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const float oa = __shfl_xor_sync(0xffffffffu, amax, o), om = __shfl_xor_sync(0xffffffffu, mx, o);
        if (oa > amax) { amax = oa; mx = om; }
    }
    if (amax == 0.0f) {
#pragma unroll
        for (int j = 0; j < 8; ++j) xq[sb * 256 + j * 32 + lane] = 0;
        if (lane == 0) xd[sb] = 0.0f;
        if (lane < 8) bs[sb * 8 + lane] = 0;
        return;
    }
    const float iscale = -127.0f / mx;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        int q = __float2int_rn(iscale * v[j]); q = min(127, q);
        xq[sb * 256 + j * 32 + lane] = (int8_t) q;
        int ssum = q;
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) ssum += __shfl_xor_sync(0xffffffffu, ssum, o);
        if (lane == 0) bs[sb * 8 + j] = ssum;
    }
    if (lane == 0) xd[sb] = 1.0f / iscale;
}

template <int WT, int NT>
__global__ void __launch_bounds__(256)
k_gemv(const GemvK a) {
    extern __shared__ __align__(16) uint8_t sm[];
    const int K = a.W.K, N = a.W.N;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint8_t * tokbase = sm;
    const size_t tb = act_tok_stride(WT, K);                 // shared memory: one activation row per token

    // ---------------------------------------------------------------- prologue: (LN) + activation quantisation
    // LayerNorm statistics: one warp per token (two passes, like the reference); quantisation: the (token, block) pairs are
    // spread over all 256 threads, each thread owning one 32-value block (no shuffles on the critical path).
    __shared__ float s_mean[8], s_rstd[8];
    if (a.ln_w) {
        for (int t = warp; t < a.n_tok; t += 8) {
            const float * xr = a.x + (int64_t) t * K;
            float s = 0.0f;
            for (int i = lane; i < K; i += 32) s += xr[i];
            const float mean = warp_sum(s) / K;
            float v = 0.0f;
            for (int i = lane; i < K; i += 32) { const float d0 = xr[i] - mean; v += d0 * d0; }
            const float rstd = 1.0f / sqrtf(warp_sum(v) / K + a.eps);
            if (lane == 0) { s_mean[t] = mean; s_rstd[t] = rstd; }
        }
        __syncthreads();
    }
    auto xval = [&](int t, int i) -> float {      // the (normalised) activation the contraction consumes
        const float v = a.x[(int64_t) t * K + i];
        return a.ln_w ? __fadd_rn(__fmul_rn(__fmul_rn(v - s_mean[t], s_rstd[t]), a.ln_w[i]), a.ln_b[i]) : v;
    };
    if (WT == WT_F16) {
        for (int i = tid; i < a.n_tok * K; i += 256) {
            const int t = i / K, e = i - t * K;
            reinterpret_cast<__half *>(tokbase + t * tb)[e] = __float2half_rn(xval(t, e));
        }
    } else if (wt_is_kquant(WT)) {
        const int nsb = K / 256;
        for (int pidx = warp; pidx < a.n_tok * nsb; pidx += 8) {
            const int t = pidx / nsb;
            q8k_quant_sb([&](int i) { return xval(t, i); }, tokbase + t * tb, K, pidx - t * nsb, lane);
        }
    } else {
        const int nb = K / 32;
        for (int pidx = tid; pidx < a.n_tok * nb; pidx += 256) {
            const int t = pidx / nb, b = pidx - t * nb;
            uint8_t * tp = tokbase + t * tb;
            float v[32]; float amax = 0.0f;
#pragma unroll
            for (int i = 0; i < 32; ++i) { v[i] = xval(t, b * 32 + i); amax = fmaxf(amax, fabsf(v[i])); }
            const float d  = amax / 127.0f;
            const float id = (amax != 0.0f) ? 127.0f / amax : 0.0f;
            uint32_t pk[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int q0 = __float2int_rn(v[4*i] * id), q1 = __float2int_rn(v[4*i+1] * id), q2 = __float2int_rn(v[4*i+2] * id), q3 = __float2int_rn(v[4*i+3] * id);
                pk[i] = (uint32_t) (q0 & 0xFF) | ((uint32_t) (q1 & 0xFF) << 8) | ((uint32_t) (q2 & 0xFF) << 16) | ((uint32_t) (q3 & 0xFF) << 24);
            }
            uint4 * dst = reinterpret_cast<uint4 *>(tp + b * 32);
            dst[0] = make_uint4(pk[0], pk[1], pk[2], pk[3]); dst[1] = make_uint4(pk[4], pk[5], pk[6], pk[7]);
            if (wt_has_min(WT)) {                                // Q8_1: {f16 d, f16 s = d * sum(q)} (quantize_row_q8_1, unrounded d)
                int sum = 0;
#pragma unroll
                for (int i = 0; i < 8; ++i) sum = __dp4a((int) pk[i], 0x01010101, sum);
                reinterpret_cast<__half2 *>(tp + K)[b] = __halves2half2(__float2half_rn(d), __float2half_rn(d * (float) sum));
            } else reinterpret_cast<float *>(tp + K)[b] = __half2float(__float2half_rn(d));
        }
    }
    __syncthreads();

    // ---------------------------------------------------------------- rows: one warp per output row
    const int nwarps_total = gridDim.x * 8;
    for (int row = blockIdx.x * 8 + warp; row < N; row += nwarps_total) {
        float acc[NT];
#pragma unroll
        for (int t = 0; t < NT; ++t) acc[t] = 0.0f;

        if (WT == WT_F16) {
            const uint4 * wr = reinterpret_cast<const uint4 *>(reinterpret_cast<const __half *>(a.W.base) + (int64_t) row * K);
            for (int c = lane; c < K / 8; c += 32) {
                const uint4 w8 = __ldg(wr + c);
                const __half2 * wh = reinterpret_cast<const __half2 *>(&w8);
#pragma unroll
                for (int t = 0; t < NT; ++t) {
                    if (t < a.n_tok) {
                        const uint4 x8 = *reinterpret_cast<const uint4 *>(tokbase + t * tb + (size_t) c * 16);
                        const __half2 * xh = reinterpret_cast<const __half2 *>(&x8);
#pragma unroll
                        for (int e = 0; e < 4; ++e) {
                            const float2 wf = __half22float2(wh[e]), xf = __half22float2(xh[e]);
                            acc[t] = fmaf(wf.x, xf.x, acc[t]); acc[t] = fmaf(wf.y, xf.y, acc[t]);
                        }
                    }
                }
            }
        } else if (WT == WT_Q4_K || WT == WT_Q5_K) {
            constexpr int BLK = (WT == WT_Q4_K) ? 144 : 176;
            const uint8_t * rowp = reinterpret_cast<const uint8_t *>(a.W.base) + (int64_t) row * (K >> 8) * BLK;
            for (int c = lane; c < K / 8; c += 32) {           // chunk of 8 weights: super-block c/32, sub-block (c%32)/4, quarter c%4
                const int sb = c >> 5, j = (c & 31) >> 2, qd = c & 3;
                const uint8_t * blk = rowp + (int64_t) sb * BLK;
                const __half2 dm = *reinterpret_cast<const __half2 *>(blk);
                int sc, mn; kq_scale_min(j, blk + 4, sc, mn);
                const uint8_t * qs = blk + 16 + (WT == WT_Q5_K ? 32 : 0) + 32 * (j >> 1) + 8 * qd;
                uint32_t w0 = (*reinterpret_cast<const uint32_t *>(qs)     >> (4 * (j & 1))) & 0x0F0F0F0Fu;
                uint32_t w1 = (*reinterpret_cast<const uint32_t *>(qs + 4) >> (4 * (j & 1))) & 0x0F0F0F0Fu;
                if (WT == WT_Q5_K) {
                    const uint8_t * qh = blk + 16 + 8 * qd;
                    w0 |= ((*reinterpret_cast<const uint32_t *>(qh)     >> j) & 0x01010101u) << 4;
                    w1 |= ((*reinterpret_cast<const uint32_t *>(qh + 4) >> j) & 0x01010101u) << 4;
                }
                const float dl = __low2float(dm) * (float) sc, ml = __high2float(dm) * (float) mn;
#pragma unroll
                for (int t = 0; t < NT; ++t) {
                    if (t < a.n_tok) {
                        const uint8_t * tp = tokbase + t * tb;
                        const int * xq = reinterpret_cast<const int *>(tp) + (sb * 256 + j * 32 + qd * 8) / 4;
                        const float d8 = reinterpret_cast<const float *>(tp + K)[sb];
                        const int xa = xq[0], xb = xq[1];
                        const int sumi = __dp4a((int) w0, xa, __dp4a((int) w1, xb, 0));
                        const int sumx = __dp4a(0x01010101, xa, __dp4a(0x01010101, xb, 0));
                        acc[t] += d8 * (dl * (float) sumi - ml * (float) sumx);
                    }
                }
            }
        } else if (WT == WT_Q3_K) {
            constexpr int BLK = 110;
            const uint8_t * rowp = reinterpret_cast<const uint8_t *>(a.W.base) + (int64_t) row * (K >> 8) * BLK;
            for (int c = lane; c < K / 8; c += 32) {           // chunk of 8 weights (half of one 16-value scale group): super-block c/32
                const int sb = c >> 5, e0 = (c & 31) * 8;
                const uint8_t * blk = rowp + (int64_t) sb * BLK;
                const int w0 = (int) q3k_q4(blk, e0), w1 = (int) q3k_q4(blk, e0 + 4);
                const int sc = q3k_scale(blk, e0 >> 4);
                const float dw = q3k_d(blk);
#pragma unroll
                for (int t = 0; t < NT; ++t) {
                    if (t < a.n_tok) {                           // ggml_vec_dot_q3_K_q8_K: (d_w d_x) * (sc * sumi)
                        const uint8_t * tp = tokbase + t * tb;
                        const int * xq = reinterpret_cast<const int *>(tp) + (sb * 256 + e0) / 4;
                        const float d8 = reinterpret_cast<const float *>(tp + K)[sb];
                        const int sumi = __dp4a(w0, xq[0], __dp4a(w1, xq[1], 0));
                        acc[t] = fmaf(dw * d8, (float) (sc * sumi), acc[t]);
                    }
                }
            }
        } else {
            const int64_t rb = (int64_t) row * (K >> 5);
            for (int c = lane; c < K / 8; c += 32) {           // chunk = quarter block
                const int b = c >> 2, qd = c & 3;
                const float dw = __half2float(a.W.d[rb + b]);
                const float mw = wt_has_min(WT) ? __half2float(a.W.m[rb + b]) : 0.0f;
                int vl, vh;
                if (WT == WT_Q8_0) {
                    const uint2 w = __ldg(reinterpret_cast<const uint2 *>(a.W.qs + (rb + b) * 32) + qd);
                    vl = (int) w.x; vh = (int) w.y;
                } else {
                    const uint32_t w = __ldg(reinterpret_cast<const uint32_t *>(a.W.qs + (rb + b) * 16) + qd);
                    uint32_t lo = w & 0x0F0F0F0Fu, hi = (w >> 4) & 0x0F0F0F0Fu;
                    if (wt_has_qh(WT)) {
                        const uint32_t qh = __ldg(a.W.qh + rb + b);
                        lo |= spread4_to_bit4(qh >> (4 * qd));
                        hi |= spread4_to_bit4(qh >> (16 + 4 * qd));
                    }
                    if (wt_has_min(WT)) { vl = (int) lo; vh = (int) hi; }
                    else if (WT == WT_Q5_0) {
                        vl = (int) __vsub4(lo, 0x10101010u); vh = (int) __vsub4(hi, 0x10101010u);
                    } else {
                        vl = (int) __vsub4(lo, 0x08080808u); vh = (int) __vsub4(hi, 0x08080808u);
                    }
                }
#pragma unroll
                for (int t = 0; t < NT; ++t) {
                    if (t < a.n_tok) {
                        const uint8_t * tp = tokbase + t * tb;
                        const int * xq = reinterpret_cast<const int *>(tp);
                        const float dx = reinterpret_cast<const float *>(tp + K)[b];
                        int xa, xb;
                        if (WT == WT_Q8_0) { xa = xq[b * 8 + 2 * qd]; xb = xq[b * 8 + 2 * qd + 1]; }
                        else               { xa = xq[b * 8 + qd];     xb = xq[b * 8 + 4 + qd]; }
                        const int sumi = __dp4a(vl, xa, __dp4a(vh, xb, 0));
                        if (wt_has_min(WT)) {                    // ggml_vec_dot_q4_1_q8_1: (d_w d_x) sumi + m_w s_x, the m term once per block
                            const __half2 ds = reinterpret_cast<const __half2 *>(tp + K)[b];
                            acc[t] = fmaf(dw * __low2float(ds), (float) sumi, acc[t]);
                            if (qd == 0) acc[t] = fmaf(mw, __high2float(ds), acc[t]);
                        } else
                        acc[t] = fmaf(dw * dx, (float) sumi, acc[t]);
                    }
                }
            }
        }

#pragma unroll
        for (int t = 0; t < NT; ++t) acc[t] = warp_sum(acc[t]);
        if (lane == 0) {
            const float bias = a.bias ? a.bias[row] : 0.0f;
            const float scl  = a.scale ? a.scale[row] : 1.0f;
#pragma unroll
            for (int t = 0; t < NT; ++t) {
                if (t < a.n_tok) {
                    float v = (acc[t] + bias) * scl;
                    if (a.act == 1) v = gelu_ref_f16(v);
                    if (a.res) v += a.res[(int64_t) t * N + row];
                    if (a.out) a.out[(int64_t) t * N + row] = v;
                    if (a.k_cache && row >= a.kv_d) {
                        const int64_t cell = a.cells[t];
                        if (row < 2 * a.kv_d) a.k_cache[cell * a.kv_d + (row - a.kv_d)] = __float2half_rn(v);
                        else                  a.v_cache[cell * a.kv_d + (row - 2 * a.kv_d)] = __float2half_rn(v);
                    }
                }
            }
        }
    }
}

template <int WT, int NT>
static void gemv_launch(const GemvK & k, cudaStream_t st) {
    const int K = k.W.K, N = k.W.N;
    const size_t smem = act_tok_stride(WT, K) * k.n_tok;
    auto kern = k_gemv<WT, NT>;
    if (smem > 48 * 1024) ensure_dyn_smem(reinterpret_cast<const void *>(kern), smem);
    int grid = (N + 7) / 8;                  // one row per warp per pass
    const int cap = 132 * 4;                 // keep the per-CTA prologue amortised over several rows
    if (grid > cap) grid = cap;
    kern<<<grid, 256, smem, st>>>(k); count_launch();
}
template <int WT>
static void gemv_nt(const GemvK & k, cudaStream_t st) {
    if (k.n_tok <= 1)      gemv_launch<WT, 1>(k, st);
    else if (k.n_tok <= 2) gemv_launch<WT, 2>(k, st);
    else if (k.n_tok <= 4) gemv_launch<WT, 4>(k, st);
    else                   gemv_launch<WT, 8>(k, st);
}
void gemv(const GemvArgs & a, cudaStream_t st) {
    // algorithmic bytes: the weight matrix once + activations in / results out (SURVEY.md section 8d)
    ProfScope prof(PC_GEMV, st, (double) a.W.N * a.W.K * wt_bpw(a.W.type) + (double) a.n_tok * (a.W.K + a.W.N) * 4, 2.0 * a.W.N * a.W.K * a.n_tok);
    GemvK k; k.W = a.W; k.x = a.x; k.n_tok = a.n_tok; k.ln_w = a.ln_w; k.ln_b = a.ln_b; k.eps = a.eps;
    k.bias = a.bias; k.scale = a.scale; k.act = a.act; k.res = a.res; k.out = a.out;
    k.k_cache = a.k_cache; k.v_cache = a.v_cache; k.cells = a.cells; k.kv_d = a.kv_d;
    switch (a.W.type) {
        case WT_F16:  gemv_nt<WT_F16>(k, st);  break;
        case WT_Q4_0: gemv_nt<WT_Q4_0>(k, st); break;
        case WT_Q5_0: gemv_nt<WT_Q5_0>(k, st); break;
        case WT_Q4_1: gemv_nt<WT_Q4_1>(k, st); break;
        case WT_Q5_1: gemv_nt<WT_Q5_1>(k, st); break;
        case WT_Q8_0: gemv_nt<WT_Q8_0>(k, st); break;
        case WT_Q4_K: gemv_nt<WT_Q4_K>(k, st); break;
        case WT_Q5_K: gemv_nt<WT_Q5_K>(k, st); break;
        case WT_Q3_K: gemv_nt<WT_Q3_K>(k, st); break;
        default: set_error("gemv: unsupported weight type %d", a.W.type);
    }
}

// =====================================================================================================================
//  GEMV v2 for the decode step: activation quantisation is a separate tiny kernel (k_act_quant, one CTA per token) and the
//  contraction uses the integer tensor-core instruction mma.sync.m16n8k32.s8 so that up to 8 sequences share one pass
//  over the weights:   D[16 rows][8 tokens] (i32) = W_q[16][32] . X_q8[32][8]   -- exactly one 32-value quant block --
//  followed by acc += D * d_w[row] * d_x[token] in f32: the same integer-dot + block-scale arithmetic as the reference's
//  vec_dot_q*_q8_0 (ggml-cpu/quants.c:365-406) and the dp4a kernel above; only the f32 summation order differs.
//  One CTA = 16 or 32 output rows (one or two m16 tiles); its 8 warps split K and reduce through shared memory.
// =====================================================================================================================
template <int MODE>   // 0: Q8_0 blocks  1: Q8_K super-blocks  2: f16  3: Q8_1 blocks
__global__ void __launch_bounds__(256)
k_act_quant(const float * __restrict__ x, int K, const float * __restrict__ ln_w, const float * __restrict__ ln_b, float eps,
            uint8_t * __restrict__ out, size_t tok_stride) {
    __shared__ float red[32];
    const int t = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float * xr = x + (int64_t) t * K;
    uint8_t * tp = out + (size_t) t * tok_stride;
    float mean = 0.0f, rstd = 1.0f;
    if (ln_w) {
        float s = 0.0f;
        for (int i = tid; i < K; i += 256) s += xr[i];
        mean = block_sum(s, red) / K;
        float v = 0.0f;
        for (int i = tid; i < K; i += 256) { const float d0 = xr[i] - mean; v += d0 * d0; }
        rstd = 1.0f / sqrtf(block_sum(v, red) / K + eps);
    }
    auto xval = [&](int i) -> float {
        const float v = xr[i];
        return ln_w ? __fadd_rn(__fmul_rn(__fmul_rn(v - mean, rstd), ln_w[i]), ln_b[i]) : v;
    };
    if (MODE == 2) {
        for (int i = tid; i < K; i += 256) reinterpret_cast<__half *>(tp)[i] = __float2half_rn(xval(i));
    } else if (MODE == 1) {
        for (int sb = warp; sb < K / 256; sb += 8) q8k_quant_sb(xval, tp, K, sb, lane);
    } else {
        // quantize_row_q8_0 / _q8_1, AVX2 form (ggml-cpu/arch/x86/quants.c): warp per block, lane per element (coalesced)
        for (int b = warp; b < K / 32; b += 8) {
            const float v = xval(b * 32 + lane);
            const float amax = warp_max(fabsf(v));
            const float d  = amax / 127.0f;
            const float id = (amax != 0.0f) ? 127.0f / amax : 0.0f;
            const int q = __float2int_rn(v * id);
            reinterpret_cast<int8_t *>(tp)[b * 32 + lane] = (int8_t) q;
            if (MODE == 3) {                                     // quantize_row_q8_1: {f16 d, f16 (d * sum q)}, d unrounded
                int sum = q;
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
                if (lane == 0) reinterpret_cast<__half2 *>(tp + K)[b] = __halves2half2(__float2half_rn(d), __float2half_rn(d * (float) sum));
            } else if (lane == 0) reinterpret_cast<float *>(tp + K)[b] = __half2float(__float2half_rn(d));
        }
    }
}

struct Gemv2K {
    QMat W; const uint8_t * act; size_t tok_stride; int n_tok;
    const float * bias, * scale; int act_fn; const float * res; float * out;
    __half * k_cache, * v_cache; const int * cells; int kv_d;
};

template <int WT, int MT>   // MT = m16 tiles per CTA (1: 16 rows -- more CTAs for the d x d matrices; 2: 32 rows)
__global__ void __launch_bounds__(256)
k_gemv_mma(const Gemv2K a) {
    __shared__ float red[8][16 * MT][9];
    const int K = a.W.K, N = a.W.N;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int g = lane >> 2, c = lane & 3;
    const int n0 = blockIdx.x * 16 * MT;
    float acc[MT][4];
#pragma unroll
    for (int mt = 0; mt < MT; ++mt) { acc[mt][0] = acc[mt][1] = acc[mt][2] = acc[mt][3] = 0.0f; }
    // rows this lane feeds into the A fragments: (m-tile, +0 / +8); clamped for the ragged last CTA (masked at the store)
    int rows[2 * MT];
#pragma unroll
    for (int i = 0; i < 2 * MT; ++i) rows[i] = min(N - 1, n0 + (i >> 1) * 16 + g + (i & 1) * 8);
    const bool tok_ok = g < a.n_tok;
    const uint8_t * actg = a.act + (size_t) (tok_ok ? g : 0) * a.tok_stride;           // token of the B fragment (column g)
    const uint8_t * act0 = a.act + (size_t) min(2 * c,     a.n_tok - 1) * a.tok_stride; // tokens of the D fragment columns
    const uint8_t * act1 = a.act + (size_t) min(2 * c + 1, a.n_tok - 1) * a.tok_stride;

    if (WT == WT_F16) {
        const __half * Wb = reinterpret_cast<const __half *>(a.W.base);
        const uint32_t * xg = reinterpret_cast<const uint32_t *>(actg);
        for (int ks = warp; ks < K / 16; ks += 8) {
            const uint32_t b0 = tok_ok ? xg[ks * 8 + c] : 0u, b1 = tok_ok ? xg[ks * 8 + 4 + c] : 0u;
#pragma unroll
            for (int mt = 0; mt < MT; ++mt) {
                const uint32_t * r0 = reinterpret_cast<const uint32_t *>(Wb + (int64_t) rows[2*mt] * K) + ks * 8;
                const uint32_t * r1 = reinterpret_cast<const uint32_t *>(Wb + (int64_t) rows[2*mt + 1] * K) + ks * 8;
                const uint32_t af[4] = { __ldg(r0 + c), __ldg(r1 + c), __ldg(r0 + 4 + c), __ldg(r1 + 4 + c) };
                mma_f16_16816(acc[mt], af, b0, b1);
            }
        }
    } else if (WT == WT_Q4_K || WT == WT_Q5_K) {
        constexpr int BLK = (WT == WT_Q4_K) ? 144 : 176;
        const int nsb = K / 256;
        const uint32_t * xg = reinterpret_cast<const uint32_t *>(actg);
        const float * d80 = reinterpret_cast<const float *>(act0 + K), * d81 = reinterpret_cast<const float *>(act1 + K);
        const int * bs0 = reinterpret_cast<const int *>(act0 + K + nsb * 4), * bs1 = reinterpret_cast<const int *>(act1 + K + nsb * 4);
        // work item = (super-block, nibble pair jj): 4 per super-block
        for (int it = warp; it < nsb * 4; it += 8) {
            const int sb = it >> 2, jj = it & 3;
            uint32_t bx[2][2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int j = 2 * jj + h;
                bx[h][0] = tok_ok ? xg[(sb * 256 + j * 32) / 4 + c] : 0u;
                bx[h][1] = tok_ok ? xg[(sb * 256 + j * 32) / 4 + 4 + c] : 0u;
            }
            const float x80 = d80[sb], x81 = d81[sb];
#pragma unroll
            for (int mt = 0; mt < MT; ++mt) {
                uint32_t wlo[2], whi[2], hlo[2] = { 0, 0 }, hhi[2] = { 0, 0 }; float dl[2][2], ml[2][2];
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const uint8_t * blk = reinterpret_cast<const uint8_t *>(a.W.base) + ((int64_t) rows[2*mt + r] * nsb + sb) * BLK;
                    const uint32_t * q32 = reinterpret_cast<const uint32_t *>(blk + 16 + (WT == WT_Q5_K ? 32 : 0) + 32 * jj);
                    wlo[r] = __ldg(q32 + c); whi[r] = __ldg(q32 + 4 + c);
                    if (WT == WT_Q5_K) { const uint32_t * h32 = reinterpret_cast<const uint32_t *>(blk + 16); hlo[r] = __ldg(h32 + c); hhi[r] = __ldg(h32 + 4 + c); }
                    const __half2 dm = *reinterpret_cast<const __half2 *>(blk);
#pragma unroll
                    for (int h = 0; h < 2; ++h) { int sc, mn; kq_scale_min(2 * jj + h, blk + 4, sc, mn); dl[r][h] = __low2float(dm) * (float) sc; ml[r][h] = __high2float(dm) * (float) mn; }
                }
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int j = 2 * jj + h;
                    uint32_t af[4];
#pragma unroll
                    for (int r = 0; r < 2; ++r) {
                        uint32_t lo = (wlo[r] >> (4 * h)) & 0x0F0F0F0Fu, hi = (whi[r] >> (4 * h)) & 0x0F0F0F0Fu;
                        if (WT == WT_Q5_K) { lo |= ((hlo[r] >> j) & 0x01010101u) << 4; hi |= ((hhi[r] >> j) & 0x01010101u) << 4; }
                        af[r] = lo; af[2 + r] = hi;
                    }
                    int dd[4]; mma_s8_16832(dd, af, bx[h][0], bx[h][1]);
                    const float s0 = (float) bs0[sb * 8 + j], s1 = (float) bs1[sb * 8 + j];
                    acc[mt][0] += x80 * (dl[0][h] * (float) dd[0] - ml[0][h] * s0);
                    acc[mt][1] += x81 * (dl[0][h] * (float) dd[1] - ml[0][h] * s1);
                    acc[mt][2] += x80 * (dl[1][h] * (float) dd[2] - ml[1][h] * s0);
                    acc[mt][3] += x81 * (dl[1][h] * (float) dd[3] - ml[1][h] * s1);
                }
            }
        }
    } else if (WT == WT_Q3_K) {
        constexpr int BLK = 110;
        const int nsb = K / 256;
        const uint32_t * xg = reinterpret_cast<const uint32_t *>(actg);
        const float * d80 = reinterpret_cast<const float *>(act0 + K), * d81 = reinterpret_cast<const float *>(act1 + K);
        for (int b = warp; b < K / 32; b += 8) {               // work item = one 32-value sub-block: two k16 products, one per scale
            const int sb = b >> 3, j = b & 7;
            const uint32_t b0 = tok_ok ? xg[b * 8 + c] : 0u, b1 = tok_ok ? xg[b * 8 + 4 + c] : 0u;
            const float x80 = d80[sb], x81 = d81[sb];
#pragma unroll
            for (int mt = 0; mt < MT; ++mt) {
                uint32_t af[4], sw = 0; float dw[2];
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const uint8_t * blk = reinterpret_cast<const uint8_t *>(a.W.base) + ((int64_t) rows[2*mt + r] * nsb + sb) * BLK;
                    af[r] = q3k_q4(blk, 32 * j + 4 * c); af[2 + r] = q3k_q4(blk, 32 * j + 16 + 4 * c);
                    sw |= ((uint32_t) (q3k_scale(blk, 2 * j) & 0xff) | ((uint32_t) (q3k_scale(blk, 2 * j + 1) & 0xff) << 8)) << (16 * r);
                    dw[r] = q3k_d(blk);
                }
                int si[4]; q3k_sumi(af, b0, b1, sw, si);
                acc[mt][0] = fmaf(dw[0] * x80, (float) si[0], acc[mt][0]);
                acc[mt][1] = fmaf(dw[0] * x81, (float) si[1], acc[mt][1]);
                acc[mt][2] = fmaf(dw[1] * x80, (float) si[2], acc[mt][2]);
                acc[mt][3] = fmaf(dw[1] * x81, (float) si[3], acc[mt][3]);
            }
        }
    } else {
        const int nblk = K >> 5;
        const uint32_t * xg = reinterpret_cast<const uint32_t *>(actg);
        const float * dx0p = reinterpret_cast<const float *>(act0 + K), * dx1p = reinterpret_cast<const float *>(act1 + K);
        constexpr int QW = (WT == WT_Q8_0) ? 8 : 4;            // 32-bit words of qs per block
#pragma unroll 5
        for (int b = warp; b < nblk; b += 8) {
            const uint32_t b0 = tok_ok ? xg[b * 8 + c] : 0u, b1 = tok_ok ? xg[b * 8 + 4 + c] : 0u;
            float dx0 = dx0p[b], dx1 = dx1p[b], sx0 = 0.0f, sx1 = 0.0f;
            if (wt_has_min(WT)) {                                // Q8_1 rows: {f16 d, f16 s} in place of the f32 scale
                const __half2 p0 = reinterpret_cast<const __half2 *>(dx0p)[b], p1 = reinterpret_cast<const __half2 *>(dx1p)[b];
                dx0 = __low2float(p0); sx0 = __high2float(p0); dx1 = __low2float(p1); sx1 = __high2float(p1);
            }
#pragma unroll
            for (int mt = 0; mt < MT; ++mt) {
                uint32_t af[4]; float dw[2], mw[2] = { 0.0f, 0.0f };
#pragma unroll
                for (int r = 0; r < 2; ++r) {
                    const int64_t bi = (int64_t) rows[2*mt + r] * nblk + b;
                    const uint32_t * q32 = reinterpret_cast<const uint32_t *>(a.W.qs) + bi * QW;
                    dw[r] = __half2float(a.W.d[bi]);
                    if (wt_has_min(WT)) mw[r] = __half2float(a.W.m[bi]);
                    if (WT == WT_Q8_0) { af[r] = __ldg(q32 + c); af[2 + r] = __ldg(q32 + 4 + c); }
                    else {
                        const uint32_t w = __ldg(q32 + c);
                        uint32_t lo = w & 0x0F0F0F0Fu, hi = (w >> 4) & 0x0F0F0F0Fu;
                        if (wt_has_qh(WT)) { const uint32_t qh = __ldg(a.W.qh + bi); lo |= spread4_to_bit4(qh >> (4 * c)); hi |= spread4_to_bit4(qh >> (16 + 4 * c)); }
                        if (wt_has_min(WT)) { af[r] = lo; af[2 + r] = hi; }
                        else if (WT == WT_Q5_0) { af[r] = __vsub4(lo, 0x10101010u); af[2 + r] = __vsub4(hi, 0x10101010u); }
                        else { af[r] = __vsub4(lo, 0x08080808u); af[2 + r] = __vsub4(hi, 0x08080808u); }
                    }
                }
                int dd[4]; mma_s8_16832(dd, af, b0, b1);
                acc[mt][0] = fmaf(dw[0] * dx0, (float) dd[0], acc[mt][0]);
                acc[mt][1] = fmaf(dw[0] * dx1, (float) dd[1], acc[mt][1]);
                acc[mt][2] = fmaf(dw[1] * dx0, (float) dd[2], acc[mt][2]);
                acc[mt][3] = fmaf(dw[1] * dx1, (float) dd[3], acc[mt][3]);
                if (wt_has_min(WT)) {                            // the block minimum against the activation block's sum (Q8_1 s)
                    acc[mt][0] = fmaf(mw[0], sx0, acc[mt][0]); acc[mt][1] = fmaf(mw[0], sx1, acc[mt][1]);
                    acc[mt][2] = fmaf(mw[1], sx0, acc[mt][2]); acc[mt][3] = fmaf(mw[1], sx1, acc[mt][3]);
                }
            }
        }
    }

    // ---- cross-warp (split-K) reduction and epilogue: thread -> (token = tid/32, row = tid%32)
#pragma unroll
    for (int mt = 0; mt < MT; ++mt)
#pragma unroll
        for (int i = 0; i < 4; ++i) red[warp][mt * 16 + g + (i >> 1) * 8][2 * c + (i & 1)] = acc[mt][i];
    __syncthreads();
    constexpr int RT = 16 * MT;
    const int t = tid / RT, rl = tid % RT, row = n0 + rl;
    if (t < 8 && t < a.n_tok && row < N) {
        float v = 0.0f;
#pragma unroll
        for (int w = 0; w < 8; ++w) v += red[w][rl][t];
        v = (v + (a.bias ? a.bias[row] : 0.0f)) * (a.scale ? a.scale[row] : 1.0f);
        if (a.act_fn == 1) v = gelu_ref_f16(v);
        if (a.res) v += a.res[(int64_t) t * N + row];
        if (a.out) a.out[(int64_t) t * N + row] = v;
        if (a.k_cache && row >= a.kv_d) {
            const int64_t cell = a.cells[t];
            if (row < 2 * a.kv_d) a.k_cache[cell * a.kv_d + (row - a.kv_d)] = __float2half_rn(v);
            else                  a.v_cache[cell * a.kv_d + (row - 2 * a.kv_d)] = __float2half_rn(v);
        }
    }
}

void gemv2(const GemvArgs & a, uint8_t * act_scratch, cudaStream_t st) {
    const int K = a.W.K, N = a.W.N;
    const size_t ts = act_tok_stride(a.W.type, K);
    {
        ProfScope prof(PC_OTHER, st, 0.0, 0.0);
        if (a.W.type == WT_F16)           k_act_quant<2><<<a.n_tok, 256, 0, st>>>(a.x, K, a.ln_w, a.ln_b, a.eps, act_scratch, ts);
        else if (wt_is_kquant(a.W.type))  k_act_quant<1><<<a.n_tok, 256, 0, st>>>(a.x, K, a.ln_w, a.ln_b, a.eps, act_scratch, ts);
        else if (wt_has_min(a.W.type))    k_act_quant<3><<<a.n_tok, 256, 0, st>>>(a.x, K, a.ln_w, a.ln_b, a.eps, act_scratch, ts);
        else                              k_act_quant<0><<<a.n_tok, 256, 0, st>>>(a.x, K, a.ln_w, a.ln_b, a.eps, act_scratch, ts);
        count_launch();
    }
    ProfScope prof(PC_GEMV, st, (double) N * K * wt_bpw(a.W.type) + (double) a.n_tok * (K + N) * 4, 2.0 * N * K * a.n_tok);
    Gemv2K k; k.W = a.W; k.act = act_scratch; k.tok_stride = ts; k.n_tok = a.n_tok; k.bias = a.bias; k.scale = a.scale; k.act_fn = a.act;
    k.res = a.res; k.out = a.out; k.k_cache = a.k_cache; k.v_cache = a.v_cache; k.cells = a.cells; k.kv_d = a.kv_d;
    // 16-row CTAs while that still leaves every SM several CTAs; 32-row CTAs for the vocabulary-sized matrix
    const bool small = N <= 8192;
    const int grid = small ? (N + 15) / 16 : (N + 31) / 32;
#define WB_GEMV2(T) do { if (small) k_gemv_mma<T, 1><<<grid, 256, 0, st>>>(k); else k_gemv_mma<T, 2><<<grid, 256, 0, st>>>(k); } while (0)
    switch (a.W.type) {
        case WT_F16:  WB_GEMV2(WT_F16);  break;
        case WT_Q4_0: WB_GEMV2(WT_Q4_0); break;
        case WT_Q5_0: WB_GEMV2(WT_Q5_0); break;
        case WT_Q4_1: WB_GEMV2(WT_Q4_1); break;
        case WT_Q5_1: WB_GEMV2(WT_Q5_1); break;
        case WT_Q8_0: WB_GEMV2(WT_Q8_0); break;
        case WT_Q4_K: WB_GEMV2(WT_Q4_K); break;
        case WT_Q5_K: WB_GEMV2(WT_Q5_K); break;
        case WT_Q3_K: WB_GEMV2(WT_Q3_K); break;
        default: set_error("gemv2: unsupported weight type %d", a.W.type); return;
    }
#undef WB_GEMV2
    count_launch();
}

// =====================================================================================================================
//  decode-step attention (ggml_flash_attn_ext on CPU: ggml-cpu/ops.cpp:8479-8715): Q is rounded to f16, K/V are f16,
//  scores and the running sums are f32 here (the CPU accumulates V in f16; f32 is strictly closer to exact).
// =====================================================================================================================
__device__ __forceinline__ float dot64_f16(const __half * __restrict__ k, const float * __restrict__ q) {
    float s = 0.0f;
    const uint4 * k4 = reinterpret_cast<const uint4 *>(k);
#pragma unroll
    for (int c = 0; c < 8; ++c) {
        const uint4 u = k4[c];
        const __half2 * h = reinterpret_cast<const __half2 *>(&u);
#pragma unroll
        for (int e = 0; e < 4; ++e) { const float2 f = __half22float2(h[e]); s = fmaf(f.x, q[c*8 + 2*e], s); s = fmaf(f.y, q[c*8 + 2*e + 1], s); }
    }
    return s;
}

// grid (n_head, n_tok), block 128.  Scores: two threads per key (4 independent 16-byte loads each); values: each warp takes
// every 4th key, each lane two features, 8 loads in flight.
__global__ void __launch_bounds__(128)
k_attn_self(const float * __restrict__ q, int ldq, const __half * __restrict__ kc, const __half * __restrict__ vc,
            const int * __restrict__ idx, int ld_idx, const int * __restrict__ n_kv, int d, float * __restrict__ out, int ldo) {
    extern __shared__ float sh[];            // qh[64] | sc[ld_idx] | part[4][64]
    __shared__ float red[32];
    const int h = blockIdx.x, t = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nk = n_kv[t];
    float * qh = sh; float * sc = sh + 64; float * part = sc + ((ld_idx + 3) & ~3);
    if (tid < 64) qh[tid] = __half2float(__float2half_rn(q[(int64_t) t * ldq + h * 64 + tid]));
    __syncthreads();
    const int * cells = idx + (int64_t) t * ld_idx;
    float m = -INFINITY;
    for (int k0 = 0; k0 < nk; k0 += 64) {
        const int key = k0 + (tid >> 1), hf = tid & 1;
        float s = 0.0f;
        if (key < nk) {
            const uint4 * k4 = reinterpret_cast<const uint4 *>(kc + (int64_t) cells[key] * d + h * 64 + hf * 32);
            uint4 u[4];
#pragma unroll
            for (int cix = 0; cix < 4; ++cix) u[cix] = k4[cix];
#pragma unroll
            for (int cix = 0; cix < 4; ++cix) {
                const __half2 * hh = reinterpret_cast<const __half2 *>(&u[cix]);
#pragma unroll
                for (int e = 0; e < 4; ++e) { const float2 f = __half22float2(hh[e]); s = fmaf(f.x, qh[hf*32 + cix*8 + 2*e], s); s = fmaf(f.y, qh[hf*32 + cix*8 + 2*e + 1], s); }
            }
        }
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        if (key < nk && hf == 0) sc[key] = s;
        if (key < nk) m = fmaxf(m, s);
    }
    m = block_max(m, red);
    float l = 0.0f;
    for (int i = tid; i < nk; i += 128) { const float p = expf(sc[i] - m); sc[i] = p; l += p; }
    l = block_sum(l, red);
    float a0 = 0.0f, a1 = 0.0f;
    for (int i0 = warp; i0 < nk; i0 += 32) {             // keys i0, i0+4, ... (8 per round)
        __half2 vv[8]; float pr[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const int i = i0 + 4 * u;
            const bool ok = i < nk;
            vv[u] = ok ? *reinterpret_cast<const __half2 *>(vc + (int64_t) cells[i] * d + h * 64 + 2 * lane) : __float2half2_rn(0.0f);
            pr[u] = ok ? sc[i] : 0.0f;
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) { const float2 f = __half22float2(vv[u]); a0 = fmaf(pr[u], f.x, a0); a1 = fmaf(pr[u], f.y, a1); }
    }
    part[warp * 64 + 2 * lane] = a0; part[warp * 64 + 2 * lane + 1] = a1;
    __syncthreads();
    if (tid < 64) out[(int64_t) t * ldo + h * 64 + tid] = (l > 0.0f) ? (part[tid] + part[64 + tid] + part[128 + tid] + part[192 + tid]) / l : 0.0f;
}
void attn_self_decode(const float * q, int ldq, const __half * kc, const __half * vc, const int * idx, int ld_idx,
                      const int * n_kv, int n_tok, int n_head, int d, float * out, int ldo, cudaStream_t st) {
    ProfScope prof(PC_ATTN, st, 0.0, 0.0);
    const size_t smem = (64 + ((ld_idx + 3) & ~3) + 256) * sizeof(float);
    k_attn_self<<<dim3(n_head, n_tok), 128, smem, st>>>(q, ldq, kc, vc, idx, ld_idx, n_kv, d, out, ldo); count_launch();
}

// grid (n_head, n_split, n_tok), block 128.  Split-KV (64 keys per CTA) with an in-kernel combine by the last CTA of each
// (token, head).  Phase 1: two threads per key (32 dims each, 4 independent 16-byte loads); phase 2: each warp owns 16 keys and
// every lane two features, 16 independent 4-byte loads in flight -- the kernel is a pure HBM stream of the cross K/V.
static constexpr int XKEYS = 64;
static constexpr int XSPLIT_MAX = 32;
__global__ void __launch_bounds__(128)
k_attn_cross(const float * __restrict__ q, int ldq, const __half * __restrict__ kc, const __half * __restrict__ vc,
             const int * __restrict__ slot, int64_t slot_stride, int n_keys, int d, float scale,
             float * __restrict__ partial, int * __restrict__ counters, float * __restrict__ out, int ldo) {
    __shared__ float qh[64];
    __shared__ float sc[XKEYS];
    __shared__ float part[4][64];
    __shared__ float red[32];
    __shared__ int   is_last;
    const int h = blockIdx.x, sp = blockIdx.y, t = blockIdx.z, tid = threadIdx.x, n_head = gridDim.x, n_split = gridDim.y;
    const int lane = tid & 31, warp = tid >> 5;
    const int k0 = sp * XKEYS;
    const __half * kb = kc + (int64_t) slot[t] * slot_stride + (int64_t) k0 * d + h * 64;
    const __half * vb = vc + (int64_t) slot[t] * slot_stride + (int64_t) k0 * d + h * 64;
    if (tid < 64) qh[tid] = __half2float(__float2half_rn(q[(int64_t) t * ldq + h * 64 + tid]));
    __syncthreads();
    {   // scores: thread -> (key = tid/2, half = tid%2)
        const int key = tid >> 1, hf = tid & 1;
        float s = 0.0f;
        if (k0 + key < n_keys) {
            const uint4 * k4 = reinterpret_cast<const uint4 *>(kb + (int64_t) key * d + hf * 32);
            uint4 u[4];
#pragma unroll
            for (int cix = 0; cix < 4; ++cix) u[cix] = __ldg(k4 + cix);
#pragma unroll
            for (int cix = 0; cix < 4; ++cix) {
                const __half2 * hh = reinterpret_cast<const __half2 *>(&u[cix]);
#pragma unroll
                for (int e = 0; e < 4; ++e) { const float2 f = __half22float2(hh[e]); s = fmaf(f.x, qh[hf*32 + cix*8 + 2*e], s); s = fmaf(f.y, qh[hf*32 + cix*8 + 2*e + 1], s); }
            }
        }
        s += __shfl_xor_sync(0xffffffffu, s, 1);
        if (hf == 0) sc[key] = (k0 + key < n_keys) ? s * scale : -INFINITY;
    }
    __syncthreads();
    float m = (tid < XKEYS) ? sc[tid] : -INFINITY;
    m = block_max(m, red);
    float pv = 0.0f;
    if (tid < XKEYS) { pv = (sc[tid] > -INFINITY) ? expf(sc[tid] - m) : 0.0f; sc[tid] = pv; }
    const float l = block_sum(pv, red);                        // block_sum ends with every thread past its barriers: sc[] is visible
    {   // out partial: warp w -> keys 16w..16w+15, lane -> features 2*lane, 2*lane+1
        float a0 = 0.0f, a1 = 0.0f;
        __half2 vv[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) {
            const int key = warp * 16 + i;
            vv[i] = (k0 + key < n_keys) ? *reinterpret_cast<const __half2 *>(vb + (int64_t) key * d + 2 * lane) : __float2half2_rn(0.0f);
        }
#pragma unroll
        for (int i = 0; i < 16; ++i) { const float2 f = __half22float2(vv[i]); const float pr = sc[warp * 16 + i]; a0 = fmaf(pr, f.x, a0); a1 = fmaf(pr, f.y, a1); }
        part[warp][2 * lane] = a0; part[warp][2 * lane + 1] = a1;
    }
    __syncthreads();
    float * pp = partial + (((int64_t) t * n_head + h) * XSPLIT_MAX + sp) * 66;
    if (tid < 64) pp[2 + tid] = part[0][tid] + part[1][tid] + part[2][tid] + part[3][tid];
    if (tid == 0) { pp[0] = m; pp[1] = l; }
    __threadfence();
    __syncthreads();
    if (tid == 0) {
        const int prev = atomicAdd(&counters[t * n_head + h], 1);
        is_last = (prev == n_split - 1);
    }
    __syncthreads();
    if (!is_last) return;
    __threadfence();
    const float * p0 = partial + ((int64_t) t * n_head + h) * XSPLIT_MAX * 66;
    float M = -INFINITY;
    for (int s = 0; s < n_split; ++s) M = fmaxf(M, p0[s * 66]);
    if (tid < 64) {
        float L = 0.0f, o = 0.0f;
        for (int s = 0; s < n_split; ++s) {
            const float w = expf(p0[s * 66] - M);
            L = fmaf(p0[s * 66 + 1], w, L);
            o = fmaf(p0[s * 66 + 2 + tid], w, o);
        }
        out[(int64_t) t * ldo + h * 64 + tid] = o / L;
    }
    if (tid == 0) counters[t * n_head + h] = 0;
}
void attn_cross_decode(const float * q, int ldq, const __half * kc, const __half * vc, const int * slot, int64_t slot_stride,
                       int n_keys, int n_tok, int n_head, int d, float scale, float * partial, int * counters,
                       float * out, int ldo, cudaStream_t st) {
    const int n_split = (n_keys + XKEYS - 1) / XKEYS;          // 24 for the padded 1536 keys
    if (n_split > XSPLIT_MAX) { set_error("attn_cross_decode: too many keys (%d)", n_keys); return; }
    ProfScope prof(PC_ATTN, st, (double) n_tok * 2.0 * n_keys * d * 2, 4.0 * n_tok * n_keys * d);
    k_attn_cross<<<dim3(n_head, n_split, n_tok), 128, 0, st>>>(q, ldq, kc, vc, slot, slot_stride, n_keys, d, scale, partial, counters, out, ldo);
    count_launch();
}

} // namespace wb

namespace wb {
// =====================================================================================================================
//  logits filter + greedy pick on the device.  Same rules, same order, same float formulas as whisper_process_logits /
//  whisper_sample_token(best=true) (src/whisper.cpp:6196-6543); only the order of the f32 summations differs, so p/plog can
//  move in the last bits while the chosen ids follow the reference's tie rule (strict >, lowest index).
// =====================================================================================================================
struct SampK { const uint32_t * mask; int eot, beg, nosp, space, suppress_blank, no_ts, max_init; };

__device__ __forceinline__ bool samp_masked(const SampK & c, const uint32_t * smask, int i, int flags, int tid0) {
    if (smask[i >> 5] & (1u << (i & 31))) return true;
    const bool is_initial = flags & 1, last_ts = flags & 2, penult_ts = flags & 4, has_ts = flags & 8, text_off = flags & 16;
    if (is_initial && c.suppress_blank && (i == c.eot || i == c.space)) return true;
    if (c.no_ts && i >= c.beg) return true;
    if (text_off && i < c.eot) return true;
    if (last_ts) { if (penult_ts) { if (i >= c.beg) return true; } else if (i < c.eot) return true; }
    if (is_initial && c.max_init >= 0 && i > c.beg + c.max_init) return true;
    if (has_ts && i >= c.beg && i < c.beg + tid0) return true;
    return false;
}
struct PI { float p; int i; };
__device__ __forceinline__ PI pi_best(PI a, PI b) { return (b.p > a.p || (b.p == a.p && b.i < a.i)) ? b : a; }
__device__ __forceinline__ PI block_best(PI v, PI * scratch) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { PI t; t.p = __shfl_xor_sync(0xffffffffu, v.p, o); t.i = __shfl_xor_sync(0xffffffffu, v.i, o); v = pi_best(v, t); }
    __syncthreads();
    if (lane == 0) scratch[warp] = v;
    __syncthreads();
    PI r = (lane < nw) ? scratch[lane] : PI{ -1.0f, 0x7fffffff };
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { PI t; t.p = __shfl_xor_sync(0xffffffffu, r.p, o); t.i = __shfl_xor_sync(0xffffffffu, r.i, o); r = pi_best(r, t); }
    return r;
}

__global__ void __launch_bounds__(1024)
k_greedy_sample(const float * __restrict__ logits, int V, const int * __restrict__ rowinfo, const SampK c, SampOut * __restrict__ out,
                const double * __restrict__ draws, int stride) {
    extern __shared__ uint32_t smask[];
    __shared__ float red[32];
    __shared__ PI redpi[32];
    __shared__ SampOut srow;
    const int row = blockIdx.x, tid = threadIdx.x;
    const float * l = logits + (int64_t) row * V;
    const int flags = rowinfo[2 * row], tid0 = rowinfo[2 * row + 1];
    for (int i = tid; i < (V + 31) / 32; i += blockDim.x) smask[i] = c.mask[i];
    __syncthreads();
    // pass 1: maxima (raw for no_speech_prob; masked overall / text / timestamps)
    float raw_max = -INFINITY, m_max = -INFINITY, ts_max = -INFINITY, text_max = -INFINITY;
    for (int i = tid; i < V; i += blockDim.x) {
        const float v = l[i];
        raw_max = fmaxf(raw_max, v);
        if (!samp_masked(c, smask, i, flags, tid0)) { m_max = fmaxf(m_max, v); if (i >= c.beg) ts_max = fmaxf(ts_max, v); else text_max = fmaxf(text_max, v); }
    }
    raw_max = block_max(raw_max, red); m_max = block_max(m_max, red); ts_max = block_max(ts_max, red); text_max = block_max(text_max, red);
    // pass 2: sums
    float raw_sum = 0.0f, m_sum = 0.0f, ts_sum = 0.0f;
    for (int i = tid; i < V; i += blockDim.x) {
        const float v = l[i];
        raw_sum += expf(v - raw_max);
        if (!samp_masked(c, smask, i, flags, tid0)) { m_sum += expf(v - m_max); if (i >= c.beg) ts_sum += expf(v - ts_max); }
    }
    raw_sum = block_sum(raw_sum, red); m_sum = block_sum(m_sum, red); ts_sum = block_sum(ts_sum, red);
    const float lse = ::logf(m_sum) + m_max;
    // "timestamp mass beats every text token" rule (whisper.cpp:6361-6388); evaluated on log-probabilities like the reference
    bool text_off = false;
    if (ts_sum > 0.0f) {
        const float ts_lp = ::logf(ts_sum) + (ts_max - lse);
        text_off = ts_lp > (text_max - lse);
    }
    // pass 3: probabilities, greedy pick, timestamp statistics
    PI best = { 0.0f, 0x7fffffff }, best_ts = { 0.0f, 0x7fffffff };
    double sum_ts = 0.0;
    for (int i = tid; i < V; i += blockDim.x) {
        if (samp_masked(c, smask, i, flags, tid0) || (text_off && i < c.beg)) continue;
        const float pr = expf(l[i] - lse);
        if (pr > best.p) best = { pr, i };
        if (i >= c.beg) { sum_ts += pr; if (pr > best_ts.p) best_ts = { pr, i }; }
    }
    best = block_best(best, redpi);
    best_ts = block_best(best_ts, redpi);
    const float sts = block_sum((float) sum_ts, red);
    if (tid == 0) {
        SampOut o;
        o.id = best.p > 0.0f ? best.i : 0;                       // result.id starts at 0 and only moves on a strictly larger prob
        o.p = best.p > 0.0f ? best.p : 0.0f;
        o.plog = best.p > 0.0f ? l[o.id] - lse : 0.0f;
        o.tid = best_ts.p > 0.0f ? best_ts.i : 0;
        o.pt = (float) ((double) (best_ts.p > 0.0f ? best_ts.p : 0.0f) / ((double) sts + 1e-10));
        o.ptsum = sts;
        if (o.id >= c.beg) { o.tid = o.id; o.pt = o.p; }
        o.nosp_raw = expf(l[c.nosp] - (::logf(raw_sum) + raw_max));
        o.raw_max = raw_max; o.raw_sum = raw_sum; o.raw_nosp = l[c.nosp];
        out[(int64_t) row * stride] = o;
        srow = o;
    }
    // ---- categorical draws (whisper_sample_token_topk, src/whisper.cpp:6545-6618 = k draws of std::discrete_distribution over probs).
    // libstdc++ normalises the probabilities by their sum (double), forms the running sums cp[i] (last one forced to 1) and returns
    // lower_bound(cp, u) for a uniform u in [0, 1): the number of cp[i] < u.  The uniforms come from the host (the decoder's own
    // mt19937 through std::generate_canonical<double, 53>, the same numbers the reference consumes); here every thread owns a
    // contiguous slice of the vocabulary, the slices are chained by a scan in double, and each draw is a count.  Only the association
    // of the double sums differs from the sequential loop (relative 1e-16: a draw changes only if u falls that close to a boundary).
    const int nd = (flags >> 8) & 0x7f;
    if (nd > 0) {
        __shared__ double sc[1024];
        __shared__ int scnt[64];
        const int S = (V + blockDim.x - 1) / blockDim.x, i0 = tid * S, i1 = min(V, i0 + S);
        auto prob = [&](int i) -> float { return (samp_masked(c, smask, i, flags, tid0) || (text_off && i < c.beg)) ? 0.0f : expf(l[i] - lse); };
        double ls = 0.0;
        for (int i = i0; i < i1; ++i) ls += (double) prob(i);
        __syncthreads();
        sc[tid] = ls;
        __syncthreads();
        for (int o = blockDim.x >> 1; o > 0; o >>= 1) { if (tid < o) sc[tid] += sc[tid + o]; __syncthreads(); }
        const double total = sc[0];
        __syncthreads();
        double ln = 0.0;
        for (int i = i0; i < i1; ++i) ln += (double) prob(i) / total;
        sc[tid] = ln;
        __syncthreads();
        for (int o = 1; o < (int) blockDim.x; o <<= 1) {           // inclusive scan (Hillis-Steele)
            const double add = tid >= o ? sc[tid - o] : 0.0;
            __syncthreads();
            sc[tid] += add;
            __syncthreads();
        }
        const double base = sc[tid] - ln;
        for (int q0 = 0; q0 < nd; q0 += 8) {
            if (tid < 64) scnt[tid] = 0;
            __syncthreads();
            double u[8]; int cnt[8];
#pragma unroll
            for (int q = 0; q < 8; ++q) { u[q] = (q0 + q < nd) ? draws[(int64_t) row * stride + q0 + q] : -1.0; cnt[q] = 0; }
            double run = base;
            for (int i = i0; i < i1; ++i) {
                run += (double) prob(i) / total;
                if (i != V - 1) {
#pragma unroll
                    for (int q = 0; q < 8; ++q) cnt[q] += (run < u[q]) ? 1 : 0;
                }
            }
#pragma unroll
            for (int q = 0; q < 8; ++q) if (cnt[q]) atomicAdd(&scnt[q], cnt[q]);
            __syncthreads();
            if (tid < 8 && q0 + tid < nd) {
                const int id = min(scnt[tid], V - 1);
                SampOut o = srow;                                        // row-level fields (written by thread 0 before the barriers above)
                o.id = id; o.p = prob(id); o.plog = l[id] - lse;
                o.tid = best_ts.p > 0.0f ? best_ts.i : c.beg;           // timestamp_stats starts from tid = token_beg in the top-k sampler
                o.pt = (float) ((double) (best_ts.p > 0.0f ? best_ts.p : 0.0f) / ((double) sts + 1e-10));
                o.ptsum = sts;
                if (o.id >= c.beg) { o.tid = o.id; o.pt = o.p; }
                out[(int64_t) row * stride + q0 + tid] = o;
            }
            __syncthreads();
        }
    }
}
void greedy_sample(const float * logits, int V, int n, const int * rowinfo, const SampCfg & cfg, SampOut * out, cudaStream_t st, const double * draws, int stride) {
    SampK c; c.mask = cfg.mask; c.eot = cfg.token_eot; c.beg = cfg.token_beg; c.nosp = cfg.token_nosp; c.space = cfg.space_id;
    c.suppress_blank = cfg.suppress_blank; c.no_ts = cfg.no_timestamps; c.max_init = cfg.max_initial_tid;
    const size_t smem = (size_t) ((V + 31) / 32) * 4;
    k_greedy_sample<<<n, 1024, smem, st>>>(logits, V, rowinfo, c, out, draws, stride < 1 ? 1 : stride); count_launch();
}

} // namespace wb
