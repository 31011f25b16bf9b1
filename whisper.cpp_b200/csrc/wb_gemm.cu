// wb_gemm.cu -- the wgmma GEMM used by every dense contraction of the encode path
// (conv stem, encoder QKV/O/MLP, cross K/V, attention scores and PV in the unfused path, decoder prompt).
//
// One CTA computes 128 (weight rows) x BN (activation rows) tiles, three warpgroups:
//   warpgroup 0    : producer   -- thread 0 streams the B tile (and the A tile for f16 weights) into a STAGES-deep smem ring by TMA;
//                                  for quantised A (first-generation launch) all 128 threads decode one weight row each (2 x 32-value
//                                  blocks per 64-wide k-block) into the 128B-swizzled K-major operand tile
//   warpgroups 1-2 : consumers  -- each owns 64 of the 128 weight rows: 4 x wgmma m64nBNk16 per k-block with the f32 accumulator in
//                                  registers, then the epilogue (bias / scale / GELU / residual), staged through shared memory in 8 KB
//                                  chunks and written with 16-byte stores
// setmaxnreg moves registers from the producer warpgroup (40, 96 when it decodes quantised rows) to the consumers (232 / 200): no spills.
// The epilogue kind (EpiKind) is a template parameter chosen at the launch site.
// The same kernel serves the first-generation launch (one tile per CTA, quantised weights decoded in the kernel) and the persistent one
// (gridDim = number of SMs, each CTA walks the tile list, weight-tile index fastest so that concurrently running CTAs share activation
// tiles in L2; quantised weights expanded to f16 beforehand by k_dequant_f16, both operands through TMA).  The producer runs ahead into the
// next tile's k-blocks while the consumers run the epilogue of the current one.
// Layout facts relied on:
//   * K-major SW128 tile: row r at byte r*128, 16-byte chunk c stored at chunk (c ^ (r & 7)); 8-row groups 1024 B apart
//   * wgmma accumulator: thread t of the warpgroup holds rows 16*(t/32) + (t%32)/4 (+8) and columns 8*j + 2*(t%4) (+1)
#include <algorithm>
#include <type_traits>
#include "wb_gemm.cuh"
#include "wb_ptx.cuh"
#include "wb_common.h"

namespace wb {

static constexpr int GEMM_THREADS  = 384;
static constexpr int A_TILE_BYTES  = 128 * 64 * 2;
// epilogue staging, per consumer warpgroup: one 8 KB chunk of output lines (see gemm_epilogue_regs) plus 16 bytes of padding per line,
// so that the fragment writes of a warp spread over the banks
static constexpr int EPI_STAGE_BYTES = 64 * (128 + 16);

template <int BN> struct GemmCfg {
    static constexpr int B_TILE_BYTES = BN * 64 * 2;
    static constexpr int STAGES = (BN == 256) ? 4 : (BN == 128 ? 6 : 8);
    static constexpr int SMEM   = STAGES * (A_TILE_BYTES + B_TILE_BYTES) + 1024 /*align slack*/ + 256 /*barriers*/ + 2 * EPI_STAGE_BYTES;
};

struct GemmKParams {
    int M, N, K, taps, nkb_per_tap, nb0;
    int a_zsel0, a_zsel1, b_zsel0, b_zsel1, a_rows_per_b0, b1_in_off;
    int n_mt, n_nt, n_tiles;        // tile list: weight tile fastest, then activation tile, then batch index
    int b_split;                    // 2: the B tensor map's box holds BN / 2 rows (the tile is fetched in two halves)
    // quantised A
    const void * a_base; const uint8_t * a_qs; const uint32_t * a_qh; const __half * a_d; const __half * a_m;
    GemmEpilogue ep;
};

__device__ __forceinline__ float gelu_ref_f16(float x) {
    // ggml CPU: table lookup on the f16-rounded input, table entries are f16(gelu(f32(x16)))  (vec.h:988-1001, ggml-cpu.c:3847).
    // Evaluated as x * sigmoid(2u) = 0.5 x (1 + tanh u) with ex2.approx + rcp.approx (a dozen instructions; tanhf made the FC1 epilogue
    // longer than its main loop).  Against the table: identical for 98.7 % of all f16 inputs, one f16 ulp of a value below 1e-2 in
    // magnitude for the rest (x < -2, where the reference's own 1 + tanhf(u) cancels) -- checked over all 37376 inputs in (-10, 10).
    if (x <= -10.0f) return 0.0f;
    if (x >=  10.0f) return x;
    const float xh = __half2float(__float2half_rn(x));
    const float e  = __expf(-1.5957691216057308f * xh * (1.0f + 0.044715f * xh * xh));
    return __half2float(__float2half_rn(__fdividef(xh, 1.0f + e)));
}

struct RawBlk { uint4 q0, q1; uint32_t qh; __half d, m; };

template <int WT>
__device__ __forceinline__ void raw_load(const GemmKParams & p, int m, int k, RawBlk & r, bool valid) {
    if (!valid) { r.q0 = r.q1 = make_uint4(0, 0, 0, 0); r.qh = 0; r.d = __float2half(0.0f); return; }
    const int64_t nblk = (int64_t) p.K >> 5;
    const int64_t bi   = (int64_t) m * nblk + (k >> 5);
    if (WT == WT_Q4_0 || WT == WT_Q5_0 || WT == WT_Q4_1 || WT == WT_Q5_1) {
        r.q0 = __ldg(reinterpret_cast<const uint4 *>(p.a_qs) + bi);
        if (wt_has_qh(WT)) r.qh = __ldg(p.a_qh + bi);
        r.d = p.a_d[bi];
        if (wt_has_min(WT)) r.m = p.a_m[bi];
    } else if (WT == WT_Q8_0) {
        r.q0 = __ldg(reinterpret_cast<const uint4 *>(p.a_qs) + 2*bi);
        r.q1 = __ldg(reinterpret_cast<const uint4 *>(p.a_qs) + 2*bi + 1);
        r.d = p.a_d[bi];
    }
}

// Epilogue kinds: chosen on the host from the GemmEpilogue (epi_kind), so that the kernel carries no per-element flag tests.
enum EpiKind : int {
    EPI_F16          = 0,   // (acc + bias) * scl -> f16 out[n][m]                          (QK, cross K/V token-major)
    EPI_F16_GELU     = 1,   // GELU(acc * scl + bias * scl) -> f16 out[n][m]               (FC1, conv1)
    EPI_F32_RES      = 2,   // acc * scl + bias * scl + res[n][m] -> f32 out[n][m]         (attention-O, FC2: in place on the residual stream)
    EPI_F16_MMAJOR   = 3,   // (acc + bias) * scl -> f16 out[m][n]                          (V^T)
    EPI_F16_HM       = 4,   // (acc + bias) * scl -> f16 out[m / 64][n][m % 64]             (cross K/V head-major)
    EPI_GENERAL      = 5,   // every flag of GemmEpilogue tested per value                  (conv2, the unfused attention, the test hook)
};

static EpiKind epi_kind(const GemmEpilogue & e) {
    const bool plain = !e.res && !e.out_mmajor && e.hm_rows == 0;
    if (e.out_f16 && plain && e.act == 0) return EPI_F16;
    if (e.out_f16 && plain && e.act == 1) return EPI_F16_GELU;
    if (e.res && !e.out_mmajor && !e.out_f16 && e.act == 0) return EPI_F32_RES;
    if (e.out_f16 && e.out_mmajor && !e.res && e.act == 0) return EPI_F16_MMAJOR;
    if (e.out_f16 && e.hm_rows > 0 && !e.out_mmajor && !e.res && e.act == 0) return EPI_F16_HM;
    return EPI_GENERAL;
}

// the value of one accumulator (weight row m, activation row n) after the epilogue arithmetic of kind EK; bias and scl belong to row m
template <int EK>
__device__ __forceinline__ float epilogue_value(const GemmEpilogue & e, int64_t roff, int m, int n, float v, float bias, float scl) {
    if constexpr (EK == EPI_F32_RES) {
        return fmaf(v, scl, bias * scl) + __ldcg(e.res + roff + (int64_t) n * e.ldr + m);
    } else if constexpr (EK == EPI_F16_GELU) {
        // GELU with the reference's f16 table semantics, a dozen instructions per value: see gelu_ref_f16 for the formula and its accuracy
        float x = __half2float(__float2half_rn(fmaf(v, scl, bias * scl)));
        x = fmaxf(x, -20.0f);                                           // gelu = 0 below -10 either way; keeps exp finite
        const float ex = __expf(x * fmaf(x * x, -0.07135481627f, -1.5957691216f));
        return __fdividef(x, 1.0f + ex);
    } else {
        return (v + bias) * scl;
    }
}

// one accumulator value through the general epilogue: every flag tested, the residual and GELU kinds recognised per value (the
// first-generation launch with quantised weights uses this for all kinds)
__device__ __forceinline__ void epilogue_elem_general(const GemmEpilogue & e, int64_t ooff, int64_t roff, int m, int n, float v, float bias, float scl) {
    if (e.res && !e.out_mmajor && !e.out_f16 && e.act == 0) {
        reinterpret_cast<float *>(e.out)[ooff + (int64_t) (n + e.n_row_off) * e.ldo + m] = epilogue_value<EPI_F32_RES>(e, roff, m, n, v, bias, scl);
        return;
    }
    if (e.act == 1 && e.out_f16 && !e.res && !e.out_mmajor && e.hm_rows == 0) {
        reinterpret_cast<__half *>(e.out)[ooff + (int64_t) (n + e.n_row_off) * e.ldo + m] = __float2half_rn(epilogue_value<EPI_F16_GELU>(e, roff, m, n, v, bias, scl));
        return;
    }
    float x = (v + bias) * scl;
    if (e.act == 1) x = gelu_ref_f16(x);
    if (e.res) x += e.res[roff + (int64_t) n * e.ldr + m];
    if (e.out_mmajor) {
        if (e.out_f16) reinterpret_cast<__half *>(e.out)[ooff + (int64_t) m * e.ldo + n] = __float2half_rn(x);
        else           reinterpret_cast<float *>(e.out)[ooff + (int64_t) m * e.ldo + n] = x;
    } else if (e.out_f16 && e.hm_rows > 0) {                           // head-major: 64 consecutive features of a key are one 128-byte row
        reinterpret_cast<__half *>(e.out)[ooff + (int64_t) (m >> 6) * e.hm_rows * 64 + (int64_t) (n + e.n_row_off) * 64 + (m & 63)] = __float2half_rn(x);
    } else if (e.out_f16) {
        reinterpret_cast<__half *>(e.out)[ooff + (int64_t) (n + e.n_row_off) * e.ldo + m] = __float2half_rn(x);
    } else {
        reinterpret_cast<float *>(e.out)[ooff + (int64_t) (n + e.n_row_off) * e.ldo + m] = x;
    }
}

template <typename T> __device__ __forceinline__ void store_pair(T * o, float lo, float hi);
template <> __device__ __forceinline__ void store_pair<__half>(__half * o, float lo, float hi) { *reinterpret_cast<__half2 *>(o) = __floats2half2_rn(lo, hi); }
template <> __device__ __forceinline__ void store_pair<float>(float * o, float lo, float hi) { *reinterpret_cast<float2 *>(o) = make_float2(lo, hi); }
template <typename T> __device__ __forceinline__ T from_f32(float x);
template <> __device__ __forceinline__ __half from_f32<__half>(float x) { return __float2half_rn(x); }
template <> __device__ __forceinline__ float  from_f32<float>(float x)  { return x; }

// epilogue of the 64 x BN accumulator of one consumer warpgroup (rows m0 .. m0 + 63 of the weight side, columns n0 .. n0 + BN - 1).
// Bias and scale are loaded once per row.  The general kind stores each value from its fragment position; the others go through the
// warpgroup's staging buffer `stage` (below).  Only the grouping of the stores differs between the two: every value is computed by the
// formula of its kind.
template <int BN, int EK>
__device__ __forceinline__ void gemm_epilogue_regs(const GemmKParams & p, const float (&acc)[BN / 2], int m0, int n0, int b0, int b1, int t,
                                                   uint8_t * stage) {
    const GemmEpilogue & e = p.ep;
    const int64_t ooff = (int64_t) b0 * e.out_b0 + (int64_t) b1 * e.out_b1;
    const int64_t roff = (int64_t) b0 * e.res_b0 + (int64_t) b1 * e.res_b1;
    if constexpr (EK == EPI_GENERAL) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = m0 + 16 * (t >> 5) + ((t & 31) >> 2) + 8 * h;
            if (m >= p.M) continue;
            const int mg = m + b0 * p.a_rows_per_b0;                    // bias / scale follow the stacked-matrix row
            const float bias = e.bias_m ? e.bias_m[mg] : 0.0f;
            const float scl  = (e.scale_m ? e.scale_m[mg] : 1.0f) * e.alpha;
#pragma unroll
            for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
                for (int c = 0; c < 2; ++c) {
                    const int n = n0 + 8 * j + 2 * (t & 3) + c;
                    if (n < p.N) epilogue_elem_general(e, ooff, roff, m, n, acc[4 * j + 2 * h + c], bias, scl);
                }
            }
        }
    } else {
        // Through shared memory: the warpgroup's 64 x BN block goes out in chunks of 8 KB.  A chunk is a set of output lines that are
        // contiguous in global memory: for the n-major kinds one line = one activation row n with the warpgroup's 64 weight rows
        // (64 f16 = 128 B, or 64 f32 = 256 B; 64 or 32 lines per chunk), for the m-major kind one line = one weight row m with 64
        // columns n (128 B; 64 lines).  The fragments are written into the chunk, then the warpgroup copies it out with 16-byte stores.
        using OutT = typename std::conditional<EK == EPI_F32_RES, float, __half>::type;
        constexpr bool MMAJ  = (EK == EPI_F16_MMAJOR);
        constexpr int  VB    = (int) sizeof(OutT);                        // bytes per value
        constexpr int  VEC   = 16 / VB;                                   // values per 16-byte vector
        constexpr int  LB    = 64 * VB;                                   // line bytes
        constexpr int  LS    = LB + 16;                                   // line stride in shared memory
        constexpr int  CN    = MMAJ ? 64 : 8192 / LB;                     // columns n per chunk
        constexpr int  LINES = MMAJ ? 64 : CN;
        static_assert(LINES * LS <= EPI_STAGE_BYTES, "epilogue chunk does not fit its staging buffer");
        constexpr int  NCH   = (BN > CN) ? BN / CN : 1;
        constexpr int  CJ    = ((BN < CN) ? BN : CN) / 8;                 // accumulator column groups per chunk
        OutT * out = reinterpret_cast<OutT *>(e.out) + ooff;
        const int bar_id = threadIdx.x >> 7;                              // one named barrier per consumer warpgroup (ids 1, 2)
        // 16-byte accesses need every line start on a 16-byte boundary
        bool vec = ((reinterpret_cast<uintptr_t>(e.out) & 15) == 0) && (ooff % VEC) == 0 && (EK == EPI_F16_HM || (e.ldo % VEC) == 0);
        if constexpr (EK == EPI_F32_RES)
            vec = vec && ((reinterpret_cast<uintptr_t>(e.res) & 15) == 0) && (roff % VEC) == 0 && (e.ldr % VEC) == 0;
        const int odd = (t >> 2) & 1;                                     // parity of this lane's rows (m0 is a multiple of 64)
        float bias[2], scl[2];
        bool mval[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = m0 + 16 * (t >> 5) + ((t & 31) >> 2) + 8 * h;
            mval[h] = m < p.M;
            const int mg = m + b0 * p.a_rows_per_b0;                      // bias / scale follow the stacked-matrix row
            bias[h] = (mval[h] && e.bias_m) ? e.bias_m[mg] : 0.0f;
            scl[h]  = ((mval[h] && e.scale_m) ? e.scale_m[mg] : 1.0f) * e.alpha;
        }
#pragma unroll
        for (int c = 0; c < NCH; ++c) {
            bar_named(bar_id, 128);                                       // the previous chunk has been copied out
#pragma unroll
            for (int jj = 0; jj < CJ; ++jj) {
                const int j = c * CJ + jj;
                const int n = n0 + 8 * j + 2 * (t & 3);
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int ml = 16 * (t >> 5) + ((t & 31) >> 2) + 8 * h;   // row inside the warpgroup's 64
                    const int m = m0 + ml;
                    float x0 = acc[4 * j + 2 * h], x1 = acc[4 * j + 2 * h + 1];
                    // the residual is added in the copy-out (same f32 addition, same operands)
                    constexpr int VK = (EK == EPI_F32_RES) ? -1 : EK;
                    if (mval[h] && n < p.N) {
                        if constexpr (VK < 0) x0 = fmaf(x0, scl[h], bias[h] * scl[h]);
                        else                  x0 = epilogue_value<EK>(e, roff, m, n, x0, bias[h], scl[h]);
                    }
                    if (mval[h] && n + 1 < p.N) {
                        if constexpr (VK < 0) x1 = fmaf(x1, scl[h], bias[h] * scl[h]);
                        else                  x1 = epilogue_value<EK>(e, roff, m, n + 1, x1, bias[h], scl[h]);
                    }
                    if constexpr (MMAJ) {
                        store_pair<OutT>(reinterpret_cast<OutT *>(stage + ml * LS) + 8 * jj + 2 * (t & 3), x0, x1);
                    } else {
                        // lanes t and t ^ 4 hold rows ml, ml ^ 1 of columns n, n + 1: after one exchange the even row's lane holds column n
                        // of both rows and the odd row's lane column n + 1, i.e. two adjacent values of one line
                        const float recv = __shfl_xor_sync(0xffffffffu, odd ? x0 : x1, 4);
                        const float lo = odd ? recv : x0, hi = odd ? x1 : recv;
                        store_pair<OutT>(reinterpret_cast<OutT *>(stage + (8 * jj + 2 * (t & 3) + odd) * LS) + (ml - odd), lo, hi);
                    }
                }
            }
            bar_named(bar_id, 128);                                       // the chunk is complete
            constexpr int VPL = LB / 16;                                  // vectors per line
#pragma unroll
            for (int v = t; v < LINES * VPL; v += 128) {
                const int line = v / VPL, q = v % VPL;
                const OutT * src = reinterpret_cast<const OutT *>(stage + line * LS + q * 16);
                OutT * dst;
                int lim;                                                  // valid values of this vector
                int64_t rrow = 0;
                if constexpr (MMAJ) {
                    const int m = m0 + line, n = n0 + c * CN + q * VEC;
                    if (m >= p.M) continue;
                    dst = out + (int64_t) m * e.ldo + n;
                    lim = p.N - n;
                } else {
                    const int n = n0 + c * CN + line, m = m0 + q * VEC;
                    if (n >= p.N) continue;
                    dst = (EK == EPI_F16_HM) ? out + (int64_t) (m >> 6) * e.hm_rows * 64 + (int64_t) (n + e.n_row_off) * 64 + (m & 63)
                                             : out + (int64_t) (n + e.n_row_off) * e.ldo + m;
                    lim = p.M - m;
                    rrow = roff + (int64_t) n * e.ldr + m;
                }
                if (lim <= 0) continue;
                if constexpr (EK == EPI_F32_RES) {
                    float4 x = *reinterpret_cast<const float4 *>(src);
                    if (vec && lim >= VEC) {
                        const float4 r = __ldcg(reinterpret_cast<const float4 *>(e.res + rrow));
                        x.x += r.x; x.y += r.y; x.z += r.z; x.w += r.w;
                        *reinterpret_cast<float4 *>(dst) = x;
                    } else {
                        const float xs[4] = { x.x, x.y, x.z, x.w };
                        for (int i = 0; i < VEC && i < lim; ++i) dst[i] = xs[i] + __ldcg(e.res + rrow + i);
                    }
                } else {
                    if (vec && lim >= VEC) *reinterpret_cast<uint4 *>(dst) = *reinterpret_cast<const uint4 *>(src);
                    else for (int i = 0; i < VEC && i < lim; ++i) dst[i] = src[i];
                }
            }
        }
    }
}

template <int BN, int WT, int EK>
__global__ void __launch_bounds__(GEMM_THREADS, 1)
gemm_kernel(const GemmKParams p, const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB) {
    using Cfg = GemmCfg<BN>;
    constexpr int STAGES = Cfg::STAGES;
    constexpr bool QUANT = (WT != WT_F16);
    // register split: the producer warpgroup (one TMA thread, or 128 row decoders for quantised weights) gives registers to the two
    // consumer warpgroups, which hold BN / 2 accumulators each.  128 * P + 256 * C = 64512 = 384 * 168, the budget at launch.
    constexpr int REGS_PRODUCER = QUANT ? 96 : 40;
    constexpr int REGS_CONSUMER = QUANT ? 200 : 232;
    static_assert(128 * REGS_PRODUCER + 256 * REGS_CONSUMER <= 384 * 168, "register split over budget");

    extern __shared__ uint8_t smem_raw[];
    uint8_t * smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
    uint8_t * sA = smem;
    uint8_t * sB = smem + STAGES * A_TILE_BYTES;
    uint64_t * bars      = reinterpret_cast<uint64_t *>(sB + STAGES * Cfg::B_TILE_BYTES);
    uint64_t * full_bar  = bars;
    uint64_t * empty_bar = bars + STAGES;

    const int warp = threadIdx.x >> 5;
    const int lane = threadIdx.x & 31;
    const int wg   = threadIdx.x >> 7;
    const int nkb  = p.taps * p.nkb_per_tap;

    if (threadIdx.x == 0) {
        tma_prefetch_desc(&tmB);
        if (!QUANT) tma_prefetch_desc(&tmA);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], QUANT ? 1 + 4 : 1);      // TMA thread (+ the 4 decoder warps)
            mbar_init(&empty_bar[s], 8);                     // the 8 consumer warps
        }
        mbar_fence_init();
    }
    __syncthreads();

    if (wg == 0) {
        // ------------------------------------------------------------------ producer warpgroup
        reg_dealloc<REGS_PRODUCER>();                        // all four warps, before any of them leaves
        if (!QUANT && warp != 0) return;
        const int row = threadIdx.x;                         // QUANT: weight row of the tile this thread decodes
        int s = 0; uint32_t ph = 0;
        for (int t = blockIdx.x; t < p.n_tiles; t += gridDim.x) {
            const int mt = t % p.n_mt, r = t / p.n_mt, nt = r % p.n_nt, z = r / p.n_nt;
            const int b0 = z % p.nb0, b1 = z / p.nb0;
            const int m0 = mt * 128, mg0 = m0 + b0 * p.a_rows_per_b0, n0 = nt * BN;
            if (warp == 0 && p.ep.res && lane > 0) {
                // the residual tile (f32, 128 features of BN rows) goes to L2 while the tile's main loop runs: the epilogue then adds it at L2
                // latency instead of stalling on HBM
                const int mw = min(128, p.M - m0);
                const float * rp = p.ep.res + (int64_t) b0 * p.ep.res_b0 + (int64_t) b1 * p.ep.res_b1 + m0;
                if (mw > 0 && (mw & 3) == 0 && ((reinterpret_cast<uintptr_t>(rp) | ((uintptr_t) p.ep.ldr * 4)) & 15) == 0)
                    for (int rr = lane - 1; rr < BN && n0 + rr < p.N; rr += 31)
                        asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" :: "l"(rp + (int64_t) (n0 + rr) * p.ep.ldr), "r"(mw * 4) : "memory");
            }
            const int m = mg0 + row;                         // QUANT: global row in the (stacked) weight matrix
            const bool mval = (m0 + row) < p.M;
            for (int kb = 0; kb < nkb; ++kb) {
                const int tap = kb / p.nkb_per_tap;
                const int k0  = (kb - tap * p.nkb_per_tap) * 64;
                if (threadIdx.x == 0) {
                    mbar_wait(&empty_bar[s], ph ^ 1);
                    mbar_arrive_expect_tx(&full_bar[s], Cfg::B_TILE_BYTES + (QUANT ? 0 : A_TILE_BYTES));
                    const int sel[4] = { 0, b0, b1 + p.b1_in_off, tap };
                    const int bh = BN / p.b_split;
                    for (int i = 0; i < p.b_split; ++i)
                        tma_load_4d(sB + s * Cfg::B_TILE_BYTES + i * bh * 128, &tmB, &full_bar[s], k0, n0 + i * bh, sel[p.b_zsel0], sel[p.b_zsel1]);
                    if (!QUANT)
                        tma_load_4d(sA + s * A_TILE_BYTES, &tmA, &full_bar[s], k0, mg0, sel[p.a_zsel0], sel[p.a_zsel1]);
                }
                if (QUANT) {
                    uint4 o[8];
#pragma unroll
                    for (int hf = 0; hf < 2; ++hf) {
                        const int k = kb * 64 + hf * 32;
                        uint4 * oh = o + 4 * hf;
                        if (!(mval && k < p.K)) {
                            oh[0] = oh[1] = oh[2] = oh[3] = make_uint4(0, 0, 0, 0);
                        } else if (WT == WT_Q4_K || WT == WT_Q5_K) {
                            constexpr int BLK = (WT == WT_Q4_K) ? 144 : 176;
                            const uint8_t * rowp = reinterpret_cast<const uint8_t *>(p.a_base) + (int64_t) m * (p.K >> 8) * BLK;
                            uint4 q[4];
                            dequant_kq_sub<WT == WT_Q5_K>(rowp + (int64_t) (k >> 8) * BLK, (k & 255) >> 5, q);
                            oh[0] = q[0]; oh[1] = q[1]; oh[2] = q[2]; oh[3] = q[3];
                        } else if (WT == WT_Q3_K) {
                            const uint8_t * rowp = reinterpret_cast<const uint8_t *>(p.a_base) + (int64_t) m * (p.K >> 8) * 110;
                            uint4 q[4];
                            dequant_q3k_sub(rowp + (int64_t) (k >> 8) * 110, (k & 255) >> 5, q);
                            oh[0] = q[0]; oh[1] = q[1]; oh[2] = q[2]; oh[3] = q[3];
                        } else {
                            RawBlk rb; uint4 q[4];
                            raw_load<WT>(p, m, k, rb, true);
                            if (WT == WT_Q4_0)      dequant_q4_0(rb.q0, rb.d, q);
                            else if (WT == WT_Q5_0) dequant_q5_0(rb.q0, rb.qh, rb.d, q);
                            else if (WT == WT_Q4_1) dequant_q4_1(rb.q0, rb.d, rb.m, q);
                            else if (WT == WT_Q5_1) dequant_q5_1(rb.q0, rb.qh, rb.d, rb.m, q);
                            else                    dequant_q8_0(rb.q0, rb.q1, rb.d, q);
                            oh[0] = q[0]; oh[1] = q[1]; oh[2] = q[2]; oh[3] = q[3];
                        }
                    }
                    mbar_wait(&empty_bar[s], ph ^ 1);
                    uint8_t * d = sA + s * A_TILE_BYTES + row * 128;
#pragma unroll
                    for (int c = 0; c < 8; ++c)
                        *reinterpret_cast<uint4 *>(d + ((c ^ (row & 7)) << 4)) = o[c];
                    fence_proxy_async_smem();
                    __syncwarp();
                    if (lane == 0) mbar_arrive(&full_bar[s]);
                }
                if (++s == STAGES) { s = 0; ph ^= 1; }
            }
            __syncwarp();
        }
        return;
    }

    // ------------------------------------------------------------------ consumer warpgroups
    reg_alloc<REGS_CONSUMER>();
    const int cw = wg - 1;                                   // rows 64*cw .. 64*cw + 63 of each 128-row weight tile
    uint8_t * epi_stage = reinterpret_cast<uint8_t *>(bars) + 256 + cw * EPI_STAGE_BYTES;
    const int t128 = threadIdx.x & 127;
    float acc[BN / 2];
    int s = 0; uint32_t ph = 0;
    for (int t = blockIdx.x; t < p.n_tiles; t += gridDim.x) {
        const int mt = t % p.n_mt, r = t / p.n_mt, nt = r % p.n_nt, z = r / p.n_nt;
        const int b0 = z % p.nb0, b1 = z / p.nb0;
        int s_prev = -1;
        for (int kb = 0; kb < nkb; ++kb) {
            mbar_wait(&full_bar[s], ph);
            wgmma_fence();
            const uint64_t adesc = wgmma_desc_sw128(smem_u32(sA + s * A_TILE_BYTES + cw * 64 * 128));
            const uint64_t bdesc = wgmma_desc_sw128(smem_u32(sB + s * Cfg::B_TILE_BYTES));
#pragma unroll
            for (int k = 0; k < 4; ++k)                      // +32 bytes per K=16 step inside the swizzle atom: +2 in the (addr >> 4) field
                wgmma_f16_ss<BN>(acc, adesc + 2*k, bdesc + 2*k, (kb | k) ? 1u : 0u);
            wgmma_commit();
            wgmma_wait<1>();                                 // the previous k-block's MMAs are done: its stage can be refilled
            wgmma_fence_regs(acc);
            if (s_prev >= 0 && lane == 0) mbar_arrive(&empty_bar[s_prev]);
            s_prev = s;
            if (++s == STAGES) { s = 0; ph ^= 1; }
        }
        wgmma_wait<0>();
        wgmma_fence_regs(acc);
        if (s_prev >= 0 && lane == 0) mbar_arrive(&empty_bar[s_prev]);
        gemm_epilogue_regs<BN, EK>(p, acc, mt * 128 + cw * 64, nt * BN, b0, b1, t128, epi_stage);
    }
}

// expand a quantised matrix (planar 32-blocks or verbatim K-quant super-blocks) to f16 rows [rows][K]; one thread = one 32-value block.
// Each value is the f16 rounding of the exact d * (q - off), i.e. what dequantize_row_* gives after one f16 store (wb_quant.cuh).
template <int WT>
__global__ void __launch_bounds__(256)
k_dequant_f16(const void * base, const uint8_t * qs, const uint32_t * qh, const __half * dd, const __half * mm, int64_t row0, int64_t n_blocks, int K, __half * out) {
    const int64_t bi = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
    if (bi >= n_blocks) return;
    const int64_t nblk = K >> 5;
    uint4 o[4];
    if (WT == WT_Q4_K || WT == WT_Q5_K) {
        constexpr int BLK = (WT == WT_Q4_K) ? 144 : 176;
        const int64_t row = bi / nblk, kb = bi - row * nblk;
        const uint8_t * sb = reinterpret_cast<const uint8_t *>(base) + ((row0 + row) * (K >> 8) + (kb >> 3)) * BLK;
        dequant_kq_sub<WT == WT_Q5_K>(sb, (int) (kb & 7), o);
    } else if (WT == WT_Q3_K) {
        const int64_t row = bi / nblk, kb = bi - row * nblk;
        dequant_q3k_sub(reinterpret_cast<const uint8_t *>(base) + ((row0 + row) * (K >> 8) + (kb >> 3)) * 110, (int) (kb & 7), o);
    } else {
        const int64_t g = row0 * nblk + bi;
        if (WT == WT_Q4_0)      dequant_q4_0(__ldg(reinterpret_cast<const uint4 *>(qs) + g), dd[g], o);
        else if (WT == WT_Q5_0) dequant_q5_0(__ldg(reinterpret_cast<const uint4 *>(qs) + g), __ldg(qh + g), dd[g], o);
        else if (WT == WT_Q4_1) dequant_q4_1(__ldg(reinterpret_cast<const uint4 *>(qs) + g), dd[g], mm[g], o);
        else if (WT == WT_Q5_1) dequant_q5_1(__ldg(reinterpret_cast<const uint4 *>(qs) + g), __ldg(qh + g), dd[g], mm[g], o);
        else                    dequant_q8_0(__ldg(reinterpret_cast<const uint4 *>(qs) + 2*g), __ldg(reinterpret_cast<const uint4 *>(qs) + 2*g + 1), dd[g], o);
    }
    uint4 * dst = reinterpret_cast<uint4 *>(out + bi * 32);
    dst[0] = o[0]; dst[1] = o[1]; dst[2] = o[2]; dst[3] = o[3];
}

// =============================================================================================== host side
typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                    const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static PFN_encodeTiled get_encode_fn() {
    static PFN_encodeTiled fn = nullptr;
    if (!fn) {
        void * p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<PFN_encodeTiled>(p);
    }
    return fn;
}

bool make_tmap_f16(CUtensorMap * out, const void * base, uint64_t k, uint64_t rows, uint64_t z2, uint64_t z3,
                   uint64_t stride_rows, uint64_t stride_z2, uint64_t stride_z3, uint32_t box_rows) {
    PFN_encodeTiled fn = get_encode_fn();
    if (!fn) { set_error("cuTensorMapEncodeTiled entry point not available"); return false; }
    cuuint64_t dims[4]    = { k, rows, z2 ? z2 : 1, z3 ? z3 : 1 };
    cuuint64_t strides[3] = { stride_rows * 2, (stride_z2 ? stride_z2 : stride_rows * rows) * 2,
                              (stride_z3 ? stride_z3 : stride_rows * rows * (z2 ? z2 : 1)) * 2 };
    cuuint32_t box[4]     = { 64, box_rows, 1, 1 };
    cuuint32_t estr[4]    = { 1, 1, 1, 1 };
    if ((reinterpret_cast<uintptr_t>(base) & 15) || (strides[0] & 15) || (strides[1] & 15) || (strides[2] & 15)) {
        set_error("make_tmap_f16: base/strides must be 16-byte aligned (base=%p strides=%llu,%llu,%llu)", base,
                  (unsigned long long) strides[0], (unsigned long long) strides[1], (unsigned long long) strides[2]);
        return false;
    }
    CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void *>(base), dims, strides, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed: %d", (int) r); return false; }
    return true;
}

static int gemm_n_sm() {
    static int n = 0;
    if (!n) { int dev = 0; cudaGetDevice(&dev); cudaDeviceProp pr; if (cudaGetDeviceProperties(&pr, dev) == cudaSuccess) n = pr.multiProcessorCount; else n = 132; }
    return n;
}

// persistent = false: one CTA per tile; true: one CTA per SM walking the tile list
template <int BN, int WT, int EK>
static cudaError_t launch_t(const GemmDesc & g, GemmKParams kp, bool persistent, cudaStream_t st) {
    auto kern = gemm_kernel<BN, WT, EK>;
    {
        const cudaError_t e = ensure_dyn_smem(reinterpret_cast<const void *>(kern), GemmCfg<BN>::SMEM);
        if (e != cudaSuccess) return e;
    }
    kp.n_mt = (g.M + 127) / 128; kp.n_nt = (g.N + BN - 1) / BN; kp.n_tiles = kp.n_mt * kp.n_nt * g.nb0 * g.nb1;
    const int grid = persistent ? std::min(kp.n_tiles, gemm_n_sm()) : kp.n_tiles;
    kern<<<grid, GEMM_THREADS, GemmCfg<BN>::SMEM, st>>>(kp, g.tmA, g.tmB);
    count_launch();
    return cudaGetLastError();
}

template <int WT, int EK>
static cudaError_t launch_bn(const GemmDesc & g, const GemmKParams & kp, bool persistent, cudaStream_t st) {
    switch (g.BN) {
        case 64:  return launch_t<64,  WT, EK>(g, kp, persistent, st);
        case 128: return launch_t<128, WT, EK>(g, kp, persistent, st);
        case 256: return launch_t<256, WT, EK>(g, kp, persistent, st);
    }
    return cudaErrorInvalidValue;
}

// f16 weights: the epilogue kind is a template parameter.  Quantised weights decoded in the kernel (first-generation launch) take the
// general epilogue, which recognises the same kinds per value with the same formulas (one instantiation per weight type and tile width)
template <int WT>
static cudaError_t launch_ek(const GemmDesc & g, const GemmKParams & kp, bool persistent, cudaStream_t st) {
    if constexpr (WT != WT_F16) {
        return launch_bn<WT, EPI_GENERAL>(g, kp, persistent, st);
    } else {
        switch (epi_kind(g.ep)) {
            case EPI_F16:        return launch_bn<WT, EPI_F16>(g, kp, persistent, st);
            case EPI_F16_GELU:   return launch_bn<WT, EPI_F16_GELU>(g, kp, persistent, st);
            case EPI_F32_RES:    return launch_bn<WT, EPI_F32_RES>(g, kp, persistent, st);
            case EPI_F16_MMAJOR: return launch_bn<WT, EPI_F16_MMAJOR>(g, kp, persistent, st);
            case EPI_F16_HM:     return launch_bn<WT, EPI_F16_HM>(g, kp, persistent, st);
            case EPI_GENERAL:    return launch_bn<WT, EPI_GENERAL>(g, kp, persistent, st);
        }
        return cudaErrorInvalidValue;
    }
}

cudaError_t dequant_to_f16(const QMat & W, int64_t rows, __half * out, cudaStream_t st) {
    const int64_t n_blocks = rows * (W.K >> 5);
    const unsigned grid = (unsigned) ((n_blocks + 255) / 256);
    switch (W.type) {
        case WT_Q4_0: k_dequant_f16<WT_Q4_0><<<grid, 256, 0, st>>>(W.base, W.qs, W.qh, W.d, W.m, 0, n_blocks, W.K, out); break;
        case WT_Q4_1: k_dequant_f16<WT_Q4_1><<<grid, 256, 0, st>>>(W.base, W.qs, W.qh, W.d, W.m, 0, n_blocks, W.K, out); break;
        case WT_Q5_0: k_dequant_f16<WT_Q5_0><<<grid, 256, 0, st>>>(W.base, W.qs, W.qh, W.d, W.m, 0, n_blocks, W.K, out); break;
        case WT_Q5_1: k_dequant_f16<WT_Q5_1><<<grid, 256, 0, st>>>(W.base, W.qs, W.qh, W.d, W.m, 0, n_blocks, W.K, out); break;
        case WT_Q8_0: k_dequant_f16<WT_Q8_0><<<grid, 256, 0, st>>>(W.base, W.qs, W.qh, W.d, W.m, 0, n_blocks, W.K, out); break;
        case WT_Q4_K: k_dequant_f16<WT_Q4_K><<<grid, 256, 0, st>>>(W.base, W.qs, W.qh, W.d, W.m, 0, n_blocks, W.K, out); break;
        case WT_Q5_K: k_dequant_f16<WT_Q5_K><<<grid, 256, 0, st>>>(W.base, W.qs, W.qh, W.d, W.m, 0, n_blocks, W.K, out); break;
        case WT_Q3_K: k_dequant_f16<WT_Q3_K><<<grid, 256, 0, st>>>(W.base, W.qs, W.qh, W.d, W.m, 0, n_blocks, W.K, out); break;
        default: return cudaErrorInvalidValue;
    }
    count_launch();
    return cudaGetLastError();
}

// expand the rows of g.A that this launch uses into g.a16 (f16 [rows][K]); rows = M x (stacked matrices)
static cudaError_t dequant_launch(const GemmDesc & g, cudaStream_t st) {
    const int64_t rows = g.a_rows_per_b0 ? (int64_t) g.a_rows_per_b0 * g.nb0 : g.M;
    QMat W = g.A; W.K = g.K;
    return dequant_to_f16(W, rows, g.a16, st);
}

cudaError_t gemm_launch(const GemmDesc & g, cudaStream_t st) {
    const double nb = (double) g.nb0 * g.nb1;
    ProfScope prof(PC_GEMM, st, nb * ((double) g.M * g.K * g.taps * wt_bpw(g.A.type) + (double) g.N * g.K * g.taps * 2 + (double) g.M * g.N * (g.ep.out_f16 ? 2 : 4)),
                   nb * 2.0 * g.M * g.N * g.K * g.taps);
    GemmKParams kp;
    kp.M = g.M; kp.N = g.N; kp.K = g.K; kp.taps = g.taps; kp.nkb_per_tap = (g.K + 63) / 64; kp.nb0 = g.nb0;
    kp.a_zsel0 = g.a_zsel[0]; kp.a_zsel1 = g.a_zsel[1]; kp.b_zsel0 = g.b_zsel[0]; kp.b_zsel1 = g.b_zsel[1];
    kp.a_rows_per_b0 = g.a_rows_per_b0; kp.b1_in_off = g.b1_in_off;
    kp.a_base = g.A.base; kp.a_qs = g.A.qs; kp.a_qh = g.A.qh; kp.a_d = g.A.d; kp.a_m = g.A.m;
    kp.ep = g.ep;
    kp.b_split = g.half_box_b ? 2 : 1;
    if (g.half_box_b && g.BN < 128) return cudaErrorInvalidValue;
    if (g.v2 && (g.A.type == WT_F16 || g.a16)) {                  // persistent kernel: both operands f16 through TMA
        if (g.A.type != WT_F16 && !g.a16_keep) { const cudaError_t e = dequant_launch(g, st); if (e != cudaSuccess) return e; }
        return launch_ek<WT_F16>(g, kp, true, st);
    }
    switch (g.A.type) {
        case WT_F16:  return launch_ek<WT_F16>(g, kp, false, st);
        case WT_Q4_0: return launch_ek<WT_Q4_0>(g, kp, false, st);
        case WT_Q5_0: return launch_ek<WT_Q5_0>(g, kp, false, st);
        case WT_Q4_1: return launch_ek<WT_Q4_1>(g, kp, false, st);
        case WT_Q5_1: return launch_ek<WT_Q5_1>(g, kp, false, st);
        case WT_Q8_0: return launch_ek<WT_Q8_0>(g, kp, false, st);
        case WT_Q4_K: return launch_ek<WT_Q4_K>(g, kp, false, st);
        case WT_Q5_K: return launch_ek<WT_Q5_K>(g, kp, false, st);
        case WT_Q3_K: return launch_ek<WT_Q3_K>(g, kp, false, st);
    }
    return cudaErrorInvalidValue;
}

} // namespace wb
