// wb_decode_mk2.cu -- second generation of the persistent decode kernel (same arithmetic per op as wb_decode_mk.cu, new schedule).
//
// What it computes is whisper_build_graph_decoder (src/whisper.cpp:2466-2844) for the rows of one whisper_batch (<= 64 rows).
//
// Why a second generation: in the first one all CTAs (one per SM) walk the same phase together.  Per layer that is ~160 us of latency-bound
// phases (GEMV of a few MB, LayerNorm, self-attention, 11 grid barriers) that leave HBM idle, followed by ~100 us of cross-attention
// that is purely HBM-bound (503 MB of cross K/V per layer at 64 rows = 90 % of the bytes of the pass).  The two kinds of work never
// overlap, so the pass sits at 0.31 of the HBM roofline although the streaming part alone runs at 0.8.
//
// Schedule of this kernel:
//   * the rows of a pass are cut into ROW GROUPS of 16 (independent sequences in steady-state decoding).  Every group walks the
//     layers on its own: its CTAs synchronise on the group's own barrier, nothing orders one group against another.
//   * grid = 2 CTAs of 8 warps per SM (cooperative launch, 103 KB of shared memory each), dealt out to the groups so that the two
//     CTAs of an SM serve different groups.  While one group streams its cross K/V the others are in their latency-bound
//     phases: HBM stays busy and the SM's issue slots are shared between a streaming CTA and a latency-bound one.
//     Groups start staggered (a.stagger_clk cycles apart) so that they do not meet in the cross-attention phase.
//   * LayerNorm is folded into the CONSUMER's row staging: a GEMV CTA pulls the 16 f32 residual rows of its group with TMA bulk
//     copies, normalises and quantises them in shared memory (one warp per row; bit-identical to the stand-alone phase of the first
//     generation) -- 8 barriers per layer instead of 11, no LayerNorm phase.
//   * a pass that holds several tokens of ONE sequence in different groups (prompt passes) sets a.global_sync: after the QKV phase
//     (KV append) all groups meet in one grid-wide barrier, because a row then attends to cells another group has just written.
// Per-row arithmetic never depends on which other rows share the pass (fixed split-K order, fixed merge orders): a batch of 64 and a
// single row give bit-identical results.
#include <cmath>
#include <type_traits>
#include "wb_decode_mk.cuh"
#include "wb_common.h"
#include "wb_dev.cuh"
#include "wb_ptx.cuh"

namespace wb {
namespace mk2 {

constexpr int T2 = 256, W2 = 8, CPS = 2, RG = 16, NGMAX = 4, MAXTOK = RG * NGMAX;
constexpr int TP = 4;                        // weight tiles a GEMV iteration keeps in flight
constexpr int CHB = 2560;                    // bytes of one staged activation row chunk (2560 int8 values or 1280 halves)
constexpr int XKEYS = 64;                    // keys per cross-attention chunk (8 warps x 8 key slots)
constexpr int PARTW = 68;

extern __shared__ __align__(128) uint8_t sm[];
constexpr int OFF_XQ   = 0;                                   // staged rows, buffer 0: [16][CHB + 16]
constexpr int OFF_XD   = OFF_XQ + RG * (CHB + 16);            // their block scales [16][CHB / 32]
constexpr int OFF_RED  = OFF_XD + RG * (CHB / 32) * 4;        // split-K partials [TP][8 warps][16][17]  |  f32 rows for LayerNorm [8][d]  |  staged rows, buffer 1
constexpr int RED_BYTES = RG * (CHB + 16) + RG * (CHB / 32) * 4;     // buffer 1 = rows + scales (46336) >= 8 * 1280 * 4 (40960) >= TP*8*16*17*4 (34816)
constexpr int RING = 6, RING_SLOT = T2 * 64;                  // cross-attention cp.async ring: 6 x 16 KB (aliases everything above)
constexpr int OFF_QSM  = RING * RING_SLOT;                    // f16-rounded query of the pair [2][64] f32
constexpr int OFF_PART = OFF_QSM + 2 * 64 * 4;                // attention warp partials [2][8][68]
constexpr int OFF_FLAG = OFF_PART + 2 * W2 * PARTW * 4;       // [16] ints, then 3 mbarriers
constexpr int OFF_MBAR = OFF_FLAG + 64;
constexpr int OFF_CTX  = OFF_MBAR + 32;                      // schedule state of the CTA (struct Ctx)
constexpr int SMEM     = OFF_CTX + 96;
static_assert(OFF_RED + RED_BYTES <= OFF_QSM, "GEMV staging must fit below the attention scratch");
static_assert(TP * W2 * 16 * 17 * 4 <= RED_BYTES && 9 * 1280 * 4 <= RED_BYTES, "reduction / LayerNorm staging area (8 rows + the LayerNorm weight)");
static_assert(RG * (1280 + 16) + 1280 * 4 <= RG * (CHB + 16), "LayerNorm bias behind the quantised rows of buffer 0");
static_assert(SMEM <= 112 * 1024, "two CTAs per SM");

#define S_XQ(b)  (reinterpret_cast<uint32_t *>(sm + ((b) ? OFF_RED : OFF_XQ)))
#define S_XD(b)  (reinterpret_cast<float *>(sm + ((b) ? OFF_RED + RG * (CHB + 16) : OFF_XD)))
#define S_RED    (reinterpret_cast<float *>(sm + OFF_RED))
#define S_F32    (reinterpret_cast<float *>(sm + OFF_RED))
#define S_PART   (reinterpret_cast<float *>(sm + OFF_PART))
#define S_FLAG   (reinterpret_cast<int *>(sm + OFF_FLAG))
#define S_MBAR   (reinterpret_cast<uint64_t *>(sm + OFF_MBAR))

// per-CTA schedule state, in shared memory (kept in a local struct it lived in local memory, and with 206 KB of the SM's 256 KB
// configured as shared memory there is almost no L1 behind local memory: every access was an L2 round trip)
struct Ctx {
    int g, ci, cg;                       // row group of this CTA, its index among / the number of the group's CTAs
    int t_base, nt;                      // rows of the group
    int NG, n_sm;
    int r_s[CPS], cnt_s[CPS];            // members of the group: CTA s * n_sm + r_s[s] + NG * m, m < cnt_s[s]
    unsigned kbar, kglob;                // barriers passed (group / all groups); written by thread 0 between two CTA barriers
    uint32_t par[3];                     // phase parities of the three mbarriers; written by thread 0 at the end of a phase
};
static_assert(sizeof(Ctx) <= 96, "Ctx area");
#define CX (*reinterpret_cast<Ctx *>(sm + OFF_CTX))

#define MK_STAMP() do { if (TRACE) { if (blockIdx.x == 0 && threadIdx.x == 0) a.trace[n_stamp] = clock64(); ++n_stamp; } } while (0)
#define MK_FINE(j) do { if (fb >= 0 && blockIdx.x == 0 && threadIdx.x == 0) a.trace[fb + (j)] = clock64(); } while (0)

__device__ __forceinline__ void l2_prefetch(const void * p, uint32_t bytes) {
    if (bytes >= 16) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" :: "l"(p), "r"(bytes & ~15u) : "memory");
}
__device__ __forceinline__ void bulk_g2s(void * dst, const void * src, uint32_t bytes, uint64_t * bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void cp_async16(uint32_t saddr, const void * g) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(saddr), "l"(g) : "memory"); }
__device__ __forceinline__ void cp_async16_hint(uint32_t saddr, const void * g, uint64_t pol) { asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" :: "r"(saddr), "l"(g), "l"(pol) : "memory"); }
__device__ __forceinline__ uint64_t policy_evict_first() { uint64_t p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ uint4 ldcg_hint(const uint4 * p, uint64_t pol) {
    uint4 v; asm volatile("ld.global.cg.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p), "l"(pol)); return v;
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }

__device__ __forceinline__ int member_cta(int i) {
    int s = 0;
    while (s + 1 < CPS && i >= CX.cnt_s[s]) { i -= CX.cnt_s[s]; ++s; }
    return s * CX.n_sm + CX.r_s[s] + CX.NG * i;
}

__device__ __forceinline__ void wait_flag(const MkArgs & a, const unsigned long long * f, unsigned long long want) {
    const long long t0 = clock64();
    unsigned long long v;
    for (;;) {
        asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(f) : "memory");
        if (v >= want) break;
        if (clock64() - t0 > (6LL << 30)) { *a.err = 1; __threadfence_system(); __trap(); }    // ~3 s: a CTA never arrived
    }
}

// Barrier of one row group.  a.bar: [16*g] arrival counter of group g (zeroed by the host before the launch), [16*4] counter of the
// all-groups barrier, [128 + 16*cta] release flags of each CTA ([0] group barriers, [1] all-groups barriers; monotonic across launches:
// a.bar_base grows by 4096 per launch).  The LAST CTA to arrive releases the others through their own flags.
__device__ __noinline__ void grp_sync(const MkArgs & a) {
    __syncthreads();
    const unsigned kb = CX.kbar + 1;
    const int cg = CX.cg;
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned long long old = atomicAdd(a.bar + 16 * CX.g, 1ULL);
        const int last = (old + 1 == (unsigned long long) kb * (unsigned long long) cg);
        S_FLAG[2] = last;
        if (last) __threadfence();
    }
    __syncthreads();
    const unsigned long long want = a.bar_base + kb;
    if (S_FLAG[2]) {
        for (int i = threadIdx.x; i < cg; i += T2)
            asm volatile("st.release.gpu.global.u64 [%0], %1;" :: "l"(a.bar + 128 + 16 * member_cta(i)), "l"(want) : "memory");
        if (threadIdx.x == 0) CX.kbar = kb;
    } else if (threadIdx.x == 0) { CX.kbar = kb; wait_flag(a, a.bar + 128 + 16 * blockIdx.x, want); }
    __syncthreads();
}
__device__ __noinline__ void all_sync(const MkArgs & a) {
    __syncthreads();
    const unsigned kg = CX.kglob + 1;
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned long long old = atomicAdd(a.bar + 16 * NGMAX, 1ULL);
        const int last = (old + 1 == (unsigned long long) kg * (unsigned long long) gridDim.x);
        S_FLAG[2] = last;
        if (last) __threadfence();
    }
    __syncthreads();
    const unsigned long long want = a.bar_base + kg;
    if (S_FLAG[2]) {
        for (int i = threadIdx.x; i < (int) gridDim.x; i += T2)
            asm volatile("st.release.gpu.global.u64 [%0], %1;" :: "l"(a.bar + 128 + 16 * i + 1), "l"(want) : "memory");
        if (threadIdx.x == 0) CX.kglob = kg;
    } else if (threadIdx.x == 0) { CX.kglob = kg; wait_flag(a, a.bar + 128 + 16 * blockIdx.x + 1, want); }
    __syncthreads();
}
// Cross-attention turn: the row groups stream their cross K / V ONE AFTER THE OTHER (ticket = layer * NG + group; a.bar[16*5] counts
// finished turns).  Left alone the groups fall into lock-step (a group that runs ahead pays the HBM latency of every weight tile the
// others then find in L2) and meet in this phase, where they share the HBM bandwidth and all wait; taking turns, a group streams at the
// full rate while the others are in their latency-bound phases, and the order of the turns keeps the groups apart.
__device__ __forceinline__ void cross_turn_wait(const MkArgs & a, int l) {
    if (threadIdx.x == 0) wait_flag(a, a.bar + 16 * (NGMAX + 1), (unsigned long long) (l * CX.NG + CX.g));
    __syncthreads();
}
__device__ __forceinline__ void cross_turn_done(const MkArgs & a) {
    if (CX.ci == 0 && threadIdx.x == 0) { __threadfence(); atomicAdd(a.bar + 16 * (NGMAX + 1), 1ULL); }
}

// one warp quantises the 32 values its lanes hold (one Q8_0 block of row t starting at element e0) -- as in wb_decode_mk.cu
template <int WT>
__device__ __forceinline__ void store_q(uint8_t * dst, int K, int t, int e0, int lane, float v) {
    if (WT == WT_F16) { reinterpret_cast<__half *>(dst)[(size_t) t * K + e0 + lane] = __float2half_rn(v); return; }
    const float amax = warp_max(fabsf(v));
    const float id = (amax != 0.0f) ? __fdividef(127.0f, amax) : 0.0f;
    reinterpret_cast<int8_t *>(dst)[(size_t) t * K + e0 + lane] = (int8_t) __float2int_rn(v * id);
    if (lane == 0) reinterpret_cast<float *>(dst + (size_t) MAXTOK * K)[t * (K >> 5) + (e0 >> 5)] = __half2float(__float2half_rn(amax * (1.0f / 127.0f)));
}

struct Epi {
    const float * bias = nullptr, * scale = nullptr; int act = 0; const float * res = nullptr; float * out = nullptr;
    __half * kc = nullptr, * vc = nullptr; int kv_d = 0;
    uint8_t * qout = nullptr;            // PAIR epilogue: quantised rows [64][N] (+ block scales) for the next GEMV
};

// L2 prefetch of the weight tiles of a later GEMV phase (tile-major: the records of a tile are contiguous); every tile once per group
__device__ __noinline__ void prefetch_w(const QMat & W) {
    if (threadIdx.x != T2 - 32) return;
    const int n_tiles = (W.N + 15) >> 4;
    const uint32_t tile_bytes = (uint32_t) (W.K / wt_tm_rec_k(W.type)) * wt_tm_rec_bytes(W.type);
    for (int tile = CX.ci, cg = CX.cg; tile < n_tiles; tile += cg)
        l2_prefetch(reinterpret_cast<const uint8_t *>(W.base) + (size_t) tile * tile_bytes, tile_bytes);
}

// LayerNorm (ggml-cpu/ops.cpp:3698-3765, two passes, then mul/add whisper.cpp:2536-2543) of one f32 row held in shared memory by one
// warp; the result goes, quantised, into staging buffer 0.  Sums are formed exactly as in the distributed phase of the first generation
// (per 128-value slice a warp sum, the slices combined by a 16-lane butterfly): same bits.
__device__ __forceinline__ void ln_load(float4 (&v)[10], const float * srow, int K) {
    const int lane = threadIdx.x & 31, nc = K >> 7;
#pragma unroll
    for (int cch = 0; cch < 10; ++cch) v[cch] = (cch < nc) ? *reinterpret_cast<const float4 *>(srow + cch * 128 + lane * 4) : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
}
// s_w / s_b: the LayerNorm weight and bias in shared memory.  All shuffles are unconditional (slices beyond K hold zeros): no divergence
// checks around them, and the compiler is free to keep the row in registers.
template <int WT>
__device__ __forceinline__ void ln_row(float4 (&v)[10], int K, const float * s_w, const float * s_b, float eps, int r, int SW, int nb) {
    const int lane = threadIdx.x & 31;
    const int nc = K >> 7;                                       // 128-value slices (<= 10)
    // two passes (mean, then squared deviations); every lane adds up its 4 values of each slice in slice order, one butterfly per pass
    float tot = 0.0f;
#pragma unroll
    for (int cch = 0; cch < 10; ++cch) tot += (v[cch].x + v[cch].y) + (v[cch].z + v[cch].w);
    const float mean = warp_sum(tot) / K;
    float qt = 0.0f;
#pragma unroll
    for (int cch = 0; cch < 10; ++cch) {
        if (cch < nc) { v[cch].x -= mean; v[cch].y -= mean; v[cch].z -= mean; v[cch].w -= mean; }
        qt += (v[cch].x * v[cch].x + v[cch].y * v[cch].y) + (v[cch].z * v[cch].z + v[cch].w * v[cch].w);
    }
    const float rstd = 1.0f / sqrtf(warp_sum(qt) / K + eps);
#pragma unroll
    for (int cch = 0; cch < 10; ++cch) {
        const int e0 = cch * 128 + lane * 4;
        const bool on = cch < nc;
        const float4 w = on ? *reinterpret_cast<const float4 *>(s_w + e0) : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        const float4 b = on ? *reinterpret_cast<const float4 *>(s_b + e0) : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        float4 y;
        y.x = __fadd_rn(__fmul_rn(__fmul_rn(v[cch].x, rstd), w.x), b.x);
        y.y = __fadd_rn(__fmul_rn(__fmul_rn(v[cch].y, rstd), w.y), b.y);
        y.z = __fadd_rn(__fmul_rn(__fmul_rn(v[cch].z, rstd), w.z), b.z);
        y.w = __fadd_rn(__fmul_rn(__fmul_rn(v[cch].w, rstd), w.w), b.w);
        if (WT == WT_F16) {
            const __half2 h0 = __floats2half2_rn(y.x, y.y), h1 = __floats2half2_rn(y.z, y.w);
            if (on) *reinterpret_cast<uint2 *>(S_XQ(0) + r * SW + (e0 >> 1)) = make_uint2(*reinterpret_cast<const uint32_t *>(&h0), *reinterpret_cast<const uint32_t *>(&h1));
        } else {
            float amax = fmaxf(fmaxf(fabsf(y.x), fabsf(y.y)), fmaxf(fabsf(y.z), fabsf(y.w)));
            amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
            amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
            amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 4));
            const float id = (amax != 0.0f) ? __fdividef(127.0f, amax) : 0.0f;
            const uint32_t q0 = (uint32_t) __float2int_rn(y.x * id) & 0xffu, q1 = (uint32_t) __float2int_rn(y.y * id) & 0xffu;
            const uint32_t q2 = (uint32_t) __float2int_rn(y.z * id) & 0xffu, q3 = (uint32_t) __float2int_rn(y.w * id) & 0xffu;
            if (on) {
                S_XQ(0)[r * SW + (e0 >> 2)] = q0 | (q1 << 8) | (q2 << 16) | (q3 << 24);
                if ((lane & 7) == 0) S_XD(0)[r * nb + (e0 >> 5)] = __half2float(__float2half_rn(amax * (1.0f / 127.0f)));
            }
        }
    }
}

// k-loop over the records of one staged chunk for NV valid tile slots (compile-time: predicated slots made ptxas spill);
// accumulates into acc.  xb: staging buffer of the chunk, rec0: first record of the chunk inside a tile, nrc: records in the chunk.
template <int WT, int NV, int TU>
__device__ __forceinline__ void kloop_chunk(float (&acc)[NV][2][4], const uint8_t * wbase, int tile0, int tstep, int nrec, int rec0, int nrc, int xb, int nbc, int SW, int nt, int NH,
                                            uint64_t * mbar, uint32_t parity, bool & staged) {
    constexpr int REC = (WT == WT_Q4_0) ? 288 : (WT == WT_Q5_0 ? 352 : (WT == WT_Q8_0 ? 544 : 512));
    constexpr int QSB = (WT == WT_Q8_0) ? 512 : 256;
    constexpr int UB = 3;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, c = lane & 3;
    const uint32_t * xq = S_XQ(xb);
    const float * xd = S_XD(xb);
    for (int kb = warp; kb < nrc; kb += W2 * UB) {
        uint4 wq[NV][UB]; uint2 wh[NV][UB]; uint32_t wd[NV][UB];
#pragma unroll
        for (int j = 0; j < NV; ++j) {
            const uint8_t * tb = wbase + ((size_t) ((tile0 + (j / TU) * tstep) * TU + j % TU) * nrec + rec0) * REC;
#pragma unroll
            for (int u = 0; u < UB; ++u) {
                const uint8_t * rec = tb + (size_t) min(kb + u * W2, nrc - 1) * REC;
                if (WT == WT_F16 || WT == WT_Q8_0) wq[j][u] = __ldg(reinterpret_cast<const uint4 *>(rec) + lane);
                else { const uint2 q2 = __ldg(reinterpret_cast<const uint2 *>(rec) + lane); wq[j][u].x = q2.x; wq[j][u].y = q2.y; }
                if (WT == WT_Q5_0) wh[j][u] = __ldg(reinterpret_cast<const uint2 *>(rec + QSB) + g);
                if (WT != WT_F16)  wd[j][u] = __ldg(reinterpret_cast<const uint32_t *>(rec + QSB + (WT == WT_Q5_0 ? 64 : 0)) + g);
            }
        }
        if (!staged) { if (mbar) mbar_wait(mbar, parity); staged = true; }       // the rows have landed (this warp's weights are in flight)
#pragma unroll
        for (int u = 0; u < UB; ++u) {
            const int b = kb + u * W2;
            if (b < nrc) {
                uint32_t bf[2][2]; float dx[2][2];
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const bool ok = h * 8 + g < nt;
                    bf[h][0] = ok ? xq[(h * 8 + g) * SW + b * 8 + c] : 0u;
                    bf[h][1] = ok ? xq[(h * 8 + g) * SW + b * 8 + 4 + c] : 0u;
                    dx[h][0] = dx[h][1] = 0.0f;
                    if (WT != WT_F16) { dx[h][0] = xd[min(h * 8 + 2 * c, nt - 1) * nbc + b]; dx[h][1] = xd[min(h * 8 + 2 * c + 1, nt - 1) * nbc + b]; }
                }
#pragma unroll
                for (int j = 0; j < NV; ++j) {
                    uint32_t af[4];
                    float dw0 = 0.0f, dw1 = 0.0f;
                    if (WT == WT_F16 || WT == WT_Q8_0) { af[0] = wq[j][u].x; af[1] = wq[j][u].y; af[2] = wq[j][u].z; af[3] = wq[j][u].w; }
                    else {
                        uint32_t lo0 = wq[j][u].x & 0x0F0F0F0Fu, hi0 = (wq[j][u].x >> 4) & 0x0F0F0F0Fu, lo1 = wq[j][u].y & 0x0F0F0F0Fu, hi1 = (wq[j][u].y >> 4) & 0x0F0F0F0Fu;
                        if (WT == WT_Q5_0) {
                            lo0 |= spread4_to_bit4(wh[j][u].x >> (4 * c)); hi0 |= spread4_to_bit4(wh[j][u].x >> (16 + 4 * c));
                            lo1 |= spread4_to_bit4(wh[j][u].y >> (4 * c)); hi1 |= spread4_to_bit4(wh[j][u].y >> (16 + 4 * c));
                            af[0] = __vsub4(lo0, 0x10101010u); af[2] = __vsub4(hi0, 0x10101010u);
                            af[1] = __vsub4(lo1, 0x10101010u); af[3] = __vsub4(hi1, 0x10101010u);
                        } else {
                            af[0] = __vsub4(lo0, 0x08080808u); af[2] = __vsub4(hi0, 0x08080808u);
                            af[1] = __vsub4(lo1, 0x08080808u); af[3] = __vsub4(hi1, 0x08080808u);
                        }
                    }
                    if (WT != WT_F16) {
                        dw0 = __half2float(__ushort_as_half((unsigned short) (wd[j][u] & 0xffffu)));
                        dw1 = __half2float(__ushort_as_half((unsigned short) (wd[j][u] >> 16)));
                    }
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        if (h < NH) {
                            if (WT == WT_F16) mma_f16_16816(acc[j][h], af, bf[h][0], bf[h][1]);
                            else {
                                int dd[4]; mma_s8_16832(dd, af, bf[h][0], bf[h][1]);
                                acc[j][h][0] = fmaf(dw0 * dx[h][0], (float) dd[0], acc[j][h][0]);
                                acc[j][h][1] = fmaf(dw0 * dx[h][1], (float) dd[1], acc[j][h][1]);
                                acc[j][h][2] = fmaf(dw1 * dx[h][0], (float) dd[2], acc[j][h][2]);
                                acc[j][h][3] = fmaf(dw1 * dx[h][1], (float) dd[3], acc[j][h][3]);
                            }
                        }
                    }
                }
            }
        }
    }
    if (!staged) { if (mbar) mbar_wait(mbar, parity); staged = true; }
}

// LayerNorm staging of a GEMV phase: the f32 residual rows of the group -> shared memory in two batches of 8 rows (TMA), one warp per
// row: LayerNorm + Q8_0 into staging buffer 0.  The second batch is requested as soon as the first sits in registers.
template <int WT>
__device__ __noinline__ void ln_stage(const MkArgs & a, const float * xf, int K, const float * ln_w, const float * ln_b, int SW, int nb) {
    const int tid = threadIdx.x, warp = tid >> 5, nt = CX.nt, t_base = CX.t_base;
    const float eps = a.eps;
    const uint32_t rb = (uint32_t) K * 4;
    const int nb1 = min(nt, 8), nb2 = nt - nb1;
    // LayerNorm weight behind the 8 rows of a batch, bias in the part of buffer 0 the quantised rows leave free (F16: the unused scale area):
    // read by every row from shared memory (a global load per 128-value slice was an L2 round trip each: 20 us per phase)
    float * s_w = S_F32 + 8 * K;
    float * s_b = (WT == WT_F16) ? reinterpret_cast<float *>(sm + OFF_XD) : reinterpret_cast<float *>(sm + OFF_XQ + RG * (K + 16));
    uint32_t par = CX.par[2];
    float4 v[10];
    if (tid == 0) { fence_proxy_async_smem(); mbar_arrive_expect_tx(S_MBAR + 2, (uint32_t) nb1 * rb + 2u * rb); }
    __syncwarp();
    if (tid < nb1) { asm volatile("fence.proxy.async;" ::: "memory"); bulk_g2s(S_F32 + tid * K, xf + (size_t) (t_base + tid) * K, rb, S_MBAR + 2); }
    else if (tid == nb1) bulk_g2s(s_w, ln_w, rb, S_MBAR + 2);
    else if (tid == nb1 + 1) bulk_g2s(s_b, ln_b, rb, S_MBAR + 2);
    mbar_wait(S_MBAR + 2, par); par ^= 1u;
    if (warp < nb1) ln_load(v, S_F32 + warp * K, K);
    if (nb2 > 0) {
        __syncthreads();                                     // batch 1 sits in registers
        if (tid == 0) { fence_proxy_async_smem(); mbar_arrive_expect_tx(S_MBAR + 2, (uint32_t) nb2 * rb); }
        __syncwarp();
        if (tid < nb2) { asm volatile("fence.proxy.async;" ::: "memory"); bulk_g2s(S_F32 + tid * K, xf + (size_t) (t_base + 8 + tid) * K, rb, S_MBAR + 2); }
    }
    if (warp < nb1) ln_row<WT>(v, K, s_w, s_b, eps, warp, SW, nb);
    if (nb2 > 0) {
        mbar_wait(S_MBAR + 2, par); par ^= 1u;
        if (warp < nb2) { ln_load(v, S_F32 + warp * K, K); ln_row<WT>(v, K, s_w, s_b, eps, 8 + warp, SW, nb); }
    }
    if (tid == 0) CX.par[2] = par;
    __syncthreads();                                         // buffer 0 complete; the f32 area is free for the reduction
}

// geometry of the staged chunks of one GEMV phase
struct Stage {
    const uint8_t * x; int K, rowb, n_ch, che, SW, nb;     // che: elements per full chunk; SW: row stride (words) of a staging buffer; nb: Q8_0 blocks of a whole row
};

// stage chunk ch of the group's rows into buffer xb (TMA bulk copies, completion on mbarrier xb); caller has made sure the buffer is free
template <int WT>
__device__ __forceinline__ void stage_chunk(const Stage & s, int ch, int xb) {
    const int c_nt = CX.nt, c_t_base = CX.t_base;
    const int tid = threadIdx.x;
    const int e0 = ch * s.che, ce = min(s.che, s.K - e0);                // elements of this chunk
    const uint32_t cb = (uint32_t) (WT == WT_F16 ? ce * 2 : ce), nbc = (uint32_t) ce >> 5;
    if (tid == 0) {
        fence_proxy_async_smem();
        mbar_arrive_expect_tx(S_MBAR + xb, (uint32_t) c_nt * (cb + (WT == WT_F16 ? 0u : nbc * 4u)));
    }
    __syncwarp();
    if (tid < c_nt) {
        asm volatile("fence.proxy.async;" ::: "memory");             // rows were written with ordinary stores (by other CTAs, before the barrier)
        bulk_g2s(S_XQ(xb) + tid * s.SW, s.x + (size_t) (c_t_base + tid) * s.rowb + (WT == WT_F16 ? (size_t) e0 * 2 : (size_t) e0), cb, S_MBAR + xb);
        if (WT != WT_F16)
            bulk_g2s(S_XD(xb) + tid * (s.che >> 5), reinterpret_cast<const float *>(s.x + (size_t) MAXTOK * s.K) + (size_t) (c_t_base + tid) * s.nb + (e0 >> 5), nbc * 4u, S_MBAR + xb);
    }
}

// y[t][n] = act((W[n,:] . x[t,:] + bias[n]) * scale[n]) + res[t][n] for the 16 rows of this CTA's group.
// The CTAs of a group deal the 16-row weight tiles out among themselves (up to TP tiles per iteration, loads issued together); the 8
// warps split K of a tile, every weight block is decoded once and multiplied with both 8-row halves (mma.sync.m16n8k32.s8 = the int8
// block dot of vec_dot_q*_q8_0 with f32 scale products); partials are reduced through shared memory in fixed order.
// x: quantised rows in global memory (actq format) staged chunk-wise (2560 bytes of a row per chunk; chunk 0 -> buffer 0, chunk 1 ->
// buffer 1 = the reduction area, both requested at the start), or -- LN -- the f32 residual rows, normalised and quantised here.
// PAIR (FC1): tiles are dealt out in pairs = 32 consecutive output features and the epilogue writes GELU(y) straight into the
// quantised-row format FC2 consumes.
template <int WT, bool PAIR, bool LN>
__device__ __noinline__ void gemv(const MkArgs & a, const QMat & W, const uint8_t * x, const float * xf, const float * ln_w, const float * ln_b, const Epi & e, int fb = -1) {
    constexpr int RK = (WT == WT_F16) ? 16 : 32;                 // K values per record
    constexpr int TU = PAIR ? 2 : 1;                             // tiles per unit of distribution
    constexpr int RLD = 17;
    const int N = W.N, K = W.K;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, cc = lane & 3;
    const int n_tiles = (N + 15) >> 4, nrec = K / RK;
    Stage s;
    s.x = x; s.K = K; s.rowb = (WT == WT_F16) ? K * 2 : K; s.nb = K >> 5;
    s.che = min(K, (WT == WT_F16) ? CHB / 2 : CHB);
    s.n_ch = (K + s.che - 1) / s.che;
    s.SW = ((WT == WT_F16 ? s.che * 2 : s.che) >> 2) + 4;
    const int c_ci = CX.ci, c_cg = CX.cg, c_t_base = CX.t_base;
    const int nt = CX.nt, NH = (nt + 7) >> 3;
    const int n_units = n_tiles / TU;                            // PAIR: N is a multiple of 32
    const int upc = c_ci < n_units ? (n_units - c_ci + c_cg - 1) / c_cg : 0;   // units of this CTA: ci, ci + cg, ...
    const int n_it = (upc * TU + TP - 1) / TP, upi = n_it ? (upc + n_it - 1) / n_it : 0;
    MK_FINE(0);
    __syncthreads();                                             // the previous users of the staging areas are done
    // state of the two staging buffers (uniform over the CTA): chunk held (requested), whether its arrival has been waited for, parity to wait on
    int have0 = -1, have1 = -1; bool done0 = false, done1 = false; uint32_t ppar0 = 0u, ppar1 = 0u;
    uint32_t par0 = CX.par[0], par1 = CX.par[1];                 // read after the barrier above; written back by thread 0 at the end
    auto request = [&](int ch, int xb) {
        stage_chunk<WT>(s, ch, xb);
        if (xb == 0) { have0 = ch; done0 = false; ppar0 = par0; par0 ^= 1u; }
        else         { have1 = ch; done1 = false; ppar1 = par1; par1 ^= 1u; }
    };
    if (LN) {
        ln_stage<WT>(a, xf, K, ln_w, ln_b, s.SW, s.nb);
        have0 = 0; done0 = true;
    } else {
        request(0, 0);
        if (s.n_ch > 1) request(1, 1);
    }
    MK_FINE(1);
    for (int it = 0; it < n_it; ++it) {
        const int u0 = it * upi, nv = TU * (min(upc, u0 + upi) - u0);           // valid tile slots of this iteration (CTA-uniform)
        const uint8_t * wbase = reinterpret_cast<const uint8_t *>(W.base);
        const int unit0 = c_ci + u0 * c_cg;                      // slot j holds tile (unit0 + (j / TU) * cg) * TU + j % TU
        auto run = [&](auto nvc) {
            constexpr int NV = decltype(nvc)::value;
            float acc[NV][2][4];
#pragma unroll
            for (int j = 0; j < NV; ++j)
#pragma unroll
                for (int h = 0; h < 2; ++h) { acc[j][h][0] = acc[j][h][1] = acc[j][h][2] = acc[j][h][3] = 0.0f; }
            for (int ch = 0; ch < s.n_ch; ++ch) {
                const int xb = ch & 1;
                const int e0 = ch * s.che, ce = min(s.che, K - e0);
                if ((xb ? have1 : have0) != ch) { __syncthreads(); request(ch, xb); }       // the buffer holds another chunk (or the reduction has overwritten it)
                bool stg = xb ? done1 : done0;
                kloop_chunk<WT, NV, TU>(acc, wbase, unit0, c_cg, nrec, e0 / RK, ce / RK, xb, s.che >> 5, s.SW, nt, NH, S_MBAR + xb, xb ? ppar1 : ppar0, stg);
                if (xb) done1 = true; else done0 = true;
            }
            if (s.n_ch > 1) __syncthreads();                     // buffer 1 (= the reduction area) may still be read by slower warps
            // split-K partials -> smem: red[tile slot j][warp][row][batch row]
#pragma unroll
            for (int j = 0; j < NV; ++j)
#pragma unroll
                for (int h = 0; h < 2; ++h)
#pragma unroll
                    for (int i = 0; i < 4; ++i) S_RED[((j * W2 + warp) * 16 + g + (i >> 1) * 8) * RLD + h * 8 + 2 * cc + (i & 1)] = acc[j][h][i];
        };
        switch (nv) {
            case 1: if (!PAIR) { run(std::integral_constant<int, 1>()); break; }
            case 2: run(std::integral_constant<int, 2>()); break;
            case 3: if (!PAIR) { run(std::integral_constant<int, 3>()); break; }
            default: run(std::integral_constant<int, 4>()); break;
        }
        have1 = -1;                                              // the reduction has overwritten buffer 1
        if (it == 0) MK_FINE(2);
        float pb[4], ps[4], pr[4];
        // epilogue operands of this thread's (at most four) outputs, fetched before the partials are read back
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int jj, tl, rl;
            if (PAIR) { const int idx = warp + W2 * i; jj = (idx >> 4) * 2 + (lane >> 4); tl = idx & 15; rl = lane & 15; }
            else      { jj = i; tl = tid >> 4; rl = tid & 15; }
            const int row = ((c_ci + (u0 + jj / TU) * c_cg) * TU + jj % TU) * 16 + rl;
            const bool ok = jj < nv && tl < nt && row < N;
            pb[i] = (ok && e.bias) ? __ldg(e.bias + row) : 0.0f;
            ps[i] = (ok && e.scale) ? __ldg(e.scale + row) : 1.0f;
            pr[i] = (ok && e.res) ? __ldcg(e.res + (size_t) (c_t_base + tl) * N + row) : 0.0f;
        }
        __syncthreads();
        if (it == 0) MK_FINE(3);
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            int jj, tl, rl;
            if (PAIR) { const int idx = warp + W2 * i; jj = (idx >> 4) * 2 + (lane >> 4); tl = idx & 15; rl = lane & 15; }
            else      { jj = i; tl = tid >> 4; rl = tid & 15; }
            const int row = ((c_ci + (u0 + jj / TU) * c_cg) * TU + jj % TU) * 16 + rl, t = c_t_base + tl;
            const bool ok = jj < nv && tl < nt && row < N;
            float v = 0.0f;
            if (ok) {
#pragma unroll
                for (int w = 0; w < W2; ++w) v += S_RED[((jj * W2 + w) * 16 + rl) * RLD + tl];
                v = (v + pb[i]) * ps[i];
                if (e.act == 1) v = gelu_ref_f16(v);
                v += pr[i];
            }
            if (PAIR) {
                // (row slot pair, token) is warp-uniform: the 32 lanes hold one Q8_0 block of the FC2 input row t (features row0 .. row0+31)
                const int idx = warp + W2 * i;
                if ((idx >> 4) * 2 < nv && tl < nt) store_q<WT>(e.qout, N, t, row - lane, lane, v);
            } else if (ok) {
                if (e.out) e.out[(size_t) t * N + row] = v;
                if (e.kc && row >= e.kv_d) {
                    const size_t cell = a.cell[t];
                    if (row < 2 * e.kv_d) e.kc[cell * e.kv_d + (row - e.kv_d)] = __float2half_rn(v);
                    else                  e.vc[cell * e.kv_d + (row - 2 * e.kv_d)] = __float2half_rn(v);
                }
            }
        }
        __syncthreads();                                         // S_RED is rewritten by the next iteration
        if (it == 0) MK_FINE(4);
    }
    // copies that were requested but never waited for (a CTA without tiles) must land before the areas are reused
    if (have0 >= 0 && !done0) mbar_wait(S_MBAR + 0, ppar0);
    if (have1 >= 0 && !done1) mbar_wait(S_MBAR + 1, ppar1);
    if (tid == 0) { CX.par[0] = par0; CX.par[1] = par1; }
    MK_FINE(5);
}

// ---- attention (arithmetic as in wb_decode_mk.cu) -------------------------------------------------------------------------------
__device__ __forceinline__ void load_q16(const float * qh, int r, float (&qv)[16]) {
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float4 v = __ldcg(reinterpret_cast<const float4 *>(qh + 8 * r + (i >> 1) * 32) + (i & 1));
        qv[4 * i]     = __half2float(__float2half_rn(v.x)); qv[4 * i + 1] = __half2float(__float2half_rn(v.y));
        qv[4 * i + 2] = __half2float(__float2half_rn(v.z)); qv[4 * i + 3] = __half2float(__float2half_rn(v.w));
    }
}
struct KV4 { uint4 k0, k1, v0, v1; };
__device__ __forceinline__ float dot16(const uint4 & k0, const uint4 & k1, const float (&q)[16]) {
    float s = 0.0f;
    const __half2 * h0 = reinterpret_cast<const __half2 *>(&k0), * h1 = reinterpret_cast<const __half2 *>(&k1);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 f = __half22float2(h0[i]), f2 = __half22float2(h1[i]);
        s = fmaf(f.x, q[2 * i], s); s = fmaf(f.y, q[2 * i + 1], s); s = fmaf(f2.x, q[8 + 2 * i], s); s = fmaf(f2.y, q[8 + 2 * i + 1], s);
    }
    return s;
}
__device__ __forceinline__ float dot16s(const uint4 & k0, const uint4 & k1, const float * q) {   // q: 16 floats in shared memory
    float s = 0.0f;
    const __half2 * h0 = reinterpret_cast<const __half2 *>(&k0), * h1 = reinterpret_cast<const __half2 *>(&k1);
#pragma unroll
    for (int i = 0; i < 4; i += 2) {
        const float4 qa = *reinterpret_cast<const float4 *>(q + 2 * i), qb = *reinterpret_cast<const float4 *>(q + 8 + 2 * i);
        const float2 f0 = __half22float2(h0[i]), f1 = __half22float2(h0[i + 1]), g0 = __half22float2(h1[i]), g1 = __half22float2(h1[i + 1]);
        s = fmaf(f0.x, qa.x, s); s = fmaf(f0.y, qa.y, s); s = fmaf(f1.x, qa.z, s); s = fmaf(f1.y, qa.w, s);
        s = fmaf(g0.x, qb.x, s); s = fmaf(g0.y, qb.y, s); s = fmaf(g1.x, qb.z, s); s = fmaf(g1.y, qb.w, s);
    }
    return s;
}
struct LaneAcc { float m, l, o[16]; };
__device__ __forceinline__ void lane_init(LaneAcc & A) { A.m = -INFINITY; A.l = 0.0f;
#pragma unroll
    for (int i = 0; i < 16; ++i) A.o[i] = 0.0f; }
__device__ __forceinline__ void lane_update(LaneAcc & A, float sc, const uint4 & v0, const uint4 & v1) {
    const float mn = fmaxf(A.m, sc);
    const float resc = __expf(A.m - mn), p = __expf(sc - mn);
    A.l = fmaf(A.l, resc, p); A.m = mn;
    const __half2 * h0 = reinterpret_cast<const __half2 *>(&v0), * h1 = reinterpret_cast<const __half2 *>(&v1);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const float2 f = __half22float2(h0[i]), f2 = __half22float2(h1[i]);
        A.o[2 * i]     = fmaf(A.o[2 * i],     resc, p * f.x);  A.o[2 * i + 1] = fmaf(A.o[2 * i + 1], resc, p * f.y);
        A.o[8 + 2 * i] = fmaf(A.o[8 + 2 * i], resc, p * f2.x); A.o[9 + 2 * i] = fmaf(A.o[9 + 2 * i], resc, p * f2.y);
    }
}
__device__ __forceinline__ void warp_merge(LaneAcc & A) {
#pragma unroll
    for (int off = 4; off < 32; off <<= 1) {
        const float m2 = __shfl_xor_sync(0xffffffffu, A.m, off), l2 = __shfl_xor_sync(0xffffffffu, A.l, off);
        const float mn = fmaxf(A.m, m2);
        const float w1 = (A.m > -INFINITY) ? __expf(A.m - mn) : 0.0f, w2 = (m2 > -INFINITY) ? __expf(m2 - mn) : 0.0f;
        A.l = A.l * w1 + l2 * w2; A.m = mn;
#pragma unroll
        for (int i = 0; i < 16; ++i) { const float o2 = __shfl_xor_sync(0xffffffffu, A.o[i], off); A.o[i] = A.o[i] * w1 + o2 * w2; }
    }
}
__device__ __forceinline__ void part_store(float * part, const LaneAcc & A, int lane) {    // lanes 0..3 write the warp partial
    if (lane < 4) {
        if (lane == 0) { part[0] = A.m; part[1] = A.l; }
#pragma unroll
        for (int i = 0; i < 16; i += 4) *reinterpret_cast<float4 *>(part + 4 + lane * 8 + (i >> 3) * 32 + (i & 7)) = make_float4(A.o[i], A.o[i + 1], A.o[i + 2], A.o[i + 3]);
    }
}
__device__ __forceinline__ float attn_merge(const float * pp, int nw, int dim, float & M, float & Lsum) {
    M = -INFINITY;
    for (int w = 0; w < nw; ++w) M = fmaxf(M, pp[w * PARTW]);
    Lsum = 0.0f;
    float o = 0.0f;
    for (int w = 0; w < nw; ++w) {
        const float mw = pp[w * PARTW];
        const float wgt = (mw > -INFINITY) ? __expf(mw - M) : 0.0f;
        Lsum = fmaf(pp[w * PARTW + 1], wgt, Lsum);
        o = fmaf(pp[w * PARTW + 4 + dim], wgt, o);
    }
    return o;
}

// self-attention over the paged cache (whisper.cpp:2603-2625) for the rows of the group.  Item = (row, head); a pair of warps takes one
// (4 items per CTA at a time).  A lane owns a key quarter; cell indices of 256 keys are requested at once, K / V of two key groups are
// double-buffered.  Same arithmetic as the first generation.
template <int WT>
__device__ __noinline__ void attn_self(const MkArgs & a, const int c_ci, const int c_cg, const int c_t_base, const int c_nt, const MkLayer & L) {
    constexpr int WPI = 2, SB = 2, CV = 8;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, grp = warp / WPI, hw = warp % WPI;
    const int d = a.d, H = a.n_head, n_pairs = c_nt * H;
    const uint64_t pol = policy_evict_first();
    const int kslot = lane >> 2, r = lane & 3;
    for (int p = c_ci * (W2 / WPI) + grp; p < n_pairs; p += c_cg * (W2 / WPI)) {
        const int tl = p / H, h = p - tl * H, t = c_t_base + tl;
        const int nk = a.nkv[t];
        const int * cells = a.idx + (size_t) t * a.ld_idx;
        float q[16];
        load_q16(a.qkv + (size_t) t * 3 * d + h * 64, r, q);
        LaneAcc A; lane_init(A);
        for (int kb = 0; kb < nk; kb += WPI * 8 * CV) {
            int cv[CV];
#pragma unroll
            for (int i = 0; i < CV; ++i) { const int k = kb + hw * 8 + i * WPI * 8 + kslot; cv[i] = (k < nk) ? __ldg(cells + k) : -1; }
            KV4 f[2][SB];
            auto fetch = [&](KV4 (&dst)[SB], int c0, int c1) {
                const int cx[SB] = { c0, c1 };
#pragma unroll
                for (int u = 0; u < SB; ++u) {
                    dst[u].k0 = dst[u].k1 = dst[u].v0 = dst[u].v1 = make_uint4(0, 0, 0, 0);
                    if (cx[u] >= 0) {
                        const size_t off = (size_t) cx[u] * d + h * 64 + r * 8;
                        const uint4 * kp = reinterpret_cast<const uint4 *>(L.kc + off), * vp = reinterpret_cast<const uint4 *>(L.vc + off);
                        dst[u].k0 = ldcg_hint(kp, pol); dst[u].k1 = ldcg_hint(kp + 4, pol); dst[u].v0 = ldcg_hint(vp, pol); dst[u].v1 = ldcg_hint(vp + 4, pol);
                    }
                }
            };
            fetch(f[0], cv[0], cv[1]);
#pragma unroll
            for (int gq = 0; gq < CV / SB; ++gq) {
                const bool more = (gq + 1 < CV / SB) && (kb + (gq + 1) * SB * WPI * 8 < nk);
                if (more) fetch(f[(gq + 1) & 1], cv[(2 * gq + 2) % CV], cv[(2 * gq + 3) % CV]);
#pragma unroll
                for (int u = 0; u < SB; ++u) {
                    float sc = dot16(f[gq & 1][u].k0, f[gq & 1][u].k1, q);
                    sc += __shfl_xor_sync(0xffffffffu, sc, 1);
                    sc += __shfl_xor_sync(0xffffffffu, sc, 2);
                    if (cv[2 * gq + u] >= 0) lane_update(A, sc, f[gq & 1][u].v0, f[gq & 1][u].v1);
                }
                if (!more) break;
            }
        }
        warp_merge(A);
        part_store(S_PART + (grp * WPI + hw) * PARTW, A, lane);
        bar_named(1 + grp, WPI * 32);
        {
            float M, Lsum;
            const float o = attn_merge(S_PART + grp * WPI * PARTW, WPI, hw * 32 + lane, M, Lsum);
            store_q<WT>(a.actq, d, t, h * 64 + hw * 32, lane, (Lsum > 0.0f) ? __fdividef(o, Lsum) : 0.0f);
        }
        bar_named(1 + grp, WPI * 32);
    }
}

// cross-attention over the n_keys padded encoder positions, zero rows included (whisper.cpp:2688-2705), for the rows of the group.
// K and V of a window live HEAD-MAJOR in HBM ([layer][head][key][64]): the keys of one (row, head) pair are one contiguous stream.
// Work unit = one (row, head) pair over ALL keys; CTA ci of the group takes the contiguous range of pairs [ci*P/cg, (ci+1)*P/cg).  Warp w,
// key slot s owns key 8w+s of every 64-key chunk; chunks are copied five ahead with cp.async into a 6-deep ring (80 KB in flight per
// CTA); every thread reads back only the 64 bytes it copied itself, so the ring needs no barrier.  The arithmetic of a pair (per-lane
// online softmax over its 24 keys, 8 key slots merged per warp, 8 warps merged in order) never depends on the rest of the batch.
__device__ __forceinline__ void cp_wait_ring() { asm volatile("cp.async.wait_group %0;" :: "n"(RING - 1) : "memory"); }

template <int WT>
__device__ __noinline__ void attn_cross(const MkArgs & a, const MkLayer & L) {
    const int c_ci = CX.ci, c_cg = CX.cg, c_t_base = CX.t_base, c_nt = CX.nt;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int d = a.d, H = a.n_head, nchp = a.n_keys / XKEYS;                 // chunks per pair
    const unsigned P = (unsigned) (c_nt * H), G = min((unsigned) c_cg, P);
    __syncthreads();                                                           // the staging areas are free
    if ((unsigned) c_ci >= G) return;
    const unsigned p0 = ((unsigned) c_ci * P) / G, p1 = (((unsigned) c_ci + 1) * P) / G;
    unsigned pl = p0, il = 0;
    int jl = 0, tl_ = (int) p0 / H, hl = (int) p0 - tl_ * H;
    const size_t head_stride = (size_t) a.n_keys * 64;
    const size_t lane_off = (size_t) (warp * 8 + (lane >> 2)) * 64 + (lane & 3) * 8;       // key 8w+s of the chunk, dims {8r.., 32+8r..}
    const uint32_t ring = (uint32_t) __cvta_generic_to_shared(sm) + tid * 16;
    const bool ef = (a.prefetch & 4) != 0;                           // stream K / V through L2 with evict-first priority: 500 MB per layer would flush weights and activations
    const uint64_t pol = policy_evict_first();
    const float kq_scale = a.kq_scale;
    // Everything the copy path needs lives in registers: the asm statements are memory barriers for the compiler, a value it has to
    // re-read from the argument structs after each of them is a dependent load in front of every chunk (measured: the per-chunk
    // a.slot[] load, an L2 round trip with this little L1, capped a CTA at 19 GB/s).  The slot of a row is fetched one row ahead.
    const __half * const xk = L.xk, * const xv = L.xv;
    const int64_t slot_stride = a.slot_stride;
    const int * const slots = a.slot + c_t_base;
    const int nt = c_nt;
    int slot_cur = slots[tl_], slot_nxt = (tl_ + 1 < nt) ? slots[tl_ + 1] : 0;
    size_t pair_off = (size_t) slot_cur * slot_stride + (size_t) hl * head_stride + lane_off;
    auto issue = [&]() {                                           // copy the next chunk (if any) into ring slot il % RING; always commits a group
        if (pl < p1) {
            const size_t off = pair_off + (size_t) (jl * XKEYS) * 64;
            const uint32_t sa = ring + (il % RING) * RING_SLOT;
            if (ef) {
                cp_async16_hint(sa, xk + off, pol); cp_async16_hint(sa + T2 * 16, xk + off + 32, pol);
                cp_async16_hint(sa + 2 * T2 * 16, xv + off, pol); cp_async16_hint(sa + 3 * T2 * 16, xv + off + 32, pol);
            } else {
                cp_async16(sa, xk + off); cp_async16(sa + T2 * 16, xk + off + 32);
                cp_async16(sa + 2 * T2 * 16, xv + off); cp_async16(sa + 3 * T2 * 16, xv + off + 32);
            }
            if (++jl == nchp) {
                jl = 0; ++pl;
                if (++hl == H) { hl = 0; ++tl_; slot_cur = slot_nxt; slot_nxt = (tl_ + 1 < nt) ? slots[tl_ + 1] : 0; }
                pair_off = (size_t) slot_cur * slot_stride + (size_t) hl * head_stride + lane_off;
            }
        }
        ++il;
        cp_commit();
    };
#pragma unroll
    for (int k = 0; k < RING - 1; ++k) issue();
    int tl = (int) p0 / H, h = (int) p0 - tl * H;
    float * qsm = reinterpret_cast<float *>(sm + OFF_QSM);        // f16-rounded query of the pair: [2][64], lane order: 16*r + 8*hi + i holds dim 32*hi + 8*r + i
    if (warp >= 2 && warp < 4) { const int dim = (warp - 2) * 32 + lane; qsm[((dim & 31) >> 3) * 16 + (dim >> 5) * 8 + (dim & 7)] = __half2float(__float2half_rn(__ldcg(a.q2 + (size_t) (c_t_base + tl) * d + h * 64 + dim))); }
    __syncthreads();
    LaneAcc A; lane_init(A);
    int buf = 0, j = 0;
    unsigned ic = 0;
    for (unsigned p = p0; p < p1; ) {
        issue();
        cp_wait_ring();                                          // this thread's copies of chunk ic have landed
        const uint8_t * sl = sm + (ic % RING) * RING_SLOT + tid * 16;
        ++ic;
        const uint4 k0 = *reinterpret_cast<const uint4 *>(sl), k1 = *reinterpret_cast<const uint4 *>(sl + T2 * 16);
        const uint4 v0 = *reinterpret_cast<const uint4 *>(sl + 2 * T2 * 16), v1 = *reinterpret_cast<const uint4 *>(sl + 3 * T2 * 16);
        float sc = dot16s(k0, k1, qsm + buf * 64 + (lane & 3) * 16);
        sc += __shfl_xor_sync(0xffffffffu, sc, 1);
        sc += __shfl_xor_sync(0xffffffffu, sc, 2);
        lane_update(A, sc * kq_scale, v0, v1);
        if (++j < nchp) continue;
        j = 0;                                                   // last chunk of the pair: merge the CTA and write the row's head
        warp_merge(A);
        part_store(S_PART + (buf * W2 + warp) * PARTW, A, lane);
        if (p + 1 < p1 && warp >= 2 && warp < 4) {               // query of the next pair
            int tn = tl, hn = h;
            if (++hn == H) { hn = 0; ++tn; }
            const int dim = (warp - 2) * 32 + lane;
            qsm[(buf ^ 1) * 64 + ((dim & 31) >> 3) * 16 + (dim >> 5) * 8 + (dim & 7)] = __half2float(__float2half_rn(__ldcg(a.q2 + (size_t) (c_t_base + tn) * d + hn * 64 + dim)));
        }
        __syncthreads();
        if (warp < 2) {                                          // merge the 8 warp partials (one output dim per thread)
            const int dim = warp * 32 + lane;
            float M, Lsum;
            const float o = attn_merge(S_PART + buf * W2 * PARTW, W2, dim, M, Lsum);
            store_q<WT>(a.actq, d, c_t_base + tl, h * 64 + warp * 32, lane, __fdividef(o, Lsum));
        }
        buf ^= 1;
        lane_init(A);
        ++p;
        if (++h == H) { h = 0; ++tl; }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");
}

__device__ __forceinline__ long long gtime() { long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
#define MK_GSTAMP(k) do { if (TRACE && CX.ci == 0 && threadIdx.x == 0) a.trace[3000 + (l * NGMAX + CX.g) * 3 + (k)] = gtime(); } while (0)
#define MK_SYNC() do { MK_STAMP(); grp_sync(a); MK_STAMP(); } while (0)
#define MK_NOP_PHASE() do { MK_STAMP(); MK_STAMP(); } while (0)

template <int WT, bool TRACE>
__global__ void __launch_bounds__(T2, CPS)
k_decode_pass2(const __grid_constant__ MkArgs a) {
    if (threadIdx.x == 0) { mbar_init(S_MBAR, 1); mbar_init(S_MBAR + 1, 1); mbar_init(S_MBAR + 2, 1); mbar_fence_init(); }
    if (threadIdx.x == 0) {
        Ctx & c = CX;
        const int n_sm = (int) gridDim.x / CPS;
        c.n_sm = n_sm;
        c.NG = (a.n_tok + RG - 1) / RG;
        const int s_me = (int) blockIdx.x / n_sm, j_me = (int) blockIdx.x - s_me * n_sm;
        c.g = (j_me + s_me) % c.NG;
        c.cg = 0; c.ci = 0;
        for (int s = 0; s < CPS; ++s) {
            c.r_s[s] = ((c.g - s) % c.NG + c.NG) % c.NG;
            c.cnt_s[s] = (c.r_s[s] < n_sm) ? (n_sm - c.r_s[s] + c.NG - 1) / c.NG : 0;
            if (s < s_me) c.ci += c.cnt_s[s];
            c.cg += c.cnt_s[s];
        }
        c.ci += (j_me - c.r_s[s_me]) / c.NG;
        c.t_base = c.g * RG; c.nt = min(RG, a.n_tok - c.t_base);
        c.kbar = 0; c.kglob = 0; c.par[0] = c.par[1] = c.par[2] = 0;
    }
    __syncthreads();
    int n_stamp = 0;
    const int d = a.d;
    const bool pf_w = a.prefetch & 1;
    const bool xserial = (a.prefetch & 8) != 0;
    if (a.stagger_clk > 0 && CX.g > 0) {                           // groups start staggered so that their HBM-bound phases do not coincide
        const long long t0 = clock64(), w = (long long) a.stagger_clk * CX.g;
        while (clock64() - t0 < w) __nanosleep(256);
    }
    MK_STAMP();
    if (pf_w) prefetch_w(a.layers[0].qkv);

    for (int l = 0; l < a.n_layer; ++l) {
        const MkLayer & L = a.layers[l];
        Epi e;
        // 1+2: LN (whisper.cpp:2536-2543) folded into QKV + KV append (2545-2599)
        MK_GSTAMP(0);
        MK_NOP_PHASE();
        e = Epi(); e.bias = L.qkv_bias; e.scale = L.qkv_scale; e.out = a.qkv; e.kc = L.kc; e.vc = L.vc; e.kv_d = d;
        gemv<WT, false, true>(a, L.qkv, nullptr, a.x, L.ln0_w, L.ln0_b, e, (TRACE && l == 1) ? 2048 + 0 : -1);
        if (pf_w) prefetch_w(L.o);
        MK_SYNC();
        if (a.global_sync) all_sync(a);                       // a row may attend to cells another group has just appended
        // 3: self-attention (2603-2625) -> quantised rows for the O projection
        if (pf_w) prefetch_w(L.cq);
        attn_self<WT>(a, CX.ci, CX.cg, CX.t_base, CX.nt, L);
        MK_SYNC();
        // 4: O + residual (2647-2659)
        e = Epi(); e.bias = L.o_bias; e.res = a.x; e.out = a.x;
        gemv<WT, false, false>(a, L.o, a.actq, nullptr, nullptr, nullptr, e, (TRACE && l == 1) ? 2048 + 8 : -1);
        if (pf_w) prefetch_w(L.co);
        MK_SYNC();
        // 5+6: LN folded into cross Q (2661-2681)
        MK_NOP_PHASE();
        e = Epi(); e.bias = L.cq_bias; e.out = a.q2;
        gemv<WT, false, true>(a, L.cq, nullptr, a.x, L.lnc_w, L.lnc_b, e, (TRACE && l == 1) ? 2048 + 16 : -1);
        if (pf_w) prefetch_w(L.fc1);
        MK_SYNC();
        // 7: cross-attention (2688-2705)
        if (xserial) cross_turn_wait(a, l);
        MK_GSTAMP(1);
        attn_cross<WT>(a, L);
        MK_SYNC();
        if (xserial) cross_turn_done(a);
        MK_GSTAMP(2);
        // 8: cross O + residual (2754-2766)
        e = Epi(); e.bias = L.co_bias; e.res = a.x; e.out = a.x;
        gemv<WT, false, false>(a, L.co, a.actq, nullptr, nullptr, nullptr, e, (TRACE && l == 1) ? 2048 + 24 : -1);
        if (pf_w) prefetch_w(L.fc2);
        MK_SYNC();
        // 9+10: LN folded into FC1 + GELU (2770-2794); the epilogue writes the quantised rows FC2 consumes
        MK_NOP_PHASE();
        e = Epi(); e.bias = L.fc1_bias; e.act = 1; e.qout = a.hq;
        gemv<WT, true, true>(a, L.fc1, nullptr, a.x, L.lnm_w, L.lnm_b, e, (TRACE && l == 1) ? 2048 + 32 : -1);
        if (pf_w) { if (l + 1 < a.n_layer) prefetch_w(a.layers[l + 1].qkv); }
        MK_STAMP(); MK_STAMP();
        MK_SYNC();
        // 11: FC2 + residual (2797-2806)
        e = Epi(); e.bias = L.fc2_bias; e.res = a.x; e.out = a.x;
        gemv<WT, false, false>(a, L.fc2, a.hq, nullptr, nullptr, nullptr, e, (TRACE && l == 1) ? 2048 + 40 : -1);
        MK_SYNC();
    }
    if (a.want_logits) {                                         // final LN + logits (2811-2827)
        MK_NOP_PHASE();
        Epi e; e.out = a.logits;
        gemv<WT, false, true>(a, a.te, nullptr, a.x, a.lnf_w, a.lnf_b, e);
        MK_STAMP();
    }
}

} // namespace mk2

int  mk2_ctas_per_sm() { return mk2::CPS; }
int  mk2_barriers(int n_layer, bool) { return 8 * n_layer; }
bool mk2_supported(int wtype, int d) { return (wtype == WT_F16 || wt_is_block32(wtype)) && d <= 1280 && (d & 127) == 0; }
size_t mk2_smem_bytes() { return mk2::SMEM; }
size_t mk2_bar_words(int n_sm) { return 128 + 16 * (size_t) mk2::CPS * n_sm; }

template <int WT, bool TRACE>
static bool mk2_launch_t(const MkArgs & a, int n_sm, cudaStream_t st) {
    const void * fn = reinterpret_cast<const void *>(mk2::k_decode_pass2<WT, TRACE>);
    static bool checked = false;
    if (!checked) {
        if (ensure_dyn_smem(fn, mk2::SMEM) != cudaSuccess) { set_error("decode kernel: cannot raise the shared-memory limit"); return false; }
        int nb = 0;
        if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, fn, mk2::T2, mk2::SMEM) != cudaSuccess || nb < mk2::CPS) {
            set_error("decode kernel: %d CTAs per SM fit, %d are needed", nb, mk2::CPS); return false;
        }
        checked = true;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(mk2::CPS * n_sm); cfg.blockDim = dim3(mk2::T2); cfg.dynamicSmemBytes = mk2::SMEM; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeCooperative; at[0].val.cooperative = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, mk2::k_decode_pass2<WT, TRACE>, a);
    if (e != cudaSuccess) { set_error("decode kernel launch: %s", cudaGetErrorString(e)); return false; }
    count_launch();
    return true;
}

bool mk2_launch(const MkArgs & a, int wtype, int n_sm, cudaStream_t st) {
    if (a.te.layout != 1) { set_error("decode kernel: weights are not in the tile-major layout"); return false; }
    if (cudaMemsetAsync(a.bar, 0, 128 * sizeof(unsigned long long), st) != cudaSuccess) { set_error("decode kernel: barrier reset failed"); return false; }
#define WB_MK(T) (a.trace ? mk2_launch_t<T, true>(a, n_sm, st) : mk2_launch_t<T, false>(a, n_sm, st))
    switch (wtype) {
        case WT_F16:  return WB_MK(WT_F16);
        case WT_Q4_0: return WB_MK(WT_Q4_0);
        case WT_Q5_0: return WB_MK(WT_Q5_0);
        case WT_Q8_0: return WB_MK(WT_Q8_0);
        default: set_error("decode kernel: unsupported weight type %d", wtype); return false;
    }
#undef WB_MK
}

} // namespace wb
