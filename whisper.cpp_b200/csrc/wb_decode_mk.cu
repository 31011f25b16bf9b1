// wb_decode_mk.cu -- one decoder pass (<= 64 rows) as a single persistent cooperative kernel.
//
// What it computes is whisper_build_graph_decoder (src/whisper.cpp:2466-2844) for the rows of one whisper_batch:
//   per layer:  LN -> QKV (+KV append) -> self-attention over the paged cache -> O + residual
//               LN -> Q -> cross-attention over the padded encoder keys       -> O + residual
//               LN -> FC1 + GELU -> FC2 + residual
//   then LN -> logits (token-embedding matrix).
// The arithmetic per op is the one of the stand-alone kernels in wb_kernels.cu (Q8_0 activation blocks + integer block
// dots like the reference CPU path -- Q8_K super-blocks for Q4_K / Q5_K weights --, f16-rounded Q, f32 softmax); this file changes HOW
// the ops are scheduled:
//   * grid = one CTA of 16 warps per SM, launched cooperatively; a phase boundary is a grid barrier instead of a kernel
//     boundary (the decode step is a chain of ~400 dependent phases of a few microseconds each); a pass of 32 rows or more is cut into
//     partitions (row groups x CTA ranges, MkView) that walk the layers on their own barriers and take turns streaming cross K/V;
//   * rows handed from one phase to the next are quantised once by their producer ("actq" rows in global memory): a
//     distributed LayerNorm -> Q8_0 phase, attention epilogues, and a quantise phase after FC1;
//   * a GEMV phase is cut by row group first: a CTA stages the 16 rows of its group with TMA bulk copies and walks 16-row
//     weight tiles, its 16 warps split K and reduce through smem.  Weights are stored tile-major (wb_quant.cuh): a warp fetches
//     the MMA operands of one (tile, block) with three fully coalesced loads -- with the planar layout every 4-byte gather cost
//     16 sectors per 128 useful bytes and the phase was L1-sector bound;
//   * cross-attention (the HBM-heavy part: 2*n_keys*d f16 per row and layer) is cut into (row, head, half of the keys) units,
//     streamed through a cp.async ring; one lane owns one key-quarter and keeps its own online-softmax state.
// Lessons that shaped the code: no pointers handed through structs (they turn shared-memory accesses into generic
// loads), no 64-bit divisions in loops, approximate reciprocals where they only feed a rounding, no register moves of
// in-flight loads, whole 32-byte sectors per load instruction, bulk copies instead of register staging for anything > 16 KB.
#include <cmath>
#include <type_traits>
#include "wb_decode_mk.cuh"
#include "wb_dtw_kernel.cuh"
#include "wb_common.h"
#include "wb_dev.cuh"
#include "wb_ptx.cuh"
#include "wb_tm.cuh"

namespace wb {

constexpr int MK_THREADS = 512, MK_WARPS = 16, MK_XKEYS = 128, MK_MAXTOK = 64, MK_RED = 4 * 16 * 16 * 17, MK_PART = 68;
constexpr int MK_TP = 4;                // weight tiles a GEMV phase keeps in flight per iteration
static_assert(MK_TP * 16 * 16 * 17 <= MK_RED, "split-K reduction buffer");
constexpr int MK_ROWB = 1280;            // bytes of one staged activation row chunk (1280 int8 values or 640 halves)

// dynamic shared memory, fixed carve-up (every phase function addresses it directly: pointers handed through a struct in
// local memory turned every access into a generic load)
extern __shared__ __align__(16) uint8_t mk_smem[];
constexpr int MK_OFF_XQ   = 0;                                                   // staged activation rows [64][SW words]
constexpr int MK_OFF_XD   = MK_OFF_XQ + MK_MAXTOK * (MK_ROWB + 16);              // their Q8_0 block scales [64][chunk/32]
constexpr int MK_OFF_RED  = MK_OFF_XD + MK_MAXTOK * (MK_ROWB / 32) * 4;          // split-K partials [MK_TP tiles][16 warps][16 rows][17]
constexpr int MK_OFF_PART = MK_OFF_RED + MK_RED * 4;                             // attention warp partials [2][16][68]: m, l, -, -, o[64]
constexpr int MK_OFF_STAT = MK_OFF_PART + 2 * MK_WARPS * MK_PART * 4;            // LayerNorm partial sums [32]
constexpr int MK_OFF_FLAG = MK_OFF_STAT + 32 * 4;                                // [16] ints
constexpr int MK_SMEM     = MK_OFF_FLAG + 16 * 4;
#define SM_XQ   (reinterpret_cast<uint32_t *>(mk_smem + MK_OFF_XQ))
#define SM_XD   (reinterpret_cast<float *>(mk_smem + MK_OFF_XD))
#define SM_RED  (reinterpret_cast<float *>(mk_smem + MK_OFF_RED))
#define SM_PART (reinterpret_cast<float *>(mk_smem + MK_OFF_PART))
#define SM_STAT (reinterpret_cast<float *>(mk_smem + MK_OFF_STAT))
#define SM_FLAG (reinterpret_cast<int *>(mk_smem + MK_OFF_FLAG))

#define MK_STAMP() do { if (TRACE) { if (blockIdx.x == 0 && threadIdx.x == 0) a.trace[n_stamp] = clock64(); ++n_stamp; } } while (0)

__device__ __forceinline__ void l2_prefetch(const void * p, uint32_t bytes) {
    if (bytes >= 16) asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" :: "l"(p), "r"(bytes & ~15u) : "memory");
}

// What a phase function knows about who shares the phase with its CTA: the CTA's index among the `nc` CTAs of its partition and the
// partition's rows [row0, row0 + n_tok).  part = -1: the whole grid (logits).
struct MkView { int ci, nc, row0, n_tok, part; };

// words of MkArgs::bar: [0] arrival counter of the grid, [8] error flag, [16 + 16*cta + w] release flags of a CTA (one 128-byte line per CTA;
// w = 0: grid barrier, 1 + p: barrier of partition p -- a flag only ever sees the targets of one counter, so it stays monotonic when the
// number of partitions changes from pass to pass), then one line per partition counter and one for the turn word
__device__ __forceinline__ unsigned long long * mk_bar_tail(const MkArgs & a, int i) { return a.bar + 16 + 16 * (size_t) gridDim.x + 16 * i; }
constexpr int MK_TRACE_TURN = 2100;     // trace slot: SM clocks partition 0 waited for its turn to stream (accumulates)

// Barrier of the CTAs of a view.  Arrival = one atomic on the view's counter; the LAST CTA to arrive releases the others by writing one
// flag per CTA (each on its own 128-byte line), and every other CTA polls only its own flag.
// turn = 1 (the barrier in front of the cross-attention, several partitions): the releasing CTA first waits until fewer than
// a.turn_slots partitions are streaming K/V and takes a slot; turn = 2 (the barrier behind it): the partition gives the slot back.  A
// partition that holds a slot never waits for another partition, and all CTAs are resident: the wait always ends.
__device__ __noinline__ void mk_grid_sync(const MkArgs & a, const MkView v, unsigned long long target, int turn) {
    unsigned long long * const cnt = v.part < 0 ? a.bar : mk_bar_tail(a, v.part);
    unsigned long long * const turn_w = mk_bar_tail(a, MK_MAX_PARTS);
    if (a.n_part == 1) turn = 0;
    __syncthreads();
    if ((a.prefetch & 32) && turn != 1) {
        // variant: arrival = a reduction without a return value, and EVERY CTA polls the counter itself -- no dependent chain
        // "atomic returns -> last arriver writes the flags -> the flags become visible" (one L2 round trip less per barrier)
        if (threadIdx.x == 0) {
            __threadfence();
            asm volatile("red.release.gpu.global.add.u64 [%0], 1;" :: "l"(cnt) : "memory");
            const long long t0 = clock64();
            unsigned long long c;
            for (;;) {
                asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(c) : "l"(cnt) : "memory");
                if (c >= target) break;
                if (clock64() - t0 > (6LL << 30)) { *a.err = 1; __threadfence_system(); __trap(); }
            }
            if (turn == 2 && v.ci == 0) atomicAdd(turn_w, ~0ULL);
        }
        __syncthreads();
        return;
    }
    if (threadIdx.x == 0) {
        __threadfence();
        const unsigned long long old = atomicAdd(cnt, 1ULL);
        SM_FLAG[2] = (old + 1 == target);
        if (old + 1 == target) {
            __threadfence();                                     // the last arriver acquires what the others released
            if (turn == 1) {
                const long long t0 = clock64();
                for (;;) {
                    unsigned long long s;
                    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(s) : "l"(turn_w) : "memory");
                    if (s < (unsigned long long) a.turn_slots && atomicCAS(turn_w, s, s + 1) == s) break;
                    if (clock64() - t0 > (6LL << 30)) { *a.err = 1; __threadfence_system(); __trap(); }
                }
                if (a.trace && v.part == 0) atomicAdd(reinterpret_cast<unsigned long long *>(a.trace) + MK_TRACE_TURN, (unsigned long long) (clock64() - t0));
            }
        }
    }
    __syncthreads();
    unsigned long long * const flags = a.bar + 16 + 16 * (size_t) (blockIdx.x - v.ci) + (v.part + 1);
    if (SM_FLAG[2]) {
        for (int i = threadIdx.x; i < v.nc; i += MK_THREADS)
            asm volatile("st.release.gpu.global.u64 [%0], %1;" :: "l"(flags + 16 * i), "l"(target) : "memory");
    } else if (threadIdx.x == 0) {
        const unsigned long long * f = flags + 16 * v.ci;
        const long long t0 = clock64();
        unsigned long long c;
        for (;;) {
            asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(c) : "l"(f) : "memory");
            if (c >= target) break;
            if (clock64() - t0 > (6LL << 30)) { *a.err = 1; __threadfence_system(); __trap(); }    // ~3 s: a CTA never arrived
        }
    }
    if (turn == 2 && v.ci == 0 && threadIdx.x == 0) atomicAdd(turn_w, ~0ULL);
    __syncthreads();
}

// ---- activation rows ("actq" format) ----------------------------------------------------------------------------------------
// Rows handed from one phase to the next are quantised ONCE by their producer and live in global memory: block-32 weight types:
// int8 [64][K] followed by f32 block scales [64][K/32]; F16 weights: half [64][K].  A GEMV phase stages them chunk-wise in smem.
// Q8_0 rows follow quantize_row_q8_0 (d = amax/127 stored as f16, q = rint(x * 127/amax)); the two quotients are formed with a
// reciprocal multiply / __fdividef: <= 2 ulp from the IEEE quotient, which only matters within 1e-6 of a rounding boundary.

// K-quant weights: rows are Q8_K (quantize_row_q8_K, ggml-quants.c:2768-2805, the arithmetic of k_act_quant<1>): int8 [64][K] followed
// by one K/8-byte record per row (the size of the Q8_0 scales, so the staging is the same): f32 d[K/256] | int16 sum[K/32] of each
// 32 quantised values (the dmin term).  A 256-value super-block needs its signed value of largest magnitude: producers that see
// less than a super-block (attention heads, FC1 tiles) write f32 rows, and a quantise phase (mk_q8k_rows) follows them.
// Q3_K uses the same rows without the sums: signed weights, one integer scale per 16 values, no minimum.
constexpr bool mk_kq(int WT) { return WT == WT_Q4_K || WT == WT_Q5_K || WT == WT_Q3_K; }

// Q4_1 / Q5_1 weights: rows are Q8_1 (quantize_row_q8_1, AVX2 form ggml-cpu/arch/x86/quants.c): the int8 values of Q8_0 (with the IEEE
// quotients 127/amax and amax/127 the reference uses), and in place of each f32 block scale the pair {f16 d, f16 s = d * sum(q)} (s from
// the unrounded d) -- same bytes per row, so staging and workspaces are those of Q8_0.  The block dot is (d_w d_x) sumi + m_w s_x.
constexpr bool mk_q1(int WT) { return WT == WT_Q4_1 || WT == WT_Q5_1; }
__device__ __forceinline__ uint32_t q8_1_pair(float d, int sum) {
    const __half2 p = __halves2half2(__float2half_rn(d), __float2half_rn(d * (float) sum));
    return *reinterpret_cast<const uint32_t *>(&p);
}

// the signed value of largest magnitude of two candidates; ties go to the larger value, so the choice does not depend on the order
// (a tie between x and -x only flips the signs of q and d together)
__device__ __forceinline__ void q8k_pick(float & amax, float & mx, float oa, float om) {
    if (oa > amax || (oa == amax && om > mx)) { amax = oa; mx = om; }
}
__device__ __forceinline__ void q8k_warp_max(float & amax, float & mx) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) q8k_pick(amax, mx, __shfl_xor_sync(0xffffffffu, amax, o), __shfl_xor_sync(0xffffffffu, mx, o));
}
// q = min(127, nearest(iscale * x)) of four values, packed; `sum` gets their sum
__device__ __forceinline__ uint32_t q8k_pack4(const float4 & y, float iscale, bool zero, int & sum) {
    int q0 = 0, q1 = 0, q2 = 0, q3 = 0;
    if (!zero) {
        q0 = min(127, __float2int_rn(iscale * y.x)); q1 = min(127, __float2int_rn(iscale * y.y));
        q2 = min(127, __float2int_rn(iscale * y.z)); q3 = min(127, __float2int_rn(iscale * y.w));
    }
    sum = (q0 + q1) + (q2 + q3);
    return ((uint32_t) q0 & 0xffu) | (((uint32_t) q1 & 0xffu) << 8) | (((uint32_t) q2 & 0xffu) << 16) | ((uint32_t) q3 << 24);
}
__device__ __forceinline__ int sum8_lanes(int s) {              // over the 8 lanes of one 32-value sub-block (4 values per lane)
    s += __shfl_xor_sync(0xffffffffu, s, 1); s += __shfl_xor_sync(0xffffffffu, s, 2); s += __shfl_xor_sync(0xffffffffu, s, 4);
    return s;
}
__device__ __forceinline__ float * q8k_d(uint8_t * dst, int K, int row) { return reinterpret_cast<float *>(dst + (size_t) MK_MAXTOK * K + (size_t) row * (K >> 3)); }

// one warp quantises the 32 values its lanes hold (one Q8_0 block of row t starting at element e0); K-quants: f32 store (see above)
template <int WT>
__device__ __forceinline__ void mk_store_q(uint8_t * dst, int K, int t, int e0, int lane, float v) {
    if (WT == WT_F16) { reinterpret_cast<__half *>(dst)[(size_t) t * K + e0 + lane] = __float2half_rn(v); return; }
    if (mk_kq(WT)) { reinterpret_cast<float *>(dst)[(size_t) t * K + e0 + lane] = v; return; }
    if (mk_q1(WT)) {
        const float amax = warp_max(fabsf(v));
        const int q = __float2int_rn(v * ((amax != 0.0f) ? 127.0f / amax : 0.0f));
        reinterpret_cast<int8_t *>(dst)[(size_t) t * K + e0 + lane] = (int8_t) q;
        const int sum = __reduce_add_sync(0xffffffffu, q);
        if (lane == 0) reinterpret_cast<uint32_t *>(dst + (size_t) MK_MAXTOK * K)[t * (K >> 5) + (e0 >> 5)] = q8_1_pair(amax / 127.0f, sum);
        return;
    }
    const float amax = warp_max(fabsf(v));
    const float id = (amax != 0.0f) ? __fdividef(127.0f, amax) : 0.0f;
    reinterpret_cast<int8_t *>(dst)[(size_t) t * K + e0 + lane] = (int8_t) __float2int_rn(v * id);
    if (lane == 0) reinterpret_cast<float *>(dst + (size_t) MK_MAXTOK * K)[t * (K >> 5) + (e0 >> 5)] = __half2float(__float2half_rn(amax * (1.0f / 127.0f)));
}

// Q8_1 of four values per lane, 8 lanes per 32-value block (amax already reduced over the 8 lanes)
__device__ __forceinline__ void mk_q8_1_store4(uint8_t * dst, int K, int row, int e0, int lane, const float4 & y, float amax) {
    const float id = (amax != 0.0f) ? 127.0f / amax : 0.0f;
    const int q0 = __float2int_rn(y.x * id), q1 = __float2int_rn(y.y * id), q2 = __float2int_rn(y.z * id), q3 = __float2int_rn(y.w * id);
    *reinterpret_cast<uint32_t *>(dst + (size_t) row * K + e0) = ((uint32_t) q0 & 0xffu) | (((uint32_t) q1 & 0xffu) << 8) | (((uint32_t) q2 & 0xffu) << 16) | ((uint32_t) q3 << 24);
    const int sum = sum8_lanes((q0 + q1) + (q2 + q3));
    if ((lane & 7) == 0) reinterpret_cast<uint32_t *>(dst + (size_t) MK_MAXTOK * K)[row * (K >> 5) + (e0 >> 5)] = q8_1_pair(amax / 127.0f, sum);
}

// LayerNorm (ggml-cpu/ops.cpp:3698-3765, two passes, then mul/add whisper.cpp:2536-2543) of the f32 residual rows, quantised into
// `dst`.  Distributed: CTA r of the view normalises its row r (one warp per 128 values); followed by a barrier.
template <int WT>
__device__ __noinline__ void mk_lnq(const MkArgs & a, const MkView v, const float * src, int K, const float * __restrict__ ln_w, const float * __restrict__ ln_b, uint8_t * dst) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int row = v.row0 + v.ci; row < v.row0 + v.n_tok; row += v.nc) {
        const bool act = warp < (K >> 7);
        const int e0 = warp * 128 + lane * 4;
        float4 v = act ? __ldcg(reinterpret_cast<const float4 *>(src + (size_t) row * K + e0)) : make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        float s = warp_sum((v.x + v.y) + (v.z + v.w));
        if (lane == 0) SM_STAT[warp] = s;
        __syncthreads();
        s = (lane < MK_WARPS) ? SM_STAT[lane] : 0.0f;
        const float mean = warp_sum(s) / K;
        float q = 0.0f;
        if (act) { v.x -= mean; v.y -= mean; v.z -= mean; v.w -= mean; q = (v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w); }
        q = warp_sum(q);
        if (lane == 0) SM_STAT[16 + warp] = q;
        __syncthreads();
        q = (lane < MK_WARPS) ? SM_STAT[16 + lane] : 0.0f;
        const float rstd = 1.0f / sqrtf(warp_sum(q) / K + a.eps);
        float4 y = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        if (act) {
            const float4 w = __ldg(reinterpret_cast<const float4 *>(ln_w + e0)), b = __ldg(reinterpret_cast<const float4 *>(ln_b + e0));
            y.x = __fadd_rn(__fmul_rn(__fmul_rn(v.x, rstd), w.x), b.x);
            y.y = __fadd_rn(__fmul_rn(__fmul_rn(v.y, rstd), w.y), b.y);
            y.z = __fadd_rn(__fmul_rn(__fmul_rn(v.z, rstd), w.z), b.z);
            y.w = __fadd_rn(__fmul_rn(__fmul_rn(v.w, rstd), w.w), b.w);
        }
        if (mk_kq(WT)) {                                         // Q8_K: a super-block is the 256 values of warps 2s, 2s + 1
            float amax = fabsf(y.x), mx = y.x;
            q8k_pick(amax, mx, fabsf(y.y), y.y); q8k_pick(amax, mx, fabsf(y.z), y.z); q8k_pick(amax, mx, fabsf(y.w), y.w);
            q8k_warp_max(amax, mx);
            if (lane == 0) { SM_PART[2 * warp] = amax; SM_PART[2 * warp + 1] = mx; }
            __syncthreads();
            if (act) {
                const int w0 = warp & ~1;
                amax = SM_PART[2 * w0]; mx = SM_PART[2 * w0 + 1];
                q8k_pick(amax, mx, SM_PART[2 * w0 + 2], SM_PART[2 * w0 + 3]);
                const float iscale = (amax != 0.0f) ? -127.0f / mx : 0.0f;
                int s;
                *reinterpret_cast<uint32_t *>(dst + (size_t) row * K + e0) = q8k_pack4(y, iscale, amax == 0.0f, s);
                s = sum8_lanes(s);
                float * dd = q8k_d(dst, K, row);
                if ((lane & 7) == 0) reinterpret_cast<short *>(dd + (K >> 8))[e0 >> 5] = (short) s;
                if (lane == 0 && (warp & 1) == 0) dd[e0 >> 8] = (amax != 0.0f) ? 1.0f / iscale : 0.0f;
            }
        } else if (act) {
            if (WT == WT_F16) {
                const __half2 h0 = __floats2half2_rn(y.x, y.y), h1 = __floats2half2_rn(y.z, y.w);
                *reinterpret_cast<uint2 *>(reinterpret_cast<__half *>(dst) + (size_t) row * K + e0) = make_uint2(*reinterpret_cast<const uint32_t *>(&h0), *reinterpret_cast<const uint32_t *>(&h1));
            } else {
                float amax = fmaxf(fmaxf(fabsf(y.x), fabsf(y.y)), fmaxf(fabsf(y.z), fabsf(y.w)));
                amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 1));
                amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 2));
                amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, 4));
                if (mk_q1(WT)) { mk_q8_1_store4(dst, K, row, e0, lane, y, amax); } else {
                const float id = (amax != 0.0f) ? __fdividef(127.0f, amax) : 0.0f;
                const uint32_t q0 = (uint32_t) __float2int_rn(y.x * id) & 0xffu, q1 = (uint32_t) __float2int_rn(y.y * id) & 0xffu;
                const uint32_t q2 = (uint32_t) __float2int_rn(y.z * id) & 0xffu, q3 = (uint32_t) __float2int_rn(y.w * id) & 0xffu;
                *reinterpret_cast<uint32_t *>(dst + (size_t) row * K + e0) = q0 | (q1 << 8) | (q2 << 16) | (q3 << 24);
                if ((lane & 7) == 0) reinterpret_cast<float *>(dst + (size_t) MK_MAXTOK * K)[row * (K >> 5) + (e0 >> 5)] = __half2float(__float2half_rn(amax * (1.0f / 127.0f)));
                }
            }
        }
        __syncthreads();
    }
}

// K-quants: f32 rows (`lds` floats apart) -> Q8_K rows, one warp per (row, super-block); followed by a barrier
__device__ __noinline__ void mk_q8k_rows(const MkView v, const float * src, int lds, int K, uint8_t * dst) {
    const int lane = threadIdx.x & 31, nsb = K >> 8, n = v.n_tok * nsb;
    for (int p = v.ci * MK_WARPS + (threadIdx.x >> 5); p < n; p += v.nc * MK_WARPS) {
        const int row = v.row0 + p / nsb, e0 = (p - (row - v.row0) * nsb) * 256 + lane * 4;
        const float4 y0 = __ldcg(reinterpret_cast<const float4 *>(src + (size_t) row * lds + e0));
        const float4 y1 = __ldcg(reinterpret_cast<const float4 *>(src + (size_t) row * lds + e0 + 128));
        float amax = fabsf(y0.x), mx = y0.x;
        q8k_pick(amax, mx, fabsf(y0.y), y0.y); q8k_pick(amax, mx, fabsf(y0.z), y0.z); q8k_pick(amax, mx, fabsf(y0.w), y0.w);
        q8k_pick(amax, mx, fabsf(y1.x), y1.x); q8k_pick(amax, mx, fabsf(y1.y), y1.y); q8k_pick(amax, mx, fabsf(y1.z), y1.z); q8k_pick(amax, mx, fabsf(y1.w), y1.w);
        q8k_warp_max(amax, mx);
        const float iscale = (amax != 0.0f) ? -127.0f / mx : 0.0f;
        int s0, s1;
        *reinterpret_cast<uint32_t *>(dst + (size_t) row * K + e0)       = q8k_pack4(y0, iscale, amax == 0.0f, s0);
        *reinterpret_cast<uint32_t *>(dst + (size_t) row * K + e0 + 128) = q8k_pack4(y1, iscale, amax == 0.0f, s1);
        s0 = sum8_lanes(s0); s1 = sum8_lanes(s1);
        float * dd = q8k_d(dst, K, row);
        if ((lane & 7) == 0) { short * ss = reinterpret_cast<short *>(dd + (K >> 8)); ss[e0 >> 5] = (short) s0; ss[(e0 >> 5) + 4] = (short) s1; }
        if (lane == 0) dd[e0 >> 8] = (amax != 0.0f) ? 1.0f / iscale : 0.0f;
    }
}

// TMA bulk copy global -> shared, completion on an mbarrier
__device__ __forceinline__ void bulk_g2s(void * dst, const void * src, uint32_t bytes, uint64_t * bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
#define SM_MBAR (reinterpret_cast<uint64_t *>(mk_smem + MK_OFF_FLAG + 32))

struct MkEpi {
    const float * bias = nullptr, * scale = nullptr; int act = 0; const float * res = nullptr; float * out = nullptr;
    __half * kc = nullptr, * vc = nullptr; int kv_d = 0;
    uint8_t * qout = nullptr;            // PAIR epilogue: quantised rows [64][N] (+ block scales) for the next GEMV
};

// L2 prefetch of weight tiles for a later GEMV phase (tile-major: the records of a tile are contiguous); every tile once per view
__device__ __noinline__ void mk_prefetch_w(const MkView v, const QMat & W) {
    if (threadIdx.x != MK_THREADS - 32) return;
    const int n_tiles = (W.N + 15) >> 4;
    const uint32_t tile_bytes = (uint32_t) (W.K / wt_tm_rec_k(W.type)) * wt_tm_rec_bytes(W.type);
    for (int tile = v.ci; tile < n_tiles; tile += v.nc)
        l2_prefetch(reinterpret_cast<const uint8_t *>(W.base) + (size_t) tile * tile_bytes, tile_bytes);
}

#define MK_FINE(j) do { if (fb >= 0 && blockIdx.x == 0 && threadIdx.x == 0) a.trace[fb + (j)] = clock64(); } while (0)

__device__ __forceinline__ void cp_async16(uint32_t saddr, const void * g) { asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(saddr), "l"(g) : "memory"); }
__device__ __forceinline__ void cp_async16_hint(uint32_t saddr, const void * g, uint64_t pol) { asm volatile("cp.async.cg.shared.global.L2::cache_hint [%0], [%1], 16, %2;" :: "r"(saddr), "l"(g), "l"(pol) : "memory"); }
__device__ __forceinline__ uint64_t policy_evict_first() { uint64_t p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p; }
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

// The activation operand of step b, half h (batch rows 8h ..) from the staged rows: the B fragment (rows >= nt read as zero) and,
// for batch rows 2c, 2c + 1 (clamped to the last row), the Q8_0 d or Q8_1 {d, s} of the block, or the Q8_K d of the super-block and
// the sum of the sub-block (mk_store_q comment).
template <int WT>
__device__ __forceinline__ TmX mk_xfrag(int b, int h, int g, int c, int SW, int nb, int nt) {
    TmX x;
    const bool ok = h * 8 + g < nt;
    x.b0 = ok ? SM_XQ[(h * 8 + g) * SW + b * 8 + c] : 0u;
    x.b1 = ok ? SM_XQ[(h * 8 + g) * SW + b * 8 + 4 + c] : 0u;
    const int r0 = min(h * 8 + 2 * c, nt - 1), r1 = min(h * 8 + 2 * c + 1, nt - 1);
    if (mk_kq(WT)) {
        x.d0 = SM_XD[r0 * nb + (b >> 3)]; x.d1 = SM_XD[r1 * nb + (b >> 3)];
        if (wt_kq_has_dmin(WT)) {
            x.s0 = (float) reinterpret_cast<const short *>(SM_XD + r0 * nb + (nb >> 3))[b];
            x.s1 = (float) reinterpret_cast<const short *>(SM_XD + r1 * nb + (nb >> 3))[b];
        }
    } else if (mk_q1(WT)) {
        const __half2 p0 = reinterpret_cast<const __half2 *>(SM_XD)[r0 * nb + b], p1 = reinterpret_cast<const __half2 *>(SM_XD)[r1 * nb + b];
        x.d0 = __low2float(p0); x.s0 = __high2float(p0); x.d1 = __low2float(p1); x.s1 = __high2float(p1);
    } else if (WT != WT_F16) {
        x.d0 = SM_XD[r0 * nb + b]; x.d1 = SM_XD[r1 * nb + b];
    }
    return x;
}

// The rows a CTA stages for a GEMV phase.  CTA v.ci serves row group v.ci % NGc of RG rows (8 for the widest F16 matrices: what fits
// the staging area) as the ci-th of the cg CTAs of that group; nt rows in NH 8-row halves, SW words per staged row.
struct MkStage { int t_base, nt, NH, SW, ci, cg; uint32_t parity; };

template <int WT>
__device__ __forceinline__ MkStage mk_rows(const MkView v, int K) {
    const int rowb = (WT == WT_F16) ? K * 2 : K;
    const int RG = (16 * (rowb + 16) <= MK_MAXTOK * (MK_ROWB + 16)) ? 16 : 8;
    const int NGc = (v.n_tok + RG - 1) / RG, grp = v.ci % NGc;
    MkStage s;
    s.SW = (rowb >> 2) + 4; s.ci = v.ci / NGc; s.cg = (v.nc - grp + NGc - 1) / NGc;
    s.t_base = v.row0 + grp * RG; s.nt = min(RG, v.n_tok - grp * RG); s.NH = (s.nt + 7) >> 3;
    return s;
}
// stage the rows of the group: one TMA bulk copy per row (+ one for its block scales), completion on an mbarrier (phase `parity`) that
// every thread waits for on its own, after it has issued its first weight loads
template <int WT>
__device__ __forceinline__ void mk_stage(MkStage & s, const uint8_t * x, int K) {
    const int tid = threadIdx.x, nb = K >> 5;
    const int rowb = (WT == WT_F16) ? K * 2 : K;
    const int ph = SM_FLAG[4];                                   // staging round (mbarrier phase parity)
    __syncthreads();                                             // everybody has read `ph`; the previous users of the buffer are done
    s.parity = (uint32_t) ph & 1u;
    if (tid == 0) {
        SM_FLAG[4] = ph + 1;
        mbar_arrive_expect_tx(SM_MBAR, (uint32_t) s.nt * (uint32_t) (rowb + (WT == WT_F16 ? 0 : nb * 4)));
    }
    if (tid < s.nt) {
        asm volatile("fence.proxy.async;" ::: "memory");         // rows were written with ordinary stores (by other CTAs, before the grid barrier)
        bulk_g2s(SM_XQ + tid * s.SW, x + (size_t) (s.t_base + tid) * rowb, (uint32_t) rowb, SM_MBAR);
        if (WT != WT_F16)
            bulk_g2s(SM_XD + tid * nb, reinterpret_cast<const float *>(x + (size_t) MK_MAXTOK * K) + (size_t) (s.t_base + tid) * nb, (uint32_t) nb * 4, SM_MBAR);
    }
}

// k-loop of one iteration of mk_gemv for NV tile slots per warp (compile-time: predicated slots made the register allocator spill);
// leaves the split-K partials of slots j0 .. j0+NV-1 in SM_RED.  KS warps split K of a slot, UB records per slot are requested together
// (always 16 / 3: the order in which a warp adds up its blocks is part of the result, and a row must not depend on how many tiles its
// CTA happens to hold).  Four slots in one call hold 12 records + 32 accumulators per lane and spilled (7.4 us per iteration against
// 2.4 us for three slots): an iteration with four slots makes two calls of two slots, same partials, no spills.
template <int WT, int NV, int TU, int KS, int UB>
__device__ __forceinline__ void mk_gemv_kloop(const MkArgs & a, const uint8_t * wbase, int tile0, int tstep, int nrec, int nb, const MkStage s, bool & staged, int fb, int j0) {
    constexpr int RLD = 17;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, g = lane >> 2, c = lane & 3, ks = warp & (KS - 1);
    float acc[NV][2][4];
#pragma unroll
    for (int j = 0; j < NV; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) { acc[j][h][0] = acc[j][h][1] = acc[j][h][2] = acc[j][h][3] = 0.0f; }
    for (int kb = ks; kb < nrec; kb += KS * UB) {
        TmW<WT> w[NV][UB];
#pragma unroll
        for (int j = 0; j < NV; ++j) {
            const size_t r0 = (size_t) ((tile0 + ((j0 + j) / TU) * tstep) * TU + (j0 + j) % TU) * nrec;
#pragma unroll
            for (int u = 0; u < UB; ++u) w[j][u] = tm_load<WT>(wbase, r0, kb + u * KS, nrec, lane, g, c);
        }
        if (!staged) { mbar_wait(SM_MBAR, s.parity); staged = true; MK_FINE(1); }     // the rows have landed (this warp's weights are in flight)
#pragma unroll
        for (int u = 0; u < UB; ++u) {
            const int b = kb + u * KS;
            if (b < nrec) {
                TmX xf[2];
#pragma unroll
                for (int h = 0; h < 2; ++h) xf[h] = mk_xfrag<WT>(b, h, g, c, s.SW, nb, s.nt);
#pragma unroll
                for (int j = 0; j < NV; ++j) {
                    const TmA f = tm_frag<WT>(w[j][u], b, c);
#pragma unroll
                    for (int h = 0; h < 2; ++h)
                        if (h < s.NH) tm_dot<WT>(f, xf[h], acc[j][h]);
                }
            }
        }
    }
    if (!staged) { mbar_wait(SM_MBAR, s.parity); staged = true; }
    // split-K partials -> smem: red[tile slot j][warp][row][batch row]
#pragma unroll
    for (int j = 0; j < NV; ++j)
        {
#pragma unroll
            for (int h = 0; h < 2; ++h)
#pragma unroll
                for (int i = 0; i < 4; ++i) SM_RED[(((j0 + j) * MK_WARPS + warp) * 16 + g + (i >> 1) * 8) * RLD + h * 8 + 2 * c + (i & 1)] = acc[j][h][i];
        }
}

// y[t][n] = act((W[n,:] . x[t,:] + bias[n]) * scale[n]) + res[t][n].
// With up to 64 rows the activations (64 x K bytes) outweigh a weight tile (16 x K x ~0.7 bytes), so the work is cut by ROW GROUP
// first: CTA c serves the 16 rows of group c % NGc (8 rows for the widest F16 matrices), stages only those rows (one TMA bulk copy
// per row + one for its block scales) and walks the weight tiles its group-mates do not take, up to four tiles per iteration with their
// loads issued together.  The 16 warps split K of a tile; every weight block is decoded once and multiplied with both 8-row halves
// (mma.sync.m16n8k32.s8); partials are reduced through smem.  x: quantised rows in global memory (actq format).  A weight tile is
// read by the NGc CTAs of the different groups (from L2, prefetched a phase ahead).
// Latency hiding inside a phase (each phase is a chain barrier -> stage -> weights -> reduce -> epilogue of a few microseconds):
// the weight loads of the first iteration are issued BEFORE the staged rows are waited for, the epilogue's bias / scale / residual
// operands are fetched before the k-loop, tiles are dealt out evenly over the iterations and slots without a tile cost nothing.
// PAIR (FC1): tiles are dealt out in pairs = 32 consecutive output features, and the epilogue writes GELU(y) straight into the
// quantised-row format FC2 consumes (one warp = one Q8_0 block of one row) -- no f32 round trip, no extra phase.
template <int WT, bool PAIR>
__device__ __noinline__ void mk_gemv(const MkArgs & a, const MkView v, const QMat & W, const uint8_t * x, const MkEpi & e, int fb = -1) {
    constexpr int UB = 3;                                        // records whose loads are issued together
    constexpr int TP = MK_TP;                                    // tile slots per iteration
    constexpr int TU = PAIR ? 2 : 1;                             // tiles per unit of distribution
    constexpr int RLD = 17;                                      // row stride of the reduction buffer (16 batch rows + pad)
    const int N = W.N, K = W.K;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int n_tiles = (N + 15) >> 4, nrec = K / wt_tm_step_k(WT), nb = K >> 5;
    MkStage s = mk_rows<WT>(v, K);
    const int ci = s.ci, cg = s.cg, t_base = s.t_base, nt = s.nt;
    const int n_units = n_tiles / TU;                            // PAIR: N is a multiple of 32
    const int upc = ci < n_units ? (n_units - ci + cg - 1) / cg : 0;            // units of this CTA: ci, ci + cg, ...
    const int n_it = (upc * TU + TP - 1) / TP, upi = n_it ? (upc + n_it - 1) / n_it : 0;   // iterations, units per iteration (even split)
    MK_FINE(0);
    mk_stage<WT>(s, x, K);
    bool staged = false;
    for (int it = 0; it < n_it; ++it) {
        const int u0 = it * upi, nv = TU * (min(upc, u0 + upi) - u0);           // valid tile slots of this iteration (CTA-uniform)
        {
            const uint8_t * wbase = reinterpret_cast<const uint8_t *>(W.base);
            const int unit0 = ci + u0 * cg;                      // slot j holds tile (unit0 + (j / TU) * cg) * TU + j % TU
            switch (nv) {
                case 1: if (!PAIR) { mk_gemv_kloop<WT, 1, TU, 16, UB>(a, wbase, unit0, cg, nrec, nb, s, staged, fb, 0); break; }
                case 2: mk_gemv_kloop<WT, 2, TU, 16, UB>(a, wbase, unit0, cg, nrec, nb, s, staged, fb, 0); break;
                case 3:
                    if (!PAIR && (mk_kq(WT) || WT == WT_Q5_1)) {     // K-quant records carry a header share (and Q5_K fifth bits), Q5_1 ones fifth bits and minima: two slots + one
                        mk_gemv_kloop<WT, 2, TU, 16, UB>(a, wbase, unit0, cg, nrec, nb, s, staged, fb, 0);
                        mk_gemv_kloop<WT, 1, TU, 16, UB>(a, wbase, unit0, cg, nrec, nb, s, staged, fb, 2);
                        break;
                    }
                    if (!PAIR) { mk_gemv_kloop<WT, 3, TU, 16, UB>(a, wbase, unit0, cg, nrec, nb, s, staged, fb, 0); break; }
                default:                                         // four slots: two passes of two (see mk_gemv_kloop)
                    mk_gemv_kloop<WT, 2, TU, 16, UB>(a, wbase, unit0, cg, nrec, nb, s, staged, fb, 0);
                    mk_gemv_kloop<WT, 2, TU, 16, UB>(a, wbase, unit0, cg, nrec, nb, s, staged, fb, 2);
                    break;
            }
        }
        if (it == 0) MK_FINE(2);
        float pb[2], ps[2], pr[2];
        // epilogue operands of this thread's (at most two) outputs, fetched before the partials go through smem (their latency hides behind the reduction)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            int jj, tl, rl;
            if (PAIR) { const int idx = warp + MK_WARPS * i; jj = (idx >> 4) * 2 + (lane >> 4); tl = idx & 15; rl = lane & 15; }
            else      { const int o = tid + MK_THREADS * i; jj = o >> 8; tl = (o & 255) >> 4; rl = o & 15; }
            const int row = ((ci + (u0 + jj / TU) * cg) * TU + jj % TU) * 16 + rl;
            const bool ok = jj < nv && tl < nt && row < N;
            pb[i] = (ok && e.bias) ? __ldg(e.bias + row) : 0.0f;
            ps[i] = (ok && e.scale) ? __ldg(e.scale + row) : 1.0f;
            pr[i] = (ok && e.res) ? __ldcg(e.res + (size_t) (t_base + tl) * N + row) : 0.0f;
        }
        __syncthreads();
        if (it == 0) MK_FINE(3);
#pragma unroll
        for (int i = 0; i < 2; ++i) {                            // epilogue: up to TP tiles x 16 batch rows x 16 weight rows, two outputs per thread
            int jj, tl, rl;
            if (PAIR) { const int idx = warp + MK_WARPS * i; jj = (idx >> 4) * 2 + (lane >> 4); tl = idx & 15; rl = lane & 15; }
            else      { const int o = tid + MK_THREADS * i; jj = o >> 8; tl = (o & 255) >> 4; rl = o & 15; }
            const int row = ((ci + (u0 + jj / TU) * cg) * TU + jj % TU) * 16 + rl, t = t_base + tl;
            const bool ok = jj < nv && tl < nt && row < N;
            float v = 0.0f;
            if (ok) {
#pragma unroll
                for (int w = 0; w < MK_WARPS; ++w) v += SM_RED[((jj * MK_WARPS + w) * 16 + rl) * RLD + tl];
                v = (v + pb[i]) * ps[i];
                if (e.act == 1) v = gelu_ref_f16(v);
                v += pr[i];
            }
            if (PAIR) {
                // (row slot pair, token) is warp-uniform: the 32 lanes hold one Q8_0 block of the FC2 input row t (features row0 .. row0+31)
                const int idx = warp + MK_WARPS * i;
                if ((idx >> 4) * 2 < nv && tl < nt) mk_store_q<WT>(e.qout, N, t, row - lane, lane, v);
            } else if (ok) {
                if (e.out) e.out[(size_t) t * N + row] = v;
                if (e.kc && row >= e.kv_d) {
                    const size_t cell = a.cell[t];
                    if (row < 2 * e.kv_d) e.kc[cell * e.kv_d + (row - e.kv_d)] = __float2half_rn(v);
                    else                  e.vc[cell * e.kv_d + (row - 2 * e.kv_d)] = __float2half_rn(v);
                }
            }
        }
        __syncthreads();                                         // SM_RED is rewritten by the next iteration
        if (it == 0) MK_FINE(4);
    }
    if (!staged) mbar_wait(SM_MBAR, s.parity);                   // a CTA without tiles still waits for its copies before the area is reused
    MK_FINE(5);
}

// Logits (token-embedding matrix, N = n_vocab, K = d): one WARP per 16-row weight tile over the whole K -- no split-K, no reduction through
// shared memory, no CTA barrier per iteration (the split-K form needs 22 iterations of ~7 us for the 3242 tiles of large-v3: 220 us for a
// 45.6 MB stream).  A lane requests 8 records of its tile at once; the rows of the CTA's group are staged as in mk_gemv.  A row's result
// is one accumulator over the blocks in ascending order: independent of the batch.
template <int WT>
__device__ __noinline__ void mk_logits_warp(const MkArgs & a, const MkView v, const QMat & W, const uint8_t * x, float * out) {
    constexpr int UB = 8;
    const int N = W.N, K = W.K;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, c = lane & 3;
    const int n_tiles = (N + 15) >> 4, nrec = K / wt_tm_step_k(WT), nb = K >> 5;
    MkStage s = mk_rows<WT>(v, K);
    mk_stage<WT>(s, x, K);
    bool staged = false;
    const uint8_t * wbase = reinterpret_cast<const uint8_t *>(W.base);
    for (int tile = s.ci * MK_WARPS + warp; tile < n_tiles; tile += s.cg * MK_WARPS) {
        float acc[2][4];
#pragma unroll
        for (int h = 0; h < 2; ++h) { acc[h][0] = acc[h][1] = acc[h][2] = acc[h][3] = 0.0f; }
        const size_t r0 = (size_t) tile * nrec;
        for (int kb = 0; kb < nrec; kb += UB) {
            TmW<WT> w[UB];
#pragma unroll
            for (int u = 0; u < UB; ++u) w[u] = tm_load<WT>(wbase, r0, kb + u, nrec, lane, g, c);
            if (!staged) { mbar_wait(SM_MBAR, s.parity); staged = true; }
#pragma unroll
            for (int u = 0; u < UB; ++u) {
                const int b = kb + u;
                if (b < nrec) {
                    const TmA f = tm_frag<WT>(w[u], b, c);
#pragma unroll
                    for (int h = 0; h < 2; ++h)
                        if (h < s.NH) tm_dot<WT>(f, mk_xfrag<WT>(b, h, g, c, s.SW, nb, s.nt), acc[h]);
                }
            }
        }
        // C fragment: acc[h][i] = weight row g + 8*(i>>1) of the tile, batch row h*8 + 2c + (i&1)
#pragma unroll
        for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int i = 0; i < 4; ++i) {
                const int row = tile * 16 + g + (i >> 1) * 8, tl = h * 8 + 2 * c + (i & 1);
                if (tl < s.nt && row < N) out[(size_t) (s.t_base + tl) * N + row] = acc[h][i];
            }
    }
    if (!staged) mbar_wait(SM_MBAR, s.parity);
}

// ---- attention -----------------------------------------------------------------------------------------------------------
// Lane quarter r of a key owns dims {8r..8r+7} and {32+8r..32+8r+7} of the head: the 4 lanes of a key then cover 64 contiguous
// bytes per load instruction (whole 32-byte sectors; 16 dims in a row per lane would use half of every sector it touches).
// One lane owns one key per step: it holds 16 of the 64 dims of that key's K and V rows (the 4 lanes of a key share the score) and
// keeps its OWN running max / sum / output over the keys it has seen -- no cross-lane traffic per key beyond the 2-step score
// reduction.  The 8 key slots of a warp are merged once at the end (warp_merge), the warps of a CTA through shared memory.
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

// sc: score of this lane's key (already reduced over the 4 lanes of the key and scaled); masked keys must not call this
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
// merge the 8 key slots of the warp (lanes with equal lane & 3); afterwards every lane holds the warp totals of its quarter
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

// merge `nw` warp partials (m, l, o[64]) at pp; returns this thread's dimension of the merged numerator, M and L by reference
__device__ __forceinline__ float attn_merge(const float * pp, int nw, int dim, float & M, float & Lsum) {
    M = -INFINITY;
    for (int w = 0; w < nw; ++w) M = fmaxf(M, pp[w * MK_PART]);
    Lsum = 0.0f;
    float o = 0.0f;
    for (int w = 0; w < nw; ++w) {
        const float mw = pp[w * MK_PART];
        const float wgt = (mw > -INFINITY) ? __expf(mw - M) : 0.0f;
        Lsum = fmaf(pp[w * MK_PART + 1], wgt, Lsum);
        o = fmaf(pp[w * MK_PART + 4 + dim], wgt, o);
    }
    return o;
}

// The cp.async ring of the attention phases: MK_RING stages of 64 bytes per thread in the GEMV staging area (idle in these phases).  One
// stage is one key quarter of a thread, K and V ([k0 | k1 | v0 | v1], 16 bytes each, MK_THREADS * 16 bytes apart); stages are copied
// MK_RING - 1 ahead of their use.  Every thread reads back only the 64 bytes it copied itself, so the ring needs no barrier -- it is an
// asynchronous extension of the register file (96 KB in flight per SM; a 6-deep ring was measured slower for the cross stream: the 40 KB of
// L1 it takes away cost the other phases more than the tail of that phase gains).  cp.async.cg reads through L2 only: K / V rows that other
// CTAs appended in this pass are seen.
constexpr int MK_RING = 4, MK_RING_SLOT = MK_THREADS * 64, MK_OFF_QSM = MK_RING * MK_RING_SLOT;
static_assert(MK_OFF_QSM + 2 * 64 * 4 <= MK_OFF_PART, "the cp.async ring must fit below the attention partials");

__device__ __forceinline__ void cp_wait_ring() { asm volatile("cp.async.wait_group %0;" :: "n"(MK_RING - 1) : "memory"); }

// copy this thread's quarter of K / V row `off` (dims {8r..8r+7}, {32+8r..32+8r+7} of a head) into the ring stage at shared address sa;
// ef: L2 evict-first
__device__ __forceinline__ void ring_copy(uint32_t sa, const __half * k, const __half * v, size_t off, bool ef, uint64_t pol) {
    if (ef) {
        cp_async16_hint(sa, k + off, pol); cp_async16_hint(sa + MK_THREADS * 16, k + off + 32, pol);
        cp_async16_hint(sa + 2 * MK_THREADS * 16, v + off, pol); cp_async16_hint(sa + 3 * MK_THREADS * 16, v + off + 32, pol);
    } else {
        cp_async16(sa, k + off); cp_async16(sa + MK_THREADS * 16, k + off + 32);
        cp_async16(sa + 2 * MK_THREADS * 16, v + off); cp_async16(sa + 3 * MK_THREADS * 16, v + off + 32);
    }
}
__device__ __forceinline__ KV4 ring_read(unsigned stage) {
    const uint8_t * sl = mk_smem + (stage % MK_RING) * MK_RING_SLOT + threadIdx.x * 16;
    KV4 f;
    f.k0 = *reinterpret_cast<const uint4 *>(sl);                      f.k1 = *reinterpret_cast<const uint4 *>(sl + MK_THREADS * 16);
    f.v0 = *reinterpret_cast<const uint4 *>(sl + 2 * MK_THREADS * 16); f.v1 = *reinterpret_cast<const uint4 *>(sl + 3 * MK_THREADS * 16);
    return f;
}

// self-attention over the paged cache (whisper.cpp:2603-2625).  Item = (row, head), taken by a pair of warps; the 8 pairs of CTA c take
// items c*8 + pair, then + 8 nc, ...  Lane (kslot, r) of warp hw of the pair owns key quarter r of the keys 8 hw + 16 i + kslot, i = 0, 1, ..
// (step i of the warp: 8 keys), and meets them in ascending order.
// A warp's steps over all its items are ONE stream through the cp.async ring: the loader copies the K / V of a step MK_RING - 1 steps ahead
// of the arithmetic, across item boundaries, so a warp pays one memory latency per phase, not a chain of them per item.  What the loader
// needs is fetched ahead too: the cell indices of 16 steps (4 per lane: lane 8s + kslot holds those of steps 4j + s of the batch; a shuffle
// hands a step's cell to the 4 lanes of its key) for the NEXT batch while the current one is copied; the key counts of the view's rows once
// per phase (lane i holds rows row0 + i, row0 + 32 + i); the query of the next item while the current one is computed.  Only the first
// index fetch of the phase is exposed.  An item's result depends on the item alone, never on which pair, CTA or view computes it.
template <int WT>
__device__ __noinline__ void mk_attn_self(const MkArgs & a, const MkView v, const MkLayer & L) {
    constexpr int WPI = 2, NPG = MK_WARPS / WPI;                 // warps per item, warp pairs per CTA
    static_assert(MK_MAXTOK <= 64, "key counts: two rows per lane");
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, grp = warp / WPI, hw = warp % WPI;
    const int d = a.d, H = a.n_head, n_items = v.n_tok * H, pstep = v.nc * NPG;
    const int kslot = lane >> 2, r = lane & 3;
    int p = v.ci * NPG + grp;                                    // item of the arithmetic
    if (p >= n_items) return;
    const int * const idx = a.idx;
    const int ld_idx = a.ld_idx;
    // cells of steps 16b .. 16b + 15 of this warp in row t (read up to the end of the index row: the copies check the key count)
    auto fetch_cells = [&](int (&c)[4], int t, int b) {
        const int * cells = idx + (size_t) t * ld_idx;
#pragma unroll
        for (int j = 0; j < 4; ++j) { const int k = 8 * hw + 16 * (16 * b + 4 * j + (lane >> 3)) + (lane & 7); c[j] = (k < ld_idx) ? __ldg(cells + k) : 0; }
    };
    int cur[4], nxt[4];                                          // cells of the loader's batch and of the batch after it
    fetch_cells(nxt, v.row0 + p / H, 0);                         // in flight with the key counts
    const int nk_lo = lane < v.n_tok ? __ldg(a.nkv + v.row0 + lane) : 0, nk_hi = lane + 32 < v.n_tok ? __ldg(a.nkv + v.row0 + 32 + lane) : 0;
    auto n_kv = [&](int t) { const int i = t - v.row0; return __shfl_sync(0xffffffffu, i < 32 ? nk_lo : nk_hi, i & 31); };
    auto n_steps = [&](int nk) { return nk > 8 * hw ? (nk - 8 * hw + 15) >> 4 : 0; };
    auto seek = [&](int q, int & t, int & h, int & nk, int & ns) {   // the first item >= q with steps for this warp (n_items: none)
        for (; q < n_items; q += pstep) {
            t = v.row0 + q / H; h = q - (t - v.row0) * H; nk = n_kv(t); ns = n_steps(nk);
            if (ns > 0) break;
        }
        return q;
    };
    // loader: item pl (row tl, head hl, nkl keys, nsl steps), its step il; pn (tn, hn, nkn, nsn): the next item with steps
    const __half * const kc = L.kc, * const vc = L.vc;
    const bool ef = (a.prefetch & 4) != 0;
    const uint64_t pol = policy_evict_first();
    const uint32_t ring = (uint32_t) __cvta_generic_to_shared(mk_smem) + tid * 16;
    int tl = 0, hl = 0, nkl = 0, nsl = 0, tn = 0, hn = 0, nkn = 0, nsn = 0, il = 0;
    int pl = seek(p, tl, hl, nkl, nsl);
    int pn = pl < n_items ? seek(pl + pstep, tn, hn, nkn, nsn) : n_items;
    if (pl != p && pl < n_items) fetch_cells(nxt, tl, 0);
    unsigned is = 0, ic = 0;                                     // stages issued / consumed
    auto issue = [&]() {                                         // copy the loader's next step (if any) into stage is; always commits a group
        if (pl < n_items) {
            const int s = il & 15;
            if (s == 0) {                                        // a new batch: its cells were requested one batch ago
#pragma unroll
                for (int j = 0; j < 4; ++j) cur[j] = nxt[j];
                if (il + 16 < nsl) fetch_cells(nxt, tl, (il >> 4) + 1);
                else if (pn < n_items) fetch_cells(nxt, tn, 0);
            }
            const int cj = (s >> 2) == 0 ? cur[0] : (s >> 2) == 1 ? cur[1] : (s >> 2) == 2 ? cur[2] : cur[3];
            const int cell = __shfl_sync(0xffffffffu, cj, (s & 3) * 8 + kslot);
            if (8 * hw + 16 * il + kslot < nkl) ring_copy(ring + (is % MK_RING) * MK_RING_SLOT, kc, vc, (size_t) cell * d + hl * 64 + r * 8, ef, pol);
            if (++il == nsl) {
                il = 0; pl = pn; tl = tn; hl = hn; nkl = nkn; nsl = nsn;
                if (pl < n_items) pn = seek(pl + pstep, tn, hn, nkn, nsn);
            }
        }
        ++is;
        cp_commit();
    };
#pragma unroll
    for (int k = 0; k < MK_RING - 1; ++k) issue();
    const float * const qkv = a.qkv;
    int t = v.row0 + p / H, h = p - (t - v.row0) * H;
    float qlo = __ldcg(qkv + (size_t) t * 3 * d + h * 64 + lane), qhi = __ldcg(qkv + (size_t) t * 3 * d + h * 64 + 32 + lane);
    for (;;) {
        // the query rounded to f16 (ggml_flash_attn_ext converts Q to f16: ggml-cpu/ops.cpp:8560-8571): q[i] = dim 8r + i, q[8 + i] = dim 32 + 8r + i
        float q[16];
        {
            const float lo = __half2float(__float2half_rn(qlo)), hi = __half2float(__float2half_rn(qhi));
#pragma unroll
            for (int i = 0; i < 8; ++i) { q[i] = __shfl_sync(0xffffffffu, lo, 8 * r + i); q[8 + i] = __shfl_sync(0xffffffffu, hi, 8 * r + i); }
        }
        const int pq = p + pstep;                                // the next item: its query is requested now
        int tq = t, hq = h;
        if (pq < n_items) {
            tq = v.row0 + pq / H; hq = pq - (tq - v.row0) * H;
            qlo = __ldcg(qkv + (size_t) tq * 3 * d + hq * 64 + lane); qhi = __ldcg(qkv + (size_t) tq * 3 * d + hq * 64 + 32 + lane);
        }
        const int nk = n_kv(t), ns = n_steps(nk);
        LaneAcc A; lane_init(A);
        for (int i = 0; i < ns; ++i) {
            issue();
            cp_wait_ring();                                      // this thread's copies of stage ic have landed
            const KV4 f = ring_read(ic++);
            float sc = dot16(f.k0, f.k1, q);
            sc += __shfl_xor_sync(0xffffffffu, sc, 1);
            sc += __shfl_xor_sync(0xffffffffu, sc, 2);
            if (8 * hw + 16 * i + kslot < nk) lane_update(A, sc, f.v0, f.v1);
        }
        warp_merge(A);
        part_store(SM_PART + (grp * WPI + hw) * MK_PART, A, lane);
        bar_named(1 + grp, WPI * 32);
        {
            float M, Lsum;
            const float o = attn_merge(SM_PART + grp * WPI * MK_PART, WPI, hw * 32 + lane, M, Lsum);
            mk_store_q<WT>(mk_kq(WT) ? reinterpret_cast<uint8_t *>(a.q2) : a.actq, d, t, h * 64 + hw * 32, lane, (Lsum > 0.0f) ? __fdividef(o, Lsum) : 0.0f);
        }
        bar_named(1 + grp, WPI * 32);
        if (pq >= n_items) break;
        p = pq; t = tq; h = hq;
    }
    cp_wait_all();                                               // the next phase stages its rows over the ring
}

// cross-attention over the n_keys padded encoder positions, zero rows included (whisper.cpp:2688-2705).
// K and V of a window live HEAD-MAJOR in HBM ([layer][head][kv_rows][64], written that way by the cross GEMM's epilogue with kv_rows =
// the engine's largest padded context): the keys of one (row, head) pair are one contiguous 192 KB stream instead of 128-byte pieces
// 2.5 KB apart.  A reduced context reads the first n_keys rows of each head's kv_rows.
// Work unit = one (row, head) pair over ALL keys; CTA b of the view takes the contiguous range [b*P/G, (b+1)*P/G) of its P pairs.  Warp w, key slot s owns
// key 8w+s of every 128-key chunk; chunks are copied three ahead with cp.async into the ring.  The arithmetic of a pair (per-lane online
// softmax over its keys, 8 key slots merged per warp, 16 warps merged per CTA, all in fixed order) never depends on which other rows share
// the pass: a batch of 64 and a single row give bit-identical results.  (The phase is HBM-bound: a CTA with one pair more than its
// neighbour is not a cost, the others simply draw more bandwidth meanwhile.)
// Keys n_audio_ctx .. n_keys - 1 are padding: their K / V rows are zero (the cross K/V buffer is zeroed when it is allocated, and an
// encode at a reduced context zeroes the rows past it in the slots it writes; the cross GEMM's epilogue writes only the n_audio_ctx real
// rows).  They stay in the softmax with
// score 0, as in the reference, but are not read: a thread whose key is padding copies nothing and feeds zero K / V to the same arithmetic.

template <int WT>
__device__ __noinline__ void mk_attn_cross(const MkArgs & a, const MkView v, const MkLayer & L) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int d = a.d, H = a.n_head, nchp = a.n_keys / MK_XKEYS;               // chunks per pair
    const unsigned P = (unsigned) (v.n_tok * H), G = min((unsigned) v.nc, P), P0 = (unsigned) (v.row0 * H);   // pairs of the view: P0 .. P0 + P - 1
    if ((unsigned) v.ci >= G) return;
    const unsigned p0 = P0 + ((unsigned) v.ci * P) / G, p1 = P0 + (((unsigned) v.ci + 1) * P) / G;
    // loader state: chunk being fetched
    unsigned pl = p0, il = 0;
    int jl = 0, tl_ = (int) p0 / H, hl = (int) p0 - tl_ * H;
    const size_t head_stride = (size_t) a.kv_rows * 64;                                   // head h of a layer starts at h * kv_rows * 64
    const int kw = warp * 8 + (lane >> 2), n_real = a.n_audio_ctx;                        // key 8w+s of the chunk ...
    const size_t lane_off = (size_t) kw * 64 + (lane & 3) * 8;                              // ... dims {8r.., 32+8r..}
    const uint32_t ring = (uint32_t) __cvta_generic_to_shared(mk_smem) + tid * 16;
    const float kq_scale = a.kq_scale;
    // everything the copy path needs in registers (the asm statements are compiler memory barriers: values re-read from the argument
    // structs after each of them are dependent loads in front of every chunk); the slot of a row is fetched one row ahead
    const __half * const xk = L.xk, * const xv = L.xv;
    const int64_t slot_stride = a.slot_stride;
    const int * const slots = a.slot;
    const int n_tok = a.n_tok;
    const bool ef = (a.prefetch & 4) != 0;
    const uint64_t pol = policy_evict_first();
    int slot_cur = slots[tl_], slot_nxt = (tl_ + 1 < n_tok) ? slots[tl_ + 1] : 0;
    size_t pair_off = (size_t) slot_cur * slot_stride + (size_t) hl * head_stride + lane_off;
    auto issue = [&]() {                                           // copy the next chunk (if any) into ring slot il % 4; always commits a group
        if (pl < p1) {
            // L2 evict-first: 500 MB of K / V per layer would otherwise flush the prefetched weights and the activations
            if (jl * MK_XKEYS + kw < n_real) ring_copy(ring + (il % MK_RING) * MK_RING_SLOT, xk, xv, pair_off + (size_t) (jl * MK_XKEYS) * 64, ef, pol);
            if (++jl == nchp) {
                jl = 0; ++pl;
                if (++hl == H) { hl = 0; ++tl_; slot_cur = slot_nxt; slot_nxt = (tl_ + 1 < n_tok) ? slots[tl_ + 1] : 0; }
                pair_off = (size_t) slot_cur * slot_stride + (size_t) hl * head_stride + lane_off;
            }
        }
        ++il;
        cp_commit();
    };
#pragma unroll
    for (int k = 0; k < MK_RING - 1; ++k) issue();
    int t = (int) p0 / H, h = (int) p0 - t * H;
    float * qsm = reinterpret_cast<float *>(mk_smem + MK_OFF_QSM);   // f16-rounded query of the pair: [2][64]
    // qsm is stored in lane order: position 16*r + 8*hi + i holds dim 32*hi + 8*r + i
    if (warp >= 2 && warp < 4) { const int dim = (warp - 2) * 32 + lane; qsm[((dim & 31) >> 3) * 16 + (dim >> 5) * 8 + (dim & 7)] = __half2float(__float2half_rn(__ldcg(a.q2 + (size_t) t * d + h * 64 + dim))); }
    __syncthreads();
    LaneAcc A; lane_init(A);
    int buf = 0, j = 0;
    unsigned ic = 0;
    for (unsigned p = p0; p < p1; ) {
        issue();
        cp_wait_ring();                                          // this thread's copies of chunk ic have landed
        KV4 f = { make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0), make_uint4(0, 0, 0, 0) };
        if (j * MK_XKEYS + kw < n_real) f = ring_read(ic);       // padding: the zero row, not read
        ++ic;
        float sc = dot16s(f.k0, f.k1, qsm + buf * 64 + (lane & 3) * 16);
        sc += __shfl_xor_sync(0xffffffffu, sc, 1);
        sc += __shfl_xor_sync(0xffffffffu, sc, 2);
        lane_update(A, sc * kq_scale, f.v0, f.v1);
        if (++j < nchp) continue;
        j = 0;                                                   // last chunk of the pair: merge the CTA and write the row's head
        warp_merge(A);
        part_store(SM_PART + (buf * MK_WARPS + warp) * MK_PART, A, lane);
        if (p + 1 < p1 && warp >= 2 && warp < 4) {               // query of the next pair
            int tn = t, hn = h;
            if (++hn == H) { hn = 0; ++tn; }
            const int dim = (warp - 2) * 32 + lane;
            qsm[(buf ^ 1) * 64 + ((dim & 31) >> 3) * 16 + (dim >> 5) * 8 + (dim & 7)] = __half2float(__float2half_rn(__ldcg(a.q2 + (size_t) tn * d + hn * 64 + dim)));
        }
        __syncthreads();
        if (warp < 2) {                                          // merge the 16 warp partials (one output dim per thread)
            const int dim = warp * 32 + lane;
            float M, Lsum;
            const float o = attn_merge(SM_PART + buf * MK_WARPS * MK_PART, MK_WARPS, dim, M, Lsum);
            // K-quants: the f32 row goes where the Q of row t was (a.qkv, rows 3d apart): whatever phase the other partitions are in, they
            // touch their own rows only
            mk_store_q<WT>(mk_kq(WT) ? reinterpret_cast<uint8_t *>(a.qkv) : a.actq, mk_kq(WT) ? 3 * d : d, t, h * 64 + warp * 32, lane, __fdividef(o, Lsum));
        }
        buf ^= 1;
        lane_init(A);
        ++p;
        if (++h == H) { h = 0; ++t; }
    }
    cp_wait_all();
}

// DTW: copy the alignment-head slices of the cross-Q rows (complete after the barrier that ended phase 6) into the capture buffer
__device__ __noinline__ void mk_dtw_capture(const MkArgs & a, const MkView v, const MkLayer & L) {
    dtw_capture_rows(a.q2 + (size_t) v.row0 * a.d, a.d, a.cap_row + v.row0, v.n_tok, L.cap_mask, L.cap_head0, a.cap, a.cap_rows, v.ci * blockDim.x + threadIdx.x, v.nc * blockDim.x);
}

#define MK_SYNC_T(turn) do { MK_STAMP(); target += v.nc; mk_grid_sync(a, v, target, turn); MK_STAMP(); } while (0)
#define MK_SYNC() MK_SYNC_T(0)
#define MK_SYNC_Q(turn) do { target += v.nc; mk_grid_sync(a, v, target, turn); } while (0)   // without trace stamps (24 per layer for every format)

template <int WT, bool TRACE>
__global__ void __launch_bounds__(MK_THREADS, 1)
k_decode_pass(const __grid_constant__ MkArgs a) {
    if (threadIdx.x == 0) { mbar_init(SM_MBAR, 1); SM_FLAG[4] = 0; mbar_fence_init(); }
    __syncthreads();
    // this CTA's partition: the view every phase of the layer loop works in
    int part = 0;
    while (part + 1 < a.n_part && (int) blockIdx.x >= mk_partition(part + 1, a.n_part, gridDim.x, a.n_tok).c0) ++part;
    const MkPart pt = mk_partition(part, a.n_part, gridDim.x, a.n_tok);
    const MkView v = { (int) blockIdx.x - pt.c0, pt.nc, pt.row0, pt.n_tok, part };
    const MkView vg = { (int) blockIdx.x, (int) gridDim.x, 0, a.n_tok, -1 };      // the whole grid: the partitions join for the logits
    unsigned long long target = a.part_base[part];
    int n_stamp = 0;
    const int d = a.d;
    const bool pf_w = a.prefetch & 1;
    MK_STAMP();
    if (pf_w) mk_prefetch_w(v, a.layers[0].qkv);

    for (int l = 0; l < a.n_layer; ++l) {
        const MkLayer & L = a.layers[l];
        MkEpi e;
        // 1: LN -> quantised rows (whisper.cpp:2536-2543)
        mk_lnq<WT>(a, v, a.x, d, L.ln0_w, L.ln0_b, a.actq);
        if (pf_w) mk_prefetch_w(v, L.o);
        MK_SYNC();
        // 2: QKV + KV append (2545-2599)
        e = MkEpi(); e.bias = L.qkv_bias; e.scale = L.qkv_scale; e.out = a.qkv; e.kc = L.kc; e.vc = L.vc; e.kv_d = d;
        mk_gemv<WT, false>(a, v, L.qkv, a.actq, e, (TRACE && l == 1) ? 2048 + 0 : -1);
        MK_SYNC();
        // 3: self-attention (2603-2625) -> quantised rows for the O projection
        if (pf_w) mk_prefetch_w(v, L.cq);
        mk_attn_self<WT>(a, v, L);
        if (mk_kq(WT)) { MK_SYNC_Q(0); mk_q8k_rows(v, a.q2, d, d, a.actq); }     // K-quants: f32 rows -> Q8_K (timed with the attention)
        MK_SYNC();
        // 4: O + residual (2647-2659)
        if (pf_w) mk_prefetch_w(v, L.co);
        e = MkEpi(); e.bias = L.o_bias; e.res = a.x; e.out = a.x;
        mk_gemv<WT, false>(a, v, L.o, a.actq, e, (TRACE && l == 1) ? 2048 + 8 : -1);
        MK_SYNC();
        // 5: LN -> quantised rows
        mk_lnq<WT>(a, v, a.x, d, L.lnc_w, L.lnc_b, a.actq);
        if (pf_w) mk_prefetch_w(v, L.fc1);
        MK_SYNC();
        // 6: cross Q (2661-2681)
        e = MkEpi(); e.bias = L.cq_bias; e.out = a.q2;
        mk_gemv<WT, false>(a, v, L.cq, a.actq, e, (TRACE && l == 1) ? 2048 + 16 : -1);
        MK_SYNC_T(1);                                            // the partition takes its turn to stream K/V ...
        // 7: cross-attention (2688-2705); DTW passes first keep the alignment-head queries of their flagged rows
        if (pf_w) mk_prefetch_w(v, L.fc2);
        if (a.cap != nullptr && L.cap_mask != 0u) mk_dtw_capture(a, v, L);
        mk_attn_cross<WT>(a, v, L);
        if (mk_kq(WT)) { MK_SYNC_Q(2); mk_q8k_rows(v, a.qkv, 3 * d, d, a.actq); }   // ... and gives it back at the first barrier behind the stream
        MK_SYNC_T(mk_kq(WT) ? 0 : 2);
        // 8: cross O + residual (2754-2766)
        e = MkEpi(); e.bias = L.co_bias; e.res = a.x; e.out = a.x;
        mk_gemv<WT, false>(a, v, L.co, a.actq, e, (TRACE && l == 1) ? 2048 + 24 : -1);
        MK_SYNC();
        // 9: LN -> quantised rows
        mk_lnq<WT>(a, v, a.x, d, L.lnm_w, L.lnm_b, a.actq);
        if (pf_w) { if (l + 1 < a.n_layer) mk_prefetch_w(v, a.layers[l + 1].qkv); else if (a.want_logits) mk_prefetch_w(vg, a.te); }
        MK_SYNC();
        // 10: FC1 + GELU (2770-2794), then the rows are quantised for FC2
        if (mk_kq(WT)) {                                         // K-quants: f32 GELU rows, then a Q8_K phase (trace slot "10b h->q8")
            e = MkEpi(); e.bias = L.fc1_bias; e.act = 1; e.out = a.h;
            mk_gemv<WT, false>(a, v, L.fc1, a.actq, e, (TRACE && l == 1) ? 2048 + 32 : -1);
            MK_STAMP(); MK_SYNC_Q(0); MK_STAMP();
            mk_q8k_rows(v, a.h, 4 * d, 4 * d, a.hq);
        } else {
            e = MkEpi(); e.bias = L.fc1_bias; e.act = 1; e.qout = a.hq;
            mk_gemv<WT, true>(a, v, L.fc1, a.actq, e, (TRACE && l == 1) ? 2048 + 32 : -1);
            MK_STAMP(); MK_STAMP();                              // (trace slot of the former FC1 -> Q8_0 phase)
        }
        MK_SYNC();
        // 11: FC2 + residual (2797-2806)
        e = MkEpi(); e.bias = L.fc2_bias; e.res = a.x; e.out = a.x;
        mk_gemv<WT, false>(a, v, L.fc2, a.hq, e, (TRACE && l == 1) ? 2048 + 40 : -1);
        MK_SYNC();
    }
    if (a.want_logits) {                                         // final LN + logits (2811-2827)
        mk_lnq<WT>(a, v, a.x, d, a.lnf_w, a.lnf_b, a.actq);
        MK_STAMP(); mk_grid_sync(a, vg, a.bar_base + gridDim.x, 0); MK_STAMP();
        if (a.prefetch & 16) mk_logits_warp<WT>(a, vg, a.te, a.actq, a.logits);
        else { MkEpi e; e.out = a.logits; mk_gemv<WT, false>(a, vg, a.te, a.actq, e); }
        MK_STAMP();
    }
}

// Test probe: one phase, set up as k_decode_pass sets up its CTAs, on a view the caller chooses; no barrier, so an ordinary launch.
template <int WT, int PHASE>
__global__ void __launch_bounds__(MK_THREADS, 1)
k_mk_probe(const __grid_constant__ MkArgs a, const __grid_constant__ MkProbe p) {
    if (threadIdx.x == 0) { mbar_init(SM_MBAR, 1); SM_FLAG[4] = 0; mbar_fence_init(); }
    __syncthreads();
    const MkView v = { (int) blockIdx.x, (int) gridDim.x, p.row0, p.n_tok, 0 };
    if constexpr (PHASE == MKP_LNQ) mk_lnq<WT>(a, v, p.src, p.K, p.scale, p.bias, p.dst);
    else if constexpr (PHASE == MKP_Q8K) mk_q8k_rows(v, p.src, p.lds, p.K, p.dst);
    else if constexpr (PHASE == MKP_GEMV) {
        MkEpi e;
        e.bias = p.bias; e.scale = p.scale; e.act = p.act; e.res = p.res; e.out = p.out; e.kc = p.kc; e.vc = p.vc; e.kv_d = p.kv_d;
        mk_gemv<WT, false>(a, v, p.W, p.x, e);
    } else if constexpr (PHASE == MKP_GEMV_PAIR) {               // as the pass's FC1 call: epilogue bias + GELU -> rows, matrix in global memory
        MkEpi e;
        e.bias = p.bias; e.act = 1; e.qout = p.dst;
        mk_gemv<WT, true>(a, v, *p.Wg, p.x, e);
    }
    else if constexpr (PHASE == MKP_LOGITS_WARP) mk_logits_warp<WT>(a, v, p.W, p.x, p.out);
    else if constexpr (PHASE == MKP_ATTN_SELF) mk_attn_self<WT>(a, v, *p.L);
    else mk_attn_cross<WT>(a, v, *p.L);
}

template <int WT, int PHASE>
static bool mk_probe_t(const MkArgs & a, const MkProbe & p, int n_cta, cudaStream_t st) {
    if (ensure_dyn_smem(reinterpret_cast<const void *>(k_mk_probe<WT, PHASE>), MK_SMEM) != cudaSuccess) {
        set_error("decode kernel probe: cannot raise the shared-memory limit"); return false;
    }
    k_mk_probe<WT, PHASE><<<n_cta, MK_THREADS, MK_SMEM, st>>>(a, p);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { set_error("decode kernel probe launch: %s", cudaGetErrorString(e)); return false; }
    return true;
}

template <int WT>
static bool mk_probe_w(const MkArgs & a, const MkProbe & p, int n_cta, cudaStream_t st) {
    switch (p.phase) {
        case MKP_LNQ:         return mk_probe_t<WT, MKP_LNQ>(a, p, n_cta, st);
        case MKP_Q8K:         if constexpr (!mk_kq(WT)) break; else return mk_probe_t<WT, MKP_Q8K>(a, p, n_cta, st);
        case MKP_GEMV:        return mk_probe_t<WT, MKP_GEMV>(a, p, n_cta, st);
        case MKP_GEMV_PAIR:   if constexpr (mk_kq(WT)) break; else return mk_probe_t<WT, MKP_GEMV_PAIR>(a, p, n_cta, st);   // K-quants: FC1 writes f32 rows
        case MKP_LOGITS_WARP: return mk_probe_t<WT, MKP_LOGITS_WARP>(a, p, n_cta, st);
        case MKP_ATTN_SELF:   return mk_probe_t<WT, MKP_ATTN_SELF>(a, p, n_cta, st);
        case MKP_ATTN_CROSS:  return mk_probe_t<WT, MKP_ATTN_CROSS>(a, p, n_cta, st);
    }
    set_error("decode kernel probe: phase %d does not exist for weight type %d", p.phase, WT);
    return false;
}

bool mk_probe_launch(const MkArgs & a, const MkProbe & p, int wtype, int n_cta, cudaStream_t st) {
    if (n_cta < 1 || p.row0 < 0 || p.n_tok < 1 || p.row0 + p.n_tok > MK_MAXTOK) { set_error("decode kernel probe: bad view"); return false; }
    switch (wtype) {
        case WT_F16:  return mk_probe_w<WT_F16>(a, p, n_cta, st);
        case WT_Q4_0: return mk_probe_w<WT_Q4_0>(a, p, n_cta, st);
        case WT_Q5_0: return mk_probe_w<WT_Q5_0>(a, p, n_cta, st);
        case WT_Q4_1: return mk_probe_w<WT_Q4_1>(a, p, n_cta, st);
        case WT_Q5_1: return mk_probe_w<WT_Q5_1>(a, p, n_cta, st);
        case WT_Q8_0: return mk_probe_w<WT_Q8_0>(a, p, n_cta, st);
        case WT_Q4_K: return mk_probe_w<WT_Q4_K>(a, p, n_cta, st);
        case WT_Q5_K: return mk_probe_w<WT_Q5_K>(a, p, n_cta, st);
        case WT_Q3_K: return mk_probe_w<WT_Q3_K>(a, p, n_cta, st);
        default: set_error("decode kernel probe: unsupported weight type %d", wtype); return false;
    }
}

bool mk_cross_head_major() {
    return true;
}
int mk_layer_barriers(int wtype) { return wt_is_kquant(wtype) ? 14 : 11; }
size_t mk_bar_words(int n_sm) { return 16 + 16 * (size_t) n_sm + 16 * (MK_MAX_PARTS + 1); }
bool mk_supported(int wtype) { return wtype == WT_F16 || wt_is_block32(wtype) || wt_is_kquant(wtype); }
size_t mk_smem_bytes(int, int) { return MK_SMEM; }
int mk_max_rows() { return MK_MAXTOK; }

template <int WT, bool TRACE>
static bool mk_launch_t(const MkArgs & a, int n_sm, cudaStream_t st) {
    const size_t smem = mk_smem_bytes(WT, a.d);
    if (ensure_dyn_smem(reinterpret_cast<const void *>(k_decode_pass<WT, TRACE>), 227 * 1024) != cudaSuccess) {
        set_error("decode megakernel: cannot raise the shared-memory limit"); return false;
    }
    if (smem > 227 * 1024) { set_error("decode megakernel: %zu bytes of shared memory needed", smem); return false; }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(n_sm); cfg.blockDim = dim3(MK_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeCooperative; at[0].val.cooperative = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    const cudaError_t e = cudaLaunchKernelEx(&cfg, k_decode_pass<WT, TRACE>, a);
    if (e != cudaSuccess) { set_error("decode megakernel launch: %s", cudaGetErrorString(e)); return false; }
    count_launch();
    return true;
}

bool mk_launch(const MkArgs & a, int wtype, int n_sm, cudaStream_t st) {
    if (a.te.layout != 1) { set_error("decode megakernel: weights are not in the tile-major layout"); return false; }
#define WB_MK(T) (a.trace ? mk_launch_t<T, true>(a, n_sm, st) : mk_launch_t<T, false>(a, n_sm, st))
    switch (wtype) {
        case WT_F16:  return WB_MK(WT_F16);
        case WT_Q4_0: return WB_MK(WT_Q4_0);
        case WT_Q5_0: return WB_MK(WT_Q5_0);
        case WT_Q4_1: return WB_MK(WT_Q4_1);
        case WT_Q5_1: return WB_MK(WT_Q5_1);
        case WT_Q8_0: return WB_MK(WT_Q8_0);
        case WT_Q4_K: return WB_MK(WT_Q4_K);
        case WT_Q5_K: return WB_MK(WT_Q5_K);
        case WT_Q3_K: return WB_MK(WT_Q3_K);
        default: set_error("decode megakernel: unsupported weight type %d", wtype); return false;
    }
#undef WB_MK
}

} // namespace wb
