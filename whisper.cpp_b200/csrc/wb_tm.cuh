// wb_tm.cuh -- the decode kernel's reader of tile-major weight records (layout: wb_quant.cuh), one per format.
// A lane's share of one MMA step (32 values; F16: 16) is fetched by tm_load into a TmW<WT> that holds only the registers of its
// format, turned into the A fragment and row scales by tm_frag, and multiplied into one 8-row half of the accumulators by tm_dot.
// Loading is a call of its own: the GEMV phases issue the loads of several steps and tiles before the first one is used.
#pragma once
#include <type_traits>
#include "wb_quant.cuh"
#include "wb_dev.cuh"

namespace wb {

struct TmNone {};
// qs words | fifth-bit words (Q3_K: hm) | scales: f16 d of rows g, g + 8 (Q4_0 / Q5_0 / Q8_0), {d, m} (Q4_1 / Q5_1), the lane's 8
// header bytes (Q4_K / Q5_K), {scale word, d word} (Q3_K)
template <int WT> struct TmW {
    std::conditional_t<WT == WT_F16 || WT == WT_Q8_0, uint4, std::conditional_t<WT == WT_Q3_K, uint32_t, uint2>> q;
    std::conditional_t<wt_has_qh(WT) || WT == WT_Q5_K || WT == WT_Q3_K, uint2, TmNone> h;
    std::conditional_t<WT == WT_F16, TmNone, std::conditional_t<wt_is_block32(WT) && !wt_has_min(WT), uint32_t, uint2>> s;
};

// step b (clamped to the last one: a lane may request past the end of K) of the tile whose steps start at step r0 = tile * nrec.
// The address is one step index times the step size: with a tile pointer and an offset the optimiser kept one 64-bit value per tile
// and record part live across the k-loop, and the GEMV phases spilled.
template <int WT>
__device__ __forceinline__ TmW<WT> tm_load(const uint8_t * wbase, size_t r0, int b, int nrec, int lane, int g, int c) {
    constexpr int STEP = wt_tm_step_bytes(WT);
    TmW<WT> w;
    b = min(b, nrec - 1);
    const uint8_t * const hdr = wbase + (r0 + (b & ~7)) * STEP;                     // K-quants: the super-block's record
    const uint8_t * const rec = wt_is_kquant(WT) ? hdr + wt_tm_sub_off(WT, b & 7) : wbase + (r0 + b) * STEP;
    w.q = __ldg(reinterpret_cast<const decltype(w.q) *>(rec) + lane);
    if constexpr (!std::is_same_v<decltype(w.h), TmNone>) w.h = __ldg(reinterpret_cast<const uint2 *>(rec + wt_tm_qs_bytes(WT)) + g);
    if constexpr (WT == WT_Q3_K)
        w.s = make_uint2(__ldg(reinterpret_cast<const uint32_t *>(hdr) + (b & 7) * 8 + g), __ldg(reinterpret_cast<const uint32_t *>(hdr + WT_TM_Q3K_D_OFF) + g));
    else if constexpr (wt_is_kquant(WT))
        w.s = __ldg(reinterpret_cast<const uint2 *>(hdr + WT_TM_KQ_HDR_ROW * (g + 8 * (c >> 1))) + (c & 1));
    else if constexpr (WT != WT_F16)
        w.s = __ldg(reinterpret_cast<const decltype(w.s) *>(rec + wt_tm_d_off(WT)) + g);
    return w;
}

// A fragment of lane 4g + c (signed int8, F16: halves) and the scales of rows g, g + 8: d0 / d1 = d (K-quants with a minimum: d sc_j),
// m0 / m1 = m (dmin m_j), sc = the Q3_K scale word
struct TmA { uint32_t a[4]; float d0, d1, m0, m1; uint32_t sc; };

__device__ __forceinline__ float tm_half(uint32_t w, int hi) { return __half2float(__ushort_as_half((unsigned short) (hi ? (w >> 16) : (w & 0xffffu)))); }

template <int WT>
__device__ __forceinline__ TmA tm_frag(const TmW<WT> & w, int b, int c) {
    TmA f;
    if constexpr (WT == WT_F16 || WT == WT_Q8_0) {
        f.a[0] = w.q.x; f.a[1] = w.q.y; f.a[2] = w.q.z; f.a[3] = w.q.w;
    } else if constexpr (WT == WT_Q3_K) {
        q3k_tm_af(w.q, w.h, c, f.a);
    } else {                                                     // nibbles (+ fifth bits) in the Q4_0 order
        f.a[0] = w.q.x & 0x0F0F0F0Fu; f.a[2] = (w.q.x >> 4) & 0x0F0F0F0Fu;
        f.a[1] = w.q.y & 0x0F0F0F0Fu; f.a[3] = (w.q.y >> 4) & 0x0F0F0F0Fu;
        if constexpr (!std::is_same_v<decltype(w.h), TmNone>) {
            f.a[0] |= spread4_to_bit4(w.h.x >> (4 * c)); f.a[2] |= spread4_to_bit4(w.h.x >> (16 + 4 * c));
            f.a[1] |= spread4_to_bit4(w.h.y >> (4 * c)); f.a[3] |= spread4_to_bit4(w.h.y >> (16 + 4 * c));
        }
        if constexpr (WT == WT_Q4_0 || WT == WT_Q5_0) {
            const uint32_t off = WT == WT_Q5_0 ? 0x10101010u : 0x08080808u;
#pragma unroll
            for (int r = 0; r < 4; ++r) f.a[r] = __vsub4(f.a[r], off);
        }
    }
    if constexpr (WT == WT_Q3_K) { f.sc = w.s.x; f.d0 = tm_half(w.s.y, 0); f.d1 = tm_half(w.s.y, 1); }
    else if constexpr (wt_is_kquant(WT)) kq_tm_scales(w.s, b & 7, c, f.d0, f.m0, f.d1, f.m1);
    else if constexpr (wt_has_min(WT)) { f.d0 = tm_half(w.s.x, 0); f.d1 = tm_half(w.s.x, 1); f.m0 = tm_half(w.s.y, 0); f.m1 = tm_half(w.s.y, 1); }
    else if constexpr (WT != WT_F16) { f.d0 = tm_half(w.s, 0); f.d1 = tm_half(w.s, 1); }
    return f;
}

// B fragment of one 8-row half of the activations (b0 / b1: values 4c .., 16 + 4c .. of batch row g) and the Q8 operands of batch
// rows 2c, 2c + 1: d0 / d1 = d, s0 / s1 = s (Q8_1) or the sub-block sum (Q8_K)
struct TmX { uint32_t b0, b1; float d0, d1, s0, s1; };

// acc[i] (weight row g + 8 (i >> 1), batch row 2c + (i & 1)) += the step's block dot, accumulated as the reference's vec_dot does
template <int WT>
__device__ __forceinline__ void tm_dot(const TmA & f, const TmX & x, float (&acc)[4]) {
    if constexpr (WT == WT_F16) {
        mma_f16_16816(acc, f.a, x.b0, x.b1);
    } else {
        int dd[4];
        if constexpr (WT == WT_Q3_K) q3k_sumi(f.a, x.b0, x.b1, f.sc, dd);
        else mma_s8_16832(dd, f.a, x.b0, x.b1);
        if constexpr (wt_kq_has_dmin(WT)) {                      // d_x (d sc_j sumi - dmin m_j sumx)
            acc[0] = fmaf(x.d0, fmaf(f.d0, (float) dd[0], -f.m0 * x.s0), acc[0]);
            acc[1] = fmaf(x.d1, fmaf(f.d0, (float) dd[1], -f.m0 * x.s1), acc[1]);
            acc[2] = fmaf(x.d0, fmaf(f.d1, (float) dd[2], -f.m1 * x.s0), acc[2]);
            acc[3] = fmaf(x.d1, fmaf(f.d1, (float) dd[3], -f.m1 * x.s1), acc[3]);
        } else if constexpr (wt_has_min(WT)) {                   // (d_w d_x) sumi, then m_w s_x
            acc[0] = fmaf(f.m0, x.s0, fmaf(f.d0 * x.d0, (float) dd[0], acc[0]));
            acc[1] = fmaf(f.m0, x.s1, fmaf(f.d0 * x.d1, (float) dd[1], acc[1]));
            acc[2] = fmaf(f.m1, x.s0, fmaf(f.d1 * x.d0, (float) dd[2], acc[2]));
            acc[3] = fmaf(f.m1, x.s1, fmaf(f.d1 * x.d1, (float) dd[3], acc[3]));
        } else {                                                 // (d_w d_x) sumi (Q3_K: sumi over the scaled 16-value halves)
            acc[0] = fmaf(f.d0 * x.d0, (float) dd[0], acc[0]);
            acc[1] = fmaf(f.d0 * x.d1, (float) dd[1], acc[1]);
            acc[2] = fmaf(f.d1 * x.d0, (float) dd[2], acc[2]);
            acc[3] = fmaf(f.d1 * x.d1, (float) dd[3], acc[3]);
        }
    }
}

} // namespace wb
