// wb_quant.cuh -- weight formats as they live in HBM, and the device-side decoders.
//
// File side (unchanged legacy ggml container): 32-value blocks block_q4_0 / block_q4_1 / block_q5_0 / block_q5_1 / block_q8_0
// (ggml/src/ggml-common.h:194-256) and 256-value super-blocks block_q4_K / block_q5_K
// (ggml-common.h:327-356) and block_q3_K (ggml-common.h:310-325).  Bit-level meaning follows
// ggml/src/ggml-quants.c:459-567 (dequantize_row_q4_0, _q5_0, _q8_0), :880-887 (get_scale_min_k4), :1529-1551 (q4_K),
// :1731-1756 (q5_K), :1305-1353 (q3_K).
//
// HBM side ("planar" layout, built once at load by wb_repack_*): the 18/22/34-byte file blocks are not
// 16-byte aligned, so every 32-block matrix [N rows][K] is split into three dense arrays
//     qs : [N][K/32][QS]   QS = 16 bytes (4/5-bit) or 32 bytes (8-bit)   -> one or two 128-bit loads per block
//     qh : [N][K/32]       uint32, the fifth bits (Q5_0 / Q5_1)
//     d  : [N][K/32]       f16 block scale
//     m  : [N][K/32]       f16 block minimum (Q4_1 / Q5_1: value = q * d + m, q unsigned)
// Total bytes are identical to the file (18 / 20 / 22 / 24 / 34 per 32 weights).  K-quant super-blocks (144 / 176 / 110 bytes) are kept verbatim (encoder side; the decoder matrices use the tile-major records below).
#pragma once
#include <cstdint>
#include <cuda_fp16.h>

namespace wb {

// numeric ids are ggml_type (ggml/include/ggml.h:390-405)
enum WType : int { WT_F32 = 0, WT_F16 = 1, WT_Q4_0 = 2, WT_Q4_1 = 3, WT_Q5_0 = 6, WT_Q5_1 = 7, WT_Q8_0 = 8, WT_Q3_K = 11, WT_Q4_K = 12, WT_Q5_K = 13 };

struct QMat {            // one weight matrix resident in HBM
    int   type = WT_F16;
    int   N = 0, K = 0;  // rows (output features), contraction length
    const void * base = nullptr; // F16: half[N][K];  K-quants: super-blocks [N][K/256]
    const uint8_t  * qs = nullptr;
    const uint32_t * qh = nullptr;
    const __half   * d  = nullptr;
    const __half   * m  = nullptr;   // Q4_1 / Q5_1 planar: block minima
    int   layout = 0;    // 0: rows (F16) / planar (32-blocks) / verbatim (K-quants); 1: tile-major records at `base` (see below)
    const __half * f16 = nullptr;  // encoder-side matrices of quantised models: f16 expansion [N][K] made once at load (TMA operand of the
                                   // persistent GEMM; each value is the f16 rounding of the exact d * (q - off)); nullptr = expand per launch
};

__host__ __device__ inline int wt_qs_bytes(int t)    { return t == WT_Q8_0 ? 32 : 16; }
__host__ __device__ constexpr bool wt_is_block32(int t) { return t == WT_Q4_0 || t == WT_Q5_0 || t == WT_Q8_0 || t == WT_Q4_1 || t == WT_Q5_1; }
__host__ __device__ constexpr bool wt_has_min(int t)    { return t == WT_Q4_1 || t == WT_Q5_1; }     // blocks with a minimum: Q8_1 activations
__host__ __device__ constexpr bool wt_has_qh(int t)     { return t == WT_Q5_0 || t == WT_Q5_1; }
// K-quants: 256-value super-blocks, Q8_K activations.  Q4_K / Q5_K have a minimum term (dmin * m against the activation sums),
// Q3_K is signed with one integer scale per 16 values
__host__ __device__ constexpr bool wt_is_kquant(int t)  { return t == WT_Q4_K || t == WT_Q5_K || t == WT_Q3_K; }
__host__ __device__ constexpr bool wt_kq_has_dmin(int t) { return t == WT_Q4_K || t == WT_Q5_K; }
__host__ __device__ inline int  wt_kq_block_bytes(int t) { return t == WT_Q4_K ? 144 : t == WT_Q5_K ? 176 : t == WT_Q3_K ? 110 : 0; }

// "Tile-major" layout of the decoder matrices (persistent decode kernel, wb_decode_mk.cu).  The matrix is cut into tiles of
// 16 output rows; for every tile and every 32-value block (F16: every 16 values) there is ONE contiguous record holding the
// operands in the register order of the warp-level MMA (lane = 4*g + c reads rows g and g+8 of the tile):
//   Q4_0 (288 B): u32 qs[32 lanes][2] = { word c of row g, word c of row g+8 }            | f16 d[8][2]  = { row g, row g+8 }
//   Q5_0 (352 B): qs as Q4_0 (256 B) | u32 qh[8][2] = { row g, row g+8 } (64 B)            | f16 d[8][2]
//   Q4_1 (320 B): qs as Q4_0, unsigned nibbles (256 B)                                     | u32 dm[8][2] = { d_g | d_g+8 << 16, m_g | m_g+8 << 16 }
//   Q5_1 (384 B): qs as Q4_1 (256 B) | qh as Q5_0 (64 B)                                   | dm as Q4_1
//   (one 8-byte load gives lane 4g + c the scales and minima of both its rows)
//   Q8_0 (544 B): u32 qs[32 lanes][4] = { w c / row g, w c / row g+8, w 4+c / row g, w 4+c / row g+8 } | f16 d[8][2]
//   F16  (512 B per 16 values): u32 a[32 lanes][4] = the m16n8k16 A fragment
// so one warp fetches a record with three fully coalesced loads.  Same bytes per weight as the file; rows >= N are zero.
// K-quants: one record per (tile, 256-value super-block), the 16 rows' super-blocks regrouped:
//   Q4_K (2304 B): u8 hdr[16 rows][16] (the file's d, dmin, scales[12] of each row)   | 8 x sub-block record (256 B):
//                  u32 qs[32 lanes][2] in the Q4_0 order, unsigned nibbles (byte i of a row's 16 = q[i] | q[i+16] << 4)
//   Q5_K (2816 B): hdr as Q4_K | 8 x sub-block record (320 B): qs as Q4_K | u32 qh[8][2] = { row g, row g+8 } (bit i = fifth bit of q[i])
// = the file's 16 x 144 / 16 x 176 bytes.  The GEMV splits K per 32-value sub-block (record + 256 + j * 256 / 320); a lane reads 8 bytes
// of the header: lane 4g + c gets bytes 8 (c & 1) .. +7 of row g + 8 (c >> 1), so a quad holds the 32 header bytes of its two rows.
// Q3_K (signed values, one integer scale per 16 values, no minimum): one 1824-byte record = a 288-byte header
//   i8 sc[8 sub-blocks][8 lane groups][4] = { row g: scale of values 0..15, of 16..31; row g + 8: the same }   (256 B; the packed
//   6-bit scales unpacked to sc - 32 at repack time) | u32 d[8] = { d_g | d_g+8 << 16 }   (32 B)
// so lane 4g + c finds the four scales of its rows for sub-block j in the word j * 8 + g, and their two d in the word 64 + g; then
// 8 x sub-block record (192 B): u32 ql[32 lanes]: byte e holds at bits 2r, 2r + 1 the low bit pair of byte e of the lane's A register r
//   (128 B) | u32 hm[8][2] = { row g, row g+8 } (bit i = hmask bit of q[i], the Q5_K arrangement) (64 B)
// = 16 x 114 bytes, 3.6 % above the file's 110 (the unpacked scales).
// (A register r of lane 4g + c: r = 0 / 1 rows g / g + 8 values 4c .. 4c + 3, r = 2 / 3 the same rows, values 16 + 4c .. 16 + 4c + 3.)
// These accessors are the only place the sizes and offsets are written down: the repack writers (wb_kernels.cu), the element reader
// dequant_elem_tm and the decode kernel's record reader (wb_tm.cuh) take them from here.
__host__ __device__ constexpr int wt_tm_rec_bytes(int t) {
    return t == WT_Q4_0 ? 288 : t == WT_Q5_0 ? 352 : t == WT_Q4_1 ? 320 : t == WT_Q5_1 ? 384 : t == WT_Q8_0 ? 544 : t == WT_F16 ? 512 : t == WT_Q4_K ? 2304 : t == WT_Q5_K ? 2816 :
           t == WT_Q3_K ? 1824 : 0;
}
__host__ __device__ constexpr int wt_tm_rec_k(int t)     { return t == WT_F16 ? 16 : wt_is_kquant(t) ? 256 : 32; }
// one MMA step: the K values a warp multiplies per record (K-quants: per sub-block record), and the record bytes per step
__host__ __device__ constexpr int wt_tm_step_k(int t)     { return t == WT_F16 ? 16 : 32; }
__host__ __device__ constexpr int wt_tm_step_bytes(int t) { return wt_tm_rec_bytes(t) / (wt_tm_rec_k(t) / wt_tm_step_k(t)); }
// inside a record (K-quants: inside a sub-block record): the qs words (Q3_K: ql), then the fifth-bit words (Q3_K: hm), then the
// 32-block types' f16 d[8][2] or {d, m} words
__host__ __device__ constexpr int wt_tm_qs_bytes(int t)   { return t == WT_Q8_0 ? 512 : t == WT_Q3_K ? 128 : 256; }
__host__ __device__ constexpr int wt_tm_d_off(int t)      { return wt_tm_qs_bytes(t) + (wt_has_qh(t) ? 64 : 0); }
// K-quants: the header (Q4_K / Q5_K: 16 bytes per row; Q3_K: the scale words, then u32 d[8] at WT_TM_Q3K_D_OFF), then the
// 32-value sub-block records
constexpr int WT_TM_KQ_HDR_ROW = 16, WT_TM_Q3K_D_OFF = 256;
__host__ __device__ constexpr int wt_tm_hdr_bytes(int t) { return t == WT_Q3_K ? WT_TM_Q3K_D_OFF + 32 : 16 * WT_TM_KQ_HDR_ROW; }
__host__ __device__ constexpr int wt_tm_sub_bytes(int t) { return t == WT_Q4_K ? 256 : t == WT_Q5_K ? 320 : t == WT_Q3_K ? 192 : 0; }
__host__ __device__ constexpr int wt_tm_sub_off(int t, int j) { return wt_tm_hdr_bytes(t) + j * wt_tm_sub_bytes(t); }
__host__ __device__ inline size_t wt_tm_bytes(int t, int N, int K) { return (size_t) ((N + 15) / 16) * (K / wt_tm_rec_k(t)) * wt_tm_rec_bytes(t); }
static_assert(wt_tm_step_bytes(WT_Q4_K) == 288 && wt_tm_step_bytes(WT_Q5_K) == 352 && wt_tm_step_bytes(WT_Q3_K) == 228, "K-quant records");
static_assert(wt_tm_sub_off(WT_Q5_K, 8) == wt_tm_rec_bytes(WT_Q5_K) && wt_tm_sub_off(WT_Q3_K, 8) == wt_tm_rec_bytes(WT_Q3_K), "K-quant records");
static_assert(wt_tm_d_off(WT_Q5_1) + 64 == wt_tm_rec_bytes(WT_Q5_1) && wt_tm_d_off(WT_Q8_0) + 32 == wt_tm_rec_bytes(WT_Q8_0), "32-block records");
// bytes per weight on disk and in HBM
__host__ __device__ inline double wt_bpw(int t) {
    switch (t) { case WT_F32: return 4; case WT_F16: return 2; case WT_Q4_0: return 18.0/32; case WT_Q5_0: return 22.0/32;
                 case WT_Q4_1: return 20.0/32; case WT_Q5_1: return 24.0/32;
                 case WT_Q8_0: return 34.0/32; case WT_Q4_K: return 144.0/256; case WT_Q5_K: return 176.0/256;
                 case WT_Q3_K: return 110.0/256; }
    return 0;
}

#ifdef __CUDACC__

// ---- helpers ------------------------------------------------------------------------------------
// spread the low 4 bits of q to bit 4 of each byte of a word: bit i -> byte i
__device__ __forceinline__ uint32_t spread4_to_bit4(uint32_t q) {
    return (((q & 0xFu) * 0x00204081u) & 0x01010101u) << 4;
}
// 4 unsigned bytes -> two half2 holding (1024 + b) exactly (0x6400 | b); (v - (1024+off)) is exact in f16, and the
// single multiply by d rounds once: the result is the f16 rounding of the exact value d*(q - off).
// (A fused fma(v, d, -(1024+off)*d) would round the constant term and lose up to d/4 -- not used.)
__device__ __forceinline__ void bytes4_to_half2x2(uint32_t b, __half2 dd, __half2 off, uint32_t & lo, uint32_t & hi) {
    const uint32_t p0 = __byte_perm(b, 0x64646464u, 0x4140); // {b0, 0x64, b1, 0x64}
    const uint32_t p1 = __byte_perm(b, 0x64646464u, 0x4342); // {b2, 0x64, b3, 0x64}
    const __half2 h0 = __hmul2(__hsub2(*reinterpret_cast<const __half2 *>(&p0), off), dd);
    const __half2 h1 = __hmul2(__hsub2(*reinterpret_cast<const __half2 *>(&p1), off), dd);
    lo = *reinterpret_cast<const uint32_t *>(&h0);
    hi = *reinterpret_cast<const uint32_t *>(&h1);
}

// ---- decode one 32-block into 32 halves (out[0..3] = 4 x 16 bytes, element order 0..31) ---------
// Rounding: each output is the f16 rounding of the exact product d*(q - off), i.e. exactly what the reference's
// dequantize_row_* (f32, exact) gives after one f16 store.
__device__ __forceinline__ void dequant_q4_0(const uint4 qs, const __half d, uint4 (&out)[4]) {
    const __half2 dd = __half2half2(d);
    const __half2 no = __float2half2_rn(1032.0f);               // 1024 + 8
    const uint32_t w[4] = { qs.x, qs.y, qs.z, qs.w };
    uint32_t lo[8], hi[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        bytes4_to_half2x2( w[i]       & 0x0F0F0F0Fu, dd, no, lo[2*i], lo[2*i+1]);   // elements 4i..4i+3
        bytes4_to_half2x2((w[i] >> 4) & 0x0F0F0F0Fu, dd, no, hi[2*i], hi[2*i+1]);   // elements 16+4i..
    }
    out[0] = make_uint4(lo[0], lo[1], lo[2], lo[3]); out[1] = make_uint4(lo[4], lo[5], lo[6], lo[7]);
    out[2] = make_uint4(hi[0], hi[1], hi[2], hi[3]); out[3] = make_uint4(hi[4], hi[5], hi[6], hi[7]);
}
__device__ __forceinline__ void dequant_q5_0(const uint4 qs, const uint32_t qh, const __half d, uint4 (&out)[4]) {
    const __half2 dd = __half2half2(d);
    const __half2 no = __float2half2_rn(1040.0f);               // 1024 + 16
    const uint32_t w[4] = { qs.x, qs.y, qs.z, qs.w };
    uint32_t lo[8], hi[8];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const uint32_t bl = ( w[i]       & 0x0F0F0F0Fu) | spread4_to_bit4(qh >> (4*i));
        const uint32_t bh = ((w[i] >> 4) & 0x0F0F0F0Fu) | spread4_to_bit4(qh >> (16 + 4*i));
        bytes4_to_half2x2(bl, dd, no, lo[2*i], lo[2*i+1]);
        bytes4_to_half2x2(bh, dd, no, hi[2*i], hi[2*i+1]);
    }
    out[0] = make_uint4(lo[0], lo[1], lo[2], lo[3]); out[1] = make_uint4(lo[4], lo[5], lo[6], lo[7]);
    out[2] = make_uint4(hi[0], hi[1], hi[2], hi[3]); out[3] = make_uint4(hi[4], hi[5], hi[6], hi[7]);
}
__device__ __forceinline__ void dequant_q8_0(const uint4 q0, const uint4 q1, const __half d, uint4 (&out)[4]) {
    const __half2 dd = __half2half2(d);
    const __half2 no = __float2half2_rn(1152.0f);               // 1024 + 128 ; bytes are biased by ^0x80
    const uint32_t w[8] = { q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w };
    uint32_t h[16];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        // (b ^ 0x80) is b + 128 as unsigned; split in two 0..255 bytes needs 0x6400|b: b < 256 occupies 8 mantissa bits: exact
        bytes4_to_half2x2(w[i] ^ 0x80808080u, dd, no, h[2*i], h[2*i+1]);
    }
    out[0] = make_uint4(h[0], h[1], h[2], h[3]);   out[1] = make_uint4(h[4], h[5], h[6], h[7]);
    out[2] = make_uint4(h[8], h[9], h[10], h[11]); out[3] = make_uint4(h[12], h[13], h[14], h[15]);
}

// Q4_1 / Q5_1: 32 unsigned values (bytes of q: element order of dequant_q4_0 / _q5_0) -> y = q * d + m evaluated in f32 (each
// product and sum rounded: dequantize_row_q4_1 / _q5_1 without contraction), then rounded once to f16
__device__ __forceinline__ void dequant_q1_bytes(const uint32_t (&lo)[4], const uint32_t (&hi)[4], float d, float m, uint4 (&out)[4]) {
    uint32_t h[16];
#pragma unroll
    for (int v = 0; v < 2; ++v)
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const uint32_t b = v ? hi[i] : lo[i];
            float f[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) f[e] = __fadd_rn(__fmul_rn((float) ((b >> (8 * e)) & 0xFFu), d), m);
            const __half2 a = __floats2half2_rn(f[0], f[1]), c = __floats2half2_rn(f[2], f[3]);
            h[8 * v + 2 * i]     = *reinterpret_cast<const uint32_t *>(&a);
            h[8 * v + 2 * i + 1] = *reinterpret_cast<const uint32_t *>(&c);
        }
    out[0] = make_uint4(h[0], h[1], h[2], h[3]);   out[1] = make_uint4(h[4], h[5], h[6], h[7]);
    out[2] = make_uint4(h[8], h[9], h[10], h[11]); out[3] = make_uint4(h[12], h[13], h[14], h[15]);
}
__device__ __forceinline__ void dequant_q4_1(const uint4 qs, const __half d, const __half m, uint4 (&out)[4]) {
    const uint32_t w[4] = { qs.x, qs.y, qs.z, qs.w };
    uint32_t lo[4], hi[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) { lo[i] = w[i] & 0x0F0F0F0Fu; hi[i] = (w[i] >> 4) & 0x0F0F0F0Fu; }
    dequant_q1_bytes(lo, hi, __half2float(d), __half2float(m), out);
}
__device__ __forceinline__ void dequant_q5_1(const uint4 qs, const uint32_t qh, const __half d, const __half m, uint4 (&out)[4]) {
    const uint32_t w[4] = { qs.x, qs.y, qs.z, qs.w };
    uint32_t lo[4], hi[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        lo[i] = ( w[i]       & 0x0F0F0F0Fu) | spread4_to_bit4(qh >> (4*i));
        hi[i] = ((w[i] >> 4) & 0x0F0F0F0Fu) | spread4_to_bit4(qh >> (16 + 4*i));
    }
    dequant_q1_bytes(lo, hi, __half2float(d), __half2float(m), out);
}

// 6-bit scale / min of sub-block j (0..7) from the 12 packed bytes (ggml-quants.c:880-887)
__device__ __forceinline__ void kq_scale_min(int j, const uint8_t * q, int & sc, int & m) {
    if (j < 4) { sc = q[j] & 63; m = q[j + 4] & 63; }
    else       { sc = (q[j + 4] & 0xF) | ((q[j - 4] >> 6) << 4); m = (q[j + 4] >> 4) | ((q[j] >> 6) << 4); }
}

// tile-major K-quant records: (d * sc_j, dmin * m_j) of the rows g and g + 8 of the tile for sub-block j, from the 8 header bytes this lane
// holds (layout above: lane 4g + c has bytes 8 (c & 1) .. + 7 of row g + 8 (c >> 1)).  Quad shuffles: the whole warp calls it with one j.
__device__ __forceinline__ void kq_tm_scales(uint2 hp, int j, int c, float & dl0, float & ml0, float & dl1, float & ml1) {
    const int sh = 8 * (j & 3);
    uint32_t part;                                               // this lane's share of (sc | m << 8) of its row (get_scale_min_k4)
    if (c & 1) {                                                 // hp = scales[4..7], scales[8..11]
        const uint32_t bz = (hp.x >> sh) & 0xffu, bw = (hp.y >> sh) & 0xffu;
        const uint32_t m = (j < 4) ? (bz & 63u) : ((bw >> 4) | ((bz >> 6) << 4));
        part = ((j < 4) ? 0u : (bw & 0xFu)) | (m << 8);
    } else {                                                     // hp = d | dmin << 16, scales[0..3]
        const uint32_t by = (hp.y >> sh) & 0xffu;
        part = (j < 4) ? (by & 63u) : ((by >> 6) << 4);
    }
    const uint32_t s  = part | __shfl_xor_sync(0xffffffffu, part, 1);
    const uint32_t dp = __shfl_xor_sync(0xffffffffu, hp.x, 1);
    const uint32_t dm = (c & 1) ? dp : hp.x;
    const uint32_t s2 = __shfl_xor_sync(0xffffffffu, s, 2), dm2 = __shfl_xor_sync(0xffffffffu, dm, 2);
    const uint32_t s0 = (c & 2) ? s2 : s, d0 = (c & 2) ? dm2 : dm, s1 = (c & 2) ? s : s2, d1 = (c & 2) ? dm : dm2;
    dl0 = __half2float(__ushort_as_half((unsigned short) (d0 & 0xffffu))) * (float) (s0 & 0xffu);
    ml0 = __half2float(__ushort_as_half((unsigned short) (d0 >> 16)))     * (float) (s0 >> 8);
    dl1 = __half2float(__ushort_as_half((unsigned short) (d1 & 0xffffu))) * (float) (s1 & 0xffu);
    ml1 = __half2float(__ushort_as_half((unsigned short) (d1 >> 16)))     * (float) (s1 >> 8);
}

// decode sub-block j (32 values) of a Q4_K / Q5_K super-block into 32 halves.
// y = d*sc*q - dmin*m  evaluated in f32 then rounded once to f16.
template <bool Q5>
__device__ __forceinline__ void dequant_kq_sub(const uint8_t * __restrict__ blk, int j, uint4 (&out)[4]) {
    const uint4 hdr = *reinterpret_cast<const uint4 *>(blk);          // d, dmin, scales[12]
    const __half2 dm = *reinterpret_cast<const __half2 *>(&hdr.x);
    const uint32_t sw[3] = { hdr.y, hdr.z, hdr.w };
    const uint8_t * sc8 = reinterpret_cast<const uint8_t *>(sw);
    int sc, mn; kq_scale_min(j, sc8, sc, mn);
    const float dl = __low2float(dm) * (float) sc;
    const float ml = __high2float(dm) * (float) mn;
    const uint8_t * qs = blk + 16 + (Q5 ? 32 : 0) + 32 * (j >> 1);
    const uint8_t * qh = blk + 16;
    const int sh = 4 * (j & 1);
    uint32_t h[16];
#pragma unroll
    for (int v = 0; v < 2; ++v) {
        const uint4 q4 = *reinterpret_cast<const uint4 *>(qs + 16 * v);
        uint4 hb = make_uint4(0, 0, 0, 0);
        if (Q5) hb = *reinterpret_cast<const uint4 *>(qh + 16 * v);
        const uint32_t w[4]  = { q4.x, q4.y, q4.z, q4.w };
        const uint32_t hw[4] = { hb.x, hb.y, hb.z, hb.w };
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            uint32_t b = (w[i] >> sh) & 0x0F0F0F0Fu;
            if (Q5) b |= ((hw[i] >> j) & 0x01010101u) << 4;
            float f[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) f[e] = dl * (float) ((b >> (8*e)) & 0xFF) - ml;
            const __half2 a = __floats2half2_rn(f[0], f[1]);
            const __half2 c = __floats2half2_rn(f[2], f[3]);
            h[8*v + 2*i]     = *reinterpret_cast<const uint32_t *>(&a);
            h[8*v + 2*i + 1] = *reinterpret_cast<const uint32_t *>(&c);
        }
    }
    out[0] = make_uint4(h[0], h[1], h[2], h[3]);   out[1] = make_uint4(h[4], h[5], h[6], h[7]);
    out[2] = make_uint4(h[8], h[9], h[10], h[11]); out[3] = make_uint4(h[12], h[13], h[14], h[15]);
}

// Q3_K verbatim super-blocks (hmask[32] qs[64] scales[12] f16 d = 110 B).  Blocks are only 2-byte aligned in a row of super-blocks,
// so words are read as two halves.
__device__ __forceinline__ uint32_t ld_u32_a2(const uint8_t * p) {
    const uint16_t * h = reinterpret_cast<const uint16_t *>(p);
    return (uint32_t) h[0] | ((uint32_t) h[1] << 16);
}
// the signed values e .. e + 3 (e % 4 == 0) of a super-block, packed as int8
__device__ __forceinline__ uint32_t q3k_q4(const uint8_t * blk, int e) {
    const int n = e >> 7, r = (e >> 5) & 3, l = e & 31;
    const uint32_t qs = ld_u32_a2(blk + 32 + 32 * n + l), hm = ld_u32_a2(blk + l);
    return __vsub4(((qs >> (2 * r)) & 0x03030303u) | (((hm >> (4 * n + r)) & 0x01010101u) << 2), 0x04040404u);
}
// integer scale of values 16 is .. 16 is + 15 (is = 0 .. 15) from the 12 packed bytes: the 6-bit value - 32
__device__ __forceinline__ int q3k_scale(const uint8_t * blk, int is) {
    const int k = is >> 2, i = is & 3;
    return (int) (((blk[96 + (k & 1) * 4 + i] >> (4 * (k >> 1))) & 0xF) | (((blk[104 + i] >> (2 * k)) & 3) << 4)) - 32;
}
__device__ __forceinline__ uint32_t q3k_dbits(const uint8_t * blk) { return *reinterpret_cast<const uint16_t *>(blk + 108); }
__device__ __forceinline__ float q3k_d(const uint8_t * blk) { return __half2float(__ushort_as_half((unsigned short) q3k_dbits(blk))); }
// (d * sc) * q of value e (0 .. 255), each product rounded in f32: dequantize_row_q3_K
__device__ __forceinline__ float q3k_elem(const uint8_t * blk, int e) {
    const int q = (int) (int8_t) ((q3k_q4(blk, e & ~3) >> (8 * (e & 3))) & 0xffu);
    return __fmul_rn(__fmul_rn(q3k_d(blk), (float) q3k_scale(blk, e >> 4)), (float) q);
}
// sub-block j (32 values) of a Q3_K super-block into 32 halves: the f16 rounding of dequantize_row_q3_K's f32 value
__device__ __forceinline__ void dequant_q3k_sub(const uint8_t * __restrict__ blk, int j, uint4 (&out)[4]) {
    const float d = q3k_d(blk);
    uint32_t h[16];
#pragma unroll
    for (int v = 0; v < 8; ++v) {
        const float dl = __fmul_rn(d, (float) q3k_scale(blk, 2 * j + (v >> 2)));
        const uint32_t q = q3k_q4(blk, 32 * j + 4 * v);
        float f[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) f[e] = __fmul_rn(dl, (float) (int) (int8_t) ((q >> (8 * e)) & 0xffu));
        const __half2 a = __floats2half2_rn(f[0], f[1]), c = __floats2half2_rn(f[2], f[3]);
        h[2 * v] = *reinterpret_cast<const uint32_t *>(&a); h[2 * v + 1] = *reinterpret_cast<const uint32_t *>(&c);
    }
    out[0] = make_uint4(h[0], h[1], h[2], h[3]);   out[1] = make_uint4(h[4], h[5], h[6], h[7]);
    out[2] = make_uint4(h[8], h[9], h[10], h[11]); out[3] = make_uint4(h[12], h[13], h[14], h[15]);
}

// bit 2 of byte e of a word -> bit e (the four high bits of Q3_K's stored values q + 4)
__device__ __forceinline__ uint32_t spread_bit2(uint32_t u) {
    return ((u >> 2) & 1u) | ((u >> 9) & 2u) | ((u >> 16) & 4u) | ((u >> 23) & 8u);
}
// Q3_K tile-major sub-block record -> the four signed A registers of lane (g, c): wl = low bit pairs, wh = hmask bits of rows g, g + 8
__device__ __forceinline__ void q3k_tm_af(uint32_t wl, uint2 wh, int c, uint32_t (&af)[4]) {
    af[0] = ( wl       & 0x03030303u) | (spread4_to_bit4(wh.x >> (4 * c)) >> 2);
    af[1] = ((wl >> 2) & 0x03030303u) | (spread4_to_bit4(wh.y >> (4 * c)) >> 2);
    af[2] = ((wl >> 4) & 0x03030303u) | (spread4_to_bit4(wh.x >> (16 + 4 * c)) >> 2);
    af[3] = ((wl >> 6) & 0x03030303u) | (spread4_to_bit4(wh.y >> (16 + 4 * c)) >> 2);
#pragma unroll
    for (int r = 0; r < 4; ++r) af[r] = __vsub4(af[r], 0x04040404u);
}
// D = A (16 x 16, s8) . B (16 x 8, s8) in s32: A = rows g / g + 8, values 4c .. 4c + 3 of lane 4g + c; B = values 4c .. 4c + 3 of column g
__device__ __forceinline__ void mma_s8_16816(int (&d)[4], const uint32_t (&a)[2], uint32_t b) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.s32.s8.s8.s32 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%7,%8,%9,%10};"
                 : "=r"(d[0]), "=r"(d[1]), "=r"(d[2]), "=r"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(b), "r"(0), "r"(0), "r"(0), "r"(0));
}
// sumi of one 32-value sub-block against its scales: two k16 integer products, combined with the rows' two 16-value scales each
// (|result| <= 2 * 16 * 4 * 127 * 32: exact in f32).  sw = the lane's scale word, d[i] as mma_s8_16832's.
__device__ __forceinline__ void q3k_sumi(const uint32_t (&af)[4], uint32_t b0, uint32_t b1, uint32_t sw, int (&s)[4]) {
    int lo[4], hi[4];
    const uint32_t a_lo[2] = { af[0], af[1] }, a_hi[2] = { af[2], af[3] };
    mma_s8_16816(lo, a_lo, b0);
    mma_s8_16816(hi, a_hi, b1);
    const int s0l = (int) (int8_t) (sw & 0xffu), s0h = (int) (int8_t) ((sw >> 8) & 0xffu);
    const int s1l = (int) (int8_t) ((sw >> 16) & 0xffu), s1h = (int) (int8_t) (sw >> 24);
    s[0] = s0l * lo[0] + s0h * hi[0]; s[1] = s0l * lo[1] + s0h * hi[1];
    s[2] = s1l * lo[2] + s1h * hi[2]; s[3] = s1l * lo[3] + s1h * hi[3];
}

#endif // __CUDACC__
} // namespace wb
