// wb_gemm.cuh -- host-side description of one wgmma GEMM launch.
//
//   C[m][n] = sum_{tap} sum_{k} A[m][tap][k] * B[n][tap][k]            (both operands K-major, f16 in smem)
//
// "A" is the weight side: 128 rows per CTA, 64 per MMA warpgroup.  It is either an f16 matrix fetched by TMA
// or a quantised matrix (planar Q4_0/Q5_0/Q8_0, verbatim Q4_K/Q5_K) whose 32-value blocks are decoded to f16 by
// the producer warpgroup straight into the 128-byte-swizzled operand tile.
// "B" is the activation side (tokens / time steps / queries): BN rows per CTA fetched by TMA.
// This replaces ggml_mul_mat (ggml/src/ggml-cpu/ggml-cpu.c:1254-1452) + the separate add/scale/gelu/cpy nodes the
// reference graphs attach to it (src/whisper.cpp:2119-2123, 2225-2239, 2309-2346, 2012-2020).
#pragma once
#include <cstdint>
#include <cuda.h>
#include <cuda_runtime.h>
#include "wb_quant.cuh"

namespace wb {

struct GemmEpilogue {
    const float * bias_m  = nullptr;  // [M] added first
    const float * scale_m = nullptr;  // [M] multiplies (acc + bias)
    float alpha = 1.0f;               // scalar factor applied with scale_m
    int   act   = 0;                  // 1: GELU with the reference's f16-table semantics (ggml-cpu/vec.h:988-1001)
    const float * res = nullptr;      // residual, f32, indexed res[n*ldr + m] (+ batch strides), added last
    int64_t ldr = 0;
    void *  out = nullptr;            // f32 or f16
    int     out_f16 = 0;
    int     out_mmajor = 0;           // 0: out[n*ldo + m]   1: out[m*ldo + n]
    int64_t ldo = 0;
    int64_t out_b0 = 0, out_b1 = 0;   // element strides of the two batch indices
    int64_t res_b0 = 0, res_b1 = 0;
    int     n_row_off = 0;            // written row index = n + n_row_off (used to leave a padding row in front)
    int64_t hm_rows = 0;              // > 0 (with out_mmajor = 0): head-major output [m / 64][hm_rows][64] instead of [n][ldo] (cross K/V)
};

struct GemmDesc {
    int M = 0, N = 0, K = 0;          // K per tap
    int taps = 1;                     // 3 for the conv stem (tap is TMA dim 2 of both operands)
    int BN = 128;                     // 64 / 128 / 256
    int nb0 = 1, nb1 = 1;             // batch extents (blockIdx.z = b1*nb0 + b0)
    // what feeds TMA coordinates z2 / z3 of each operand: 0 = zero, 1 = b0, 2 = b1, 3 = tap
    int a_zsel[2] = { 0, 0 };
    int b_zsel[2] = { 1, 2 };
    int b1_in_off = 0;                // added to b1 when it is used as a TMA coordinate (one window of a batched buffer per launch)
    int a_rows_per_b0 = 0;            // A row offset = b0 * a_rows_per_b0 (stacked weights: one launch, many matrices)
    QMat A;                           // weight side; type WT_F16 => tmA used
    CUtensorMap tmA;                  // valid when A.type == WT_F16, or when a16 is set (then it maps a16)
    __half * a16 = nullptr;           // quantised A: f16 scratch [rows][K] the persistent kernel's launch expands A into (shared by all launches of a stream)
    int v2 = 0;                       // 1: persistent launch (one CTA per SM walks the tile list), A in f16 through TMA
    int half_box_b = 0;               // 1: tmB was built with box_rows = BN / 2 (BN >= 128); the B tile is fetched as two halves
    int a16_keep = 0;                 // 1: a16 already holds this matrix (a launch sequence over the same weights expands them once)
    CUtensorMap tmB;
    GemmEpilogue ep;
};

// 4-D tensor map over f16 data: dims {k, rows, z2, z3}; strides in ELEMENTS for dims 1..3; box = {64, box_rows, 1, 1};
// 128-byte swizzle.  Returns false (and sets wb error text) on failure.
bool make_tmap_f16(CUtensorMap * out, const void * base, uint64_t k, uint64_t rows, uint64_t z2, uint64_t z3,
                   uint64_t stride_rows, uint64_t stride_z2, uint64_t stride_z3, uint32_t box_rows);

// enqueue on `stream`; returns cudaError
cudaError_t gemm_launch(const GemmDesc & g, cudaStream_t stream);

// expand `rows` rows of a quantised matrix (planar 32-blocks or verbatim K-quants) to f16 [rows][K]
cudaError_t dequant_to_f16(const QMat & W, int64_t rows, __half * out, cudaStream_t stream);

} // namespace wb
