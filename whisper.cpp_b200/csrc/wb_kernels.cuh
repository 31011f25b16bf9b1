// wb_kernels.cuh -- launchers of the non-GEMM kernels (see wb_kernels.cu for the reference lines each follows).
#pragma once
#include <cstdint>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include "wb_quant.cuh"

namespace wb {

// ---- conversions / weight re-layout -------------------------------------------------------------------------------
void f32_to_f16(const float * src, __half * dst, int64_t n, cudaStream_t st);
void f16_to_f32(const __half * src, float * dst, int64_t n, cudaStream_t st);
// file-layout 32-blocks (18/22/34 B each, [rows][K/32]) -> planar arrays of `dst` (already offset to the first row)
bool repack_block32_into(int wtype, const uint8_t * file_blocks_dev, const QMat & dst, int rows, int K, cudaStream_t st);
// convenience for tests: carve the planar arrays out of one buffer
bool repack_block32(int wtype, const uint8_t * file_blocks_dev, uint8_t * dst, int N, int K, QMat * out, cudaStream_t st);
// file-layout rows (32-blocks, K-quant super-blocks, or f16 rows for WT_F16) -> tile-major records (wb_quant.cuh) of `dst` (layout 1)
// starting at row row_off (multiple of 16)
bool repack_tile_major(int wtype, const uint8_t * file_rows_dev, const QMat & dst, int row_off, int rows, cudaStream_t st);
// every element of W through the embedding reader (dequant_elem): f32 [N][K] (test hook)
void dequant_rows_f32(const QMat & W, float * out, cudaStream_t st);

// ---- log-mel (src/whisper.cpp:3005-3272) ---------------------------------------------------------------------------
// pcm: n_samples f32 on device.  mel: [n_mel][n_len] f32 with n_len = (n_samples + 480000)/160.  gmax: 1 float scratch.
void mel_spectrogram(const float * pcm, int n_samples, const float * filters, int n_mel, float * mel, int n_len,
                     float * gmax_scratch, cudaStream_t st);
// window of 2*n_ctx frames starting at `seek` -> time-major f16 [2*n_ctx + 2][n_mel], rows 0 and 2*n_ctx+1 zero
// (src/whisper.cpp:2389-2411: frames past n_len are zero)
void mel_window_f16(const float * mel, int n_len, int n_mel, int seek, int n_frames, __half * out, cudaStream_t st);

// ---- LayerNorm (ggml-cpu/ops.cpp:3698-3765 two-pass + mul/add, src/whisper.cpp:2108-2115) ---------------------------
// out16 and/or out32 may be null
void layernorm(const float * x, const float * w, const float * b, float eps, int rows, int d,
               __half * out16, float * out32, cudaStream_t st);

// ---- unfused attention helper: softmax over rows of f32 scores -> f16 probabilities --------------------------------
void softmax_rows_f16(const float * s, __half * p, int64_t rows, int cols, cudaStream_t st);

// ---- fused encoder self-attention (wb_fattn.cu).  qk: f16 [n_win][T][ld_qk], head h at columns h*64, K at +k_off;
// vt: f16 [n_win][H*64][Tp] (V transposed, zero beyond T); out: f16 [n_win*T][ldo]
bool fattn_encoder(const __half * qk, int ld_qk, int k_off, const __half * vt, int T, int Tp, int H, int n_win, float scale,
                   __half * out, int ldo, cudaStream_t st);

// ---- decoder step (src/whisper.cpp:2466-2844) -----------------------------------------------------------------------
// x[t][:] = dequant(d_te[token[t]]) + d_pe[pos[t]]   (get_rows + add, whisper.cpp:2523-2526)
void dec_embed(const QMat & te, const float * pe, const int * tokens, const int * pos, int n_tok, int d, float * x, cudaStream_t st);

struct GemvArgs {
    QMat W;                       // [N][K]
    const float * x = nullptr;    // [n_tok][K] f32 (ldx = K)
    int n_tok = 1;                // 1..8
    const float * ln_w = nullptr; // optional fused LayerNorm of x before the contraction
    const float * ln_b = nullptr;
    float eps = 1e-5f;
    const float * bias = nullptr;   // [N]
    const float * scale = nullptr;  // [N] multiplies (acc + bias)
    int act = 0;                    // 1: GELU (reference f16-table semantics)
    const float * res = nullptr;    // [n_tok][N] added last (may alias out)
    float * out = nullptr;          // [n_tok][N] f32 (nullable when only the KV store is wanted)
    // optional KV append (decoder self-attention): rows [kv_d, 2kv_d) -> k_cache, [2kv_d, 3kv_d) -> v_cache, rounded to f16
    __half * k_cache = nullptr; __half * v_cache = nullptr; const int * cells = nullptr; int kv_d = 0;
};
// bytes of one token's activation row as both GEMVs hold it (v1: in shared memory, v2: in act_scratch), padded to 16:
// int8 q[K] | f32 d[K/32] (Q8_0) or {f16 d, f16 s}[K/32] (Q8_1) | f32 d[K/256] + int sum[K/32] (Q8_K); F16 weights: half[K]
__host__ __device__ inline size_t act_tok_stride(int wtype, int K) {
    const size_t b = wtype == WT_F16 ? (size_t) K * 2 : (size_t) K + (wt_is_kquant(wtype) ? (size_t) (K / 256) * 4 : 0) + (size_t) (K / 32) * 4;
    return (b + 15) & ~size_t(15);
}
void gemv(const GemvArgs & a, cudaStream_t st);            // v1: dp4a, activation quantisation inside every CTA
// v2: k_act_quant (one CTA per token) + int8 tensor-core block dots, 16 or 32 rows per CTA.  act_scratch: >= 8 * act_tok_stride bytes
void gemv2(const GemvArgs & a, uint8_t * act_scratch, cudaStream_t st);

// self-attention for n_tok query tokens over a paged KV cache.  q: [n_tok][d] f32 (already scaled),
// k/v cache: [n_cells][d] f16 for this layer.  idx[t*ld_idx + i], i < n_kv[t] lists the cells token t may attend to.
void attn_self_decode(const float * q, int ldq, const __half * kc, const __half * vc, const int * idx, int ld_idx,
                      const int * n_kv, int n_tok, int n_head, int d, float * out, int ldo, cudaStream_t st);
// cross-attention over the 1536 padded keys (zero rows included, whisper.cpp:2689-2703). kc/vc: per-token base pointers
// are kc + slot[t]*slot_stride.  partial: scratch [n_tok][n_head][NSPLIT][66] f32, counters: [n_tok][n_head] ints (zeroed).
void attn_cross_decode(const float * q, int ldq, const __half * kc, const __half * vc, const int * slot, int64_t slot_stride,
                       int n_keys, int n_tok, int n_head, int d, float scale, float * partial, int * counters,
                       float * out, int ldo, cudaStream_t st);


// ---- on-device logits filter + greedy pick (whisper_process_logits + whisper_sample_token(best), src/whisper.cpp:6196-6543)
struct SampCfg {                 // uniform for all rows of a pass
    const uint32_t * mask = nullptr;   // device bit mask [ceil(V/32)]: statically suppressed token ids
    int token_eot = 0, token_beg = 0, token_nosp = 0, space_id = -1;
    int suppress_blank = 1, no_timestamps = 0;
    int max_initial_tid = -1;          // round(max_initial_ts / precision), -1 = rule disabled
};
struct SampOut { int id, tid; float p, plog, pt, ptsum, nosp_raw;
                 float raw_max, raw_sum, raw_nosp; };    // unfiltered row: max logit, sum of exp(l - max), logit of the no-speech token
// rowinfo[2*r] flags: bit0 is_initial, bit1 last token was a timestamp, bit2 penultimate was (or < 2 tokens), bit3 has_ts,
// bit4 text tokens disabled by max_tokens, bits 8-14: number of categorical draws wanted for the row (beam search: whisper_sample_token_topk,
// src/whisper.cpp:6545-6618; 0 = greedy pick only); rowinfo[2*r+1] = seek_delta/2.  logits: [n][V] f32 on device (not modified).
// out: [n][stride] (entry 0 of a row: the greedy pick, or draw 0 when draws are wanted); draws: [n][stride] uniforms in [0, 1) from the host.
void greedy_sample(const float * logits, int V, int n, const int * rowinfo, const SampCfg & cfg, SampOut * out, cudaStream_t st,
                   const double * draws = nullptr, int stride = 1);
constexpr int SAMP_MAX_DRAWS = 64;
// tokens[t] < 0 is replaced by samp[-1 - tokens[t]].id: a row whose token is the pick of an earlier pass's sampler (run-ahead passes)
void tok_resolve(int * tokens, const SampOut * samp, int n_tok, cudaStream_t st);

} // namespace wb
