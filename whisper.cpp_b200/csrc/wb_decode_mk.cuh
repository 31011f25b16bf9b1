// wb_decode_mk.cuh -- the text decoder step (whisper_build_graph_decoder, src/whisper.cpp:2466-2844) as ONE persistent
// cooperative kernel: one CTA per SM walks all layers, phases are separated by a grid-wide barrier instead of kernel
// boundaries, and the weights of the next phase are pulled into L2 while the current phase computes.
#pragma once
#include <cstdint>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include "wb_quant.cuh"

namespace wb {

struct MkLayer {                      // one text layer: weights (model) + this engine's KV pointers
    QMat qkv, o, cq, co, fc1, fc2;
    const float * ln0_w, * ln0_b, * lnc_w, * lnc_b, * lnm_w, * lnm_b;
    const float * qkv_bias, * qkv_scale, * o_bias, * cq_bias, * co_bias, * fc1_bias, * fc2_bias;
    __half * kc, * vc;                // self-attention KV of this layer: [n_cells][d]
    const __half * xk, * xv;          // cross-attention K / V of this layer in slot 0: [Tp][d]
    uint32_t cap_mask; int cap_head0; // DTW: alignment heads of this layer (bit h = head h) and the capture head of the lowest (wb_dtw_kernel.cuh)
};

// A pass with enough rows is cut into partitions: partition p owns whole 16-row groups [p*G/NP, (p+1)*G/NP) of the G row groups and the
// CTAs [p*n_cta/NP, (p+1)*n_cta/NP), and walks the layers on its own barrier, so that one partition streams cross K/V from HBM while
// the others are in their latency-bound phases.  A row's arithmetic does not depend on how many CTAs share a phase: NP changes no bit.
constexpr int MK_MAX_PARTS = 4;
struct MkPart { int c0, nc, row0, n_tok; };                       // first CTA / CTAs, first row / rows of a partition
__host__ __device__ inline MkPart mk_partition(int p, int n_part, int n_cta, int n_tok) {
    const int G = (n_tok + 15) >> 4, g0 = p * G / n_part, g1 = (p + 1) * G / n_part;
    const int c0 = p * n_cta / n_part, c1 = (p + 1) * n_cta / n_part;
    const int r0 = g0 * 16, r1 = g1 * 16 < n_tok ? g1 * 16 : n_tok;
    return MkPart{ c0, c1 - c0, r0, r1 - r0 };
}

struct MkArgs {
    const MkLayer * layers; int n_layer;
    int d, n_head, n_tok, n_keys, ld_idx, n_vocab, want_logits;
    int n_audio_ctx;                  // encoder positions of the cross K/V (<= n_keys): keys n_audio_ctx .. n_keys - 1 are zero rows
    int kv_rows;                      // rows per head of the cross K/V buffer (>= n_keys): the producer's layout, not the pass's key count
    const int * tok, * pos, * cell, * slot, * nkv, * idx;      // per-row integers of this pass (device)
    int64_t slot_stride;              // elements between the cross KV of consecutive slots
    float kq_scale, eps;
    QMat te; const float * pe;        // token embedding (also the logits matrix) and positional embedding
    const float * lnf_w, * lnf_b;     // final LayerNorm
    float * x, * qkv, * q2, * logits;                         // f32 workspaces: [R][d], [R][3d], [R][d], [R][V]   (R = mk_max_rows())
    float * h;                        // FC1 + GELU output [R][4d]
    uint8_t * actq, * hq;             // quantised rows handed between phases: K = d (>= R*d*2 + R*d/8 bytes) and K = 4d
    float * xpart; int * xcnt;        // cross-attention partials [R*H][16][66] and arrival counters [R*H]
    unsigned long long * bar;         // barriers (mk_bar_words): arrival counters (monotonic, never reset) of the grid and of each partition, release flags per CTA, the turn word
    unsigned long long bar_base;      // value of the grid counter when this launch starts
    unsigned long long part_base[MK_MAX_PARTS];   // ... and of the partitions' counters
    int n_part = 1;                   // partitions of this pass (mk_partition): CTA ranges that walk the layers on their own barriers
    int turn_slots = 1;               // partitions that may stream cross K/V at the same time
    int * err;                        // set to 1 when a barrier wait times out
    long long * trace;                // optional: phase time stamps of CTA 0 (see MK_STAMP)
    float * cap = nullptr; const int * cap_row = nullptr; int cap_rows = 0;   // DTW capture: null when no row of the pass has a capture index
    int prefetch;                     // bit0: next-phase weights -> L2, bit1: cross KV -> L2 one phase ahead
};

// barriers one launch passes: per layer on the partitions' counters (every CTA of partition p arrives at counter p), plus the grid-wide
// one in front of the logits.  The host keeps bar_base / part_base in step.
int  mk_layer_barriers(int wtype);
size_t mk_bar_words(int n_sm);      // 64-bit words of MkArgs::bar
bool mk_supported(int wtype);
size_t mk_smem_bytes(int wtype, int d);
bool mk_cross_head_major();        // cross K/V of a window is expected head-major ([layer][head][key][64])
int  mk_max_rows();                 // rows (sequences x tokens) one launch can take
// cooperative launch on `st`; grid = number of SMs.  Returns false (with the error set) when the launch is refused.
bool mk_launch(const MkArgs & a, int wtype, int n_sm, cudaStream_t st);

// Test probe (wb200_dbg_mk_phase): ONE phase of the pass run by an ordinary launch of n_cta CTAs on the rows [row0, row0 + n_tok), with
// the pass's shared-memory carve-up and the same phase functions.  The GEMV phase with the token-embedding matrix is the split-K logits.
enum MkProbePhase { MKP_LNQ = 0, MKP_Q8K = 1, MKP_GEMV = 2, MKP_GEMV_PAIR = 3, MKP_LOGITS_WARP = 4, MKP_ATTN_SELF = 5, MKP_ATTN_CROSS = 6 };
struct MkProbe {
    int phase, row0, n_tok;
    QMat W;                            // GEMV / logits: tile-major weights
    const QMat * Wg;                   // the same in device memory (FC1: the pass hands that phase only layer matrices, which live there)
    const uint8_t * x;                 // GEMV / logits: actq rows (K = W.K)
    const float * bias, * scale, * res; int act;   // GEMV epilogue (res [64][N]); LN: scale = ln_w, bias = ln_b
    float * out;                       // GEMV / logits: f32 [64][N]
    __half * kc, * vc; int kv_d;       // GEMV: K / V append at MkArgs::cell
    const float * src; int lds, K;     // LN / Q8_K: f32 rows `lds` apart, K values each
    uint8_t * dst;                     // LN / Q8_K / FC1 PAIR: actq rows
    const MkLayer * L;                 // attention (device memory, as MkArgs::layers): kc, vc (self), xk, xv (cross)
};
bool mk_probe_launch(const MkArgs & a, const MkProbe & p, int wtype, int n_cta, cudaStream_t st);

} // namespace wb
