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

struct MkArgs {
    const MkLayer * layers; int n_layer;
    int d, n_head, n_tok, n_keys, ld_idx, n_vocab, want_logits;
    const int * tok, * pos, * cell, * slot, * nkv, * idx;      // per-row integers of this pass (device)
    int64_t slot_stride;              // elements between the cross KV of consecutive slots
    float kq_scale, eps;
    QMat te; const float * pe;        // token embedding (also the logits matrix) and positional embedding
    const float * lnf_w, * lnf_b;     // final LayerNorm
    float * x, * qkv, * q2, * logits;                         // f32 workspaces: [R][d], [R][3d], [R][d], [R][V]   (R = mk_max_rows())
    float * h;                        // FC1 + GELU output [R][4d]
    uint8_t * actq, * hq;             // quantised rows handed between phases: K = d (>= R*d*2 + R*d/8 bytes) and K = 4d
    float * xpart; int * xcnt;        // cross-attention partials [R*H][16][66] and arrival counters [R*H]
    unsigned long long * bar;         // grid barrier: [0] arrival counter (monotonic, never reset), [16 + 16*cta] release flag of each CTA
    unsigned long long bar_base;      // its value when this launch starts
    int * err;                        // set to 1 when a barrier wait times out
    long long * trace;                // optional: phase time stamps of CTA 0 (see MK_STAMP)
    float * cap = nullptr; const int * cap_row = nullptr; int cap_rows = 0;   // DTW capture (generation 1 only): null when no row of the pass has a capture index
    int prefetch;                     // bit0: next-phase weights -> L2, bit1: cross KV -> L2 one phase ahead
    // second generation (wb_decode_mk2.cu) only:
    int global_sync = 0;              // a row attends to self-KV cells another row GROUP writes in this pass: all groups meet after the KV append
    int stagger_clk = 0;              // SM cycles between the starts of consecutive row groups
};

// number of grid barriers one launch passes (host keeps bar_base in step)
int  mk_barriers(int wtype, int n_layer, bool want_logits);
bool mk_supported(int wtype);
size_t mk_smem_bytes(int wtype, int d);
bool mk_cross_head_major();        // cross K/V of a window is expected head-major ([layer][head][key][64])
int  mk_max_rows();                 // rows (sequences x tokens) one launch can take
// cooperative launch on `st`; grid = number of SMs.  Returns false (with the error set) when the launch is refused.
bool mk_launch(const MkArgs & a, int wtype, int n_sm, cudaStream_t st);

// ---- second generation (wb_decode_mk2.cu): row groups of 16 walk the layers independently, two CTAs per SM ----
int  mk2_ctas_per_sm();
bool mk2_supported(int wtype, int d);
size_t mk2_smem_bytes();
size_t mk2_bar_words(int n_sm);     // 64-bit words of MkArgs::bar: [0..127] counters (zeroed by mk2_launch), then 16 per CTA (release flags)
// cooperative launch on `st`; grid = 2 x number of SMs.  a.bar_base must grow by 4096 per launch.
bool mk2_launch(const MkArgs & a, int wtype, int n_sm, cudaStream_t st);

} // namespace wb
