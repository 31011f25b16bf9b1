// wb_engine.h -- device-side execution of the four Whisper graphs for one `whisper_state`.
//
// Replaces whisper_encode_internal (src/whisper.cpp:2366-2464: conv + encoder + cross graphs) and
// whisper_decode_internal (src/whisper.cpp:2856-2986) together with the ggml scheduler underneath them.
// A state owns: the PCM / mel buffers, the encoder workspaces for up to `cap_win` 30-s windows processed in ONE
// batched pass, the cross-attention KV of each window ("slot"), the paged self-attention KV pool and the decode
// workspaces.  All work of a state is enqueued on its own CUDA stream.
#pragma once
#include <map>
#include <string>
#include <utility>
#include <vector>
#include "wb_model.h"
#include "wb_gemm.cuh"
#include "wb_kernels.cuh"
#include "wb_decode_mk.cuh"
#include "wb_dtw_kernel.cuh"

namespace wb {

struct EncPlan;   // tensor maps + launch descriptors for a given (n_ctx, n_win)

struct DecToken { // one row of a decode batch (whisper_batch, src/whisper.cpp:472-480)
    int32_t token, pos, seq, slot; bool want_logits;
};

// Per-state audio front-end: PCM and log-mel live on the device; independent of the (possibly shared) Engine.
struct FrontEnd {
    const Model * m = nullptr;
    cudaStream_t st = nullptr;
    DevBuf<float> pcm, mel, gmax;
    int n_len = 0, n_len_org = 0, n_mel = 0;
    int pcm_resident = 0;            // samples already in `pcm` (wb200_pcm_upload); pcm_to_mel(nullptr, n) then skips the H2D copy
    cudaEvent_t ev0 = nullptr, ev1 = nullptr;
    float last_mel_ms = 0.0f;
    ~FrontEnd();
    bool init(const Model * model);
    bool pcm_upload(const float * samples, int n_samples);
    bool pcm_to_mel(const float * samples, int n_samples, bool samples_on_device = false);
    bool set_mel(const float * data, int n_len, int n_mel);
};

// one 30-s window to encode: where its mel lives and which cross-KV slot it fills
struct EncSrc { const float * mel; int n_len; int n_mel; int seek; int slot; };

struct Engine {
    const Model * m = nullptr;
    cudaStream_t  st = nullptr;
    int cap_win = 1;                 // windows that can be encoded/decoded together
    int n_cells = 0;                 // self-KV pool size (cells) = cap_win * cps
    int cps = 0;                     // self-KV cells per slot; GGML_PAD(n_text_ctx,256) * factor (whisper.cpp:3402, 7167-7172)
    bool debug_taps = false;
    bool fused_attn = true;          // WB200_UNFUSED_ATTN=1 selects the 3-kernel path (scores -> softmax -> PV through HBM)

    // ---- encoder workspaces
    int Tp_max = 0;
    DevBuf<__half> mel_win, h1, xn, qk, vt, P, attn, hfc, enc16;
    DevBuf<float>  x, S, enc32, conv32;
    DevBuf<__half> wf16;             // f16 expansion of the quantised matrix the current encoder GEMM multiplies (wb_gemm.cu, k_dequant_f16)
    bool gemm_v2 = true;             // WB200_GEMM_V1=1 selects the first-generation kernel (in-kernel dequantisation, one tile per CTA)
    DevBuf<__half> kv_cross;         // [cap_win][2][Lt][Tp][d]; with the persistent decode kernel (use_mk) each [Tp][d] block is head-major [d/64][Tp][64]
    int enc_n_ctx = 0, enc_n_win = 0;   // what the last encode produced
    std::vector<int> slot_ctx;       // per cross-KV slot: encoder positions of its last encode (0: never encoded); states of one pool may differ
    int slot_n_ctx(int slot) const { return slot_ctx[(size_t) slot] > 0 ? slot_ctx[(size_t) slot] : m->hp.n_audio_ctx; }
    EncPlan * plan = nullptr;

    // ---- decoder
    DevBuf<__half> kv_k, kv_v;       // [Lt][n_cells][d]
    DevBuf<float>  dx, dqkv, dattn, dq2, dh, dlogits, xpart;
    DevBuf<uint8_t> dhq;              // quantised FC1 output rows of the persistent kernel
    DevBuf<uint8_t> act_scratch;      // quantised activations of the current GEMV (k_act_quant -> k_gemv_mma)
    bool gemv_v2 = true;             // WB200_GEMV_V1=1 selects the dp4a kernel
    // persistent decode kernel (wb_decode_mk.cu); WB200_MEGAKERNEL=0 selects the kernel-per-op chain
    // DTW token timestamps (wb_dtw_kernel.cuh): a decode row with a capture index >= 0 leaves the cross-attention queries of the alignment
    // heads in dtw_q [capture head][capture index][64].  Capture heads are the distinct alignment heads ordered by (layer, head).
    std::vector<uint32_t> dtw_layer_mask;   // per text layer: bit h = head h is an alignment head
    std::vector<int> dtw_layer_head0;       // per text layer: capture head of its lowest alignment head
    int dtw_n_heads = 0, dtw_cap_rows = 0;  // alignment heads of the context; rows dtw_q holds per capture head
    DevBuf<float> dtw_q, dtw_out; DevBuf<int> dtw_heads_dev, dtw_req_dev; DevBuf<int64_t> dtw_req_out;
    bool pass_capture = false;              // the current pass has rows with a capture index (chain: k_dtw_capture; persistent kernel: generation 1)
    bool dtw_set_heads(const std::vector<std::pair<int, int>> & heads);   // (text layer, head) in the context's order; once, before any pass
    bool dtw_reserve(int n_rows);
    // alignment weights of several DTW passes in one launch: req = 4 ints per request (first capture index, slot, tokens, audio positions);
    // out[r] receives [heads][audio positions][tokens] of request r.  Then the warping paths of all of them on the device (DtwPaths):
    // path = 2 ints per request (audio positions of the window M, sot_len); tok[r] / time[r] receive request r's path (dtw_path's output)
    bool dtw_weights(const std::vector<int> & req, const std::vector<int> & path, std::vector<std::vector<float> *> & out,
                     std::vector<std::vector<int32_t> *> & tok, std::vector<std::vector<int32_t> *> & time);
    DtwPaths dtw_paths;
    bool use_mk = false;
    int  max_rows = 8;               // rows per decode pass: 64 with the persistent kernel, 8 with the chain
    int  n_sm = 0, mk_prefetch = 61;     // bit0: next-phase weights -> L2; bit2: K / V streams with L2 evict-first priority; bit4: logits one warp per weight tile
    DevBuf<MkLayer> mk_layers;
    DevBuf<unsigned long long> mk_bar;   // barrier words of the persistent kernel (mk_bar_words)
    unsigned long long mk_bar_total = 0, mk_bar_part[MK_MAX_PARTS] = {};   // arrivals so far at the grid's counter and at the partitions' counters
    int mk_parts = 4, mk_turns = 2;      // partitions of a pass of 32 rows or more; partitions that may stream cross K/V at the same time
    std::vector<uint32_t> cell_group; uint32_t cell_stamp = 0;   // host scratch: which row group appends a cell in the current pass
    bool mk_build_table();
    // WB200_MK_TRACE=<file>: per-phase clock stamps of CTA 0, averaged over all passes, written when the engine is destroyed
    DevBuf<long long> mk_trace; std::vector<double> mk_trace_sum, mk_fine; uint64_t mk_trace_n = 0; double mk_turn_clk = 0.0; std::string mk_trace_path; double sm_ghz = 1.0;
    void mk_trace_collect(int n_layer, bool logits);
    void mk_trace_dump();
    DevBuf<int>    dints, xcnt;      // packed per-step integers: tokens | pos | cells | slot | n_kv | rowinfo[2] | capture index | idx[...]
    DevBuf<uint32_t> samp_mask;      // static suppression bit mask of the on-device sampler
    uint64_t samp_mask_key = 0;
    // A decode pass runs in one of PASS_SLOTS slots: its pinned row table, its sampler output (device and pinned) and the events around it.
    // The pool keeps up to three passes in flight (a run-ahead pass, an ordinary pass behind it, the next run-ahead pass: wb_api.cpp,
    // Group::run), so the host may fill one slot's table while the passes of the others are queued or running.  Device workspaces stay
    // single: stream order serialises the passes.
    static constexpr int PASS_SLOTS = 3;
    struct PassSlot {
        int * hints = nullptr;       // pinned mirror of dints for this pass
        SampOut * hsamp = nullptr;   // pinned [max_rows][SAMP_MAX_DRAWS]
        cudaEvent_t ev0 = nullptr, ev1 = nullptr;   // around the pass; ev1 follows its device-to-host copy
        bool busy = false;           // enqueued and not yet waited for
        int n = 0, draw_stride = 1; bool any_logits = false;
    };
    PassSlot pslot[PASS_SLOTS];
    DevBuf<SampOut> dsamp;           // [PASS_SLOTS][max_rows][SAMP_MAX_DRAWS]
    SampOut * dsamp_of(int slot) const { return dsamp.p + (size_t) slot * max_rows * SAMP_MAX_DRAWS; }
    SampOut * hsamp = nullptr;       // = pslot[slot].hsamp of the pass being enqueued
    DevBuf<double> ddraws; double * hdraws = nullptr;   // uniforms of the categorical draws of a pass [max_rows][stride] (device / pinned)
    int draw_stride = 1;             // entries per row of dsamp / ddraws in the current pass
    int * hints = nullptr;           // = pslot[slot].hints of the pass being enqueued
    int cur_slot = 0;
    float * hlogits = nullptr;       // pinned [8][n_vocab]
    int ld_idx = 0;
    // CUDA graphs of one decode pass, keyed by (rows, logits?, n_keys); rebuilt when buffers move
    struct StepGraph { cudaGraphExec_t exec = nullptr; uint64_t launches = 0; int seen = 0; };
    std::map<uint64_t, StepGraph> graphs;
    bool use_graphs = true;
    void drop_graphs();

    // device-event timers of the last encode: [1]=conv (incl. window staging) [2]=encoder [3]=cross  ([0] unused: mel is FrontEnd)
    cudaEvent_t ev[8] = { nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr };   // [5],[6]: k_dtw_qk; [6],[7]: DTW paths
    float last_ms[4] = { 0, 0, 0, 0 };

    ~Engine();
    bool init(const Model * model, int cap_windows);
    bool set_cells(int n);           // private engine (one slot): (re)allocate the self-KV pool; contents are lost
    // change the number of slots and/or the self-KV cells per slot; cross-KV and self-KV contents of the surviving slots are preserved.
    // The caller guarantees that no pass is in flight (Group::grow_locked).
    bool resize(int new_cap, int new_cps);
  private:
    bool alloc_encoder_ws();
  public:

    // encode `n_win` windows in one batched pass; window w reads srcs[w].mel at frame srcs[w].seek and fills cross-KV slot srcs[w].slot
    bool encode(const EncSrc * srcs, int n_win, int n_ctx);

    // decode a batch (<= max_rows rows per pass internally).  idx lists: for row j, cells[j] is where its K/V go and
    // (kv_idx[j*ld .. +n_kv[j]]) the cells it attends to.  logits_out[j]: host buffer of n_vocab floats for rows with want_logits.
    // The slots of the rows of one pass must hold cross K/V of the same context length (slot_n_ctx); a pass that mixes them is an error.
    // the kernels of one pass (<= max_rows rows) on `st`; every row's slot holds cross K/V of n_audio_ctx positions, n_keys = pad256 of it
    bool decode_pass_enqueue(int n, bool any_logits, int n_keys, int n_audio_ctx, const SampCfg * samp, bool tok_indirect = false);
    // samp != nullptr: logits stay on the device; the filter + greedy pick run there (rowinfo: 2 ints per row, samp_out: host [n_rows])
    bool decode(const DecToken * rows, int n_rows, const int * cells, const int * kv_idx, int ld, const int * n_kv, float * const * logits_out,
                const SampCfg * samp = nullptr, const int * rowinfo = nullptr, SampOut * samp_out = nullptr,
                const double * draws = nullptr, int stride = 1,    // draws: [n_rows][stride] uniforms (rows asking for categorical draws, rowinfo bits 8-14); samp_out: [n_rows][stride]
                const int * cap_idx = nullptr);                    // per row: DTW capture index or -1 (null: no row is captured)
    // The two halves of one pass of `decode` (n_rows <= max_rows): enqueue it into a free slot (returned in *slot) without waiting, and wait
    // for it.  tok_src (may be null): per row -1, or the entry of dsamp (dsamp_of(s) + row of an earlier pass of slot s) whose token the row
    // takes; that pass precedes this one in stream order, so its output is complete and is read before this pass's sampler runs.
    // After pass_wait(slot) the pass's sampler output is pslot[slot].hsamp until the slot is enqueued again.
    bool pass_enqueue(const DecToken * rows, int n_rows, const int * cells, const int * kv_idx, int ld, const int * n_kv, const SampCfg * samp,
                      const int * rowinfo, const double * draws, int stride, const int * cap_idx, const int * tok_src, int * slot);
    bool pass_wait(int slot);
    bool set_samp_mask(uint64_t key, const std::vector<uint32_t> & bits);
};

} // namespace wb
