// wb_state.h -- host-side objects behind the opaque whisper_context / whisper_state handles.
// Mirrors the roles (not the code) of whisper_context / whisper_state / whisper_decoder / whisper_kv_cache in
// src/whisper.cpp:692-717, 783-820, 834-952.
#pragma once
#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <memory>
#include <mutex>
#include <random>
#include <string>
#include <utility>
#include <vector>
#include "../../include/whisper_b200.h"
#include "wb_engine.h"
#include "wb_grammar.h"
#include "wb_vad.h"

namespace wb {

constexpr int MAX_DECODERS = 8;               // WHISPER_MAX_DECODERS (src/whisper.cpp:142)

// Unified self-attention KV bookkeeping shared by all decoders of a state (src/whisper.cpp:692-717, 1019-1137).
// A cell holds one position of one or more sequences; beam-search reshuffles only touch this metadata.
struct KvCells {
    struct Cell { int pos = -1; uint32_t seqs = 0; };
    uint32_t head = 0, size = 0, n = 0;
    std::vector<Cell> cells;
    void reset(uint32_t n_cells) { size = n_cells; head = 0; n = 0; cells.assign(n_cells, Cell()); }
    void clear() { for (auto & c : cells) c = Cell(); head = 0; }
    bool find_slot(const int * pos, const int * seq, uint32_t n_tokens);
    int  cell_max() const;
    void seq_rm(int seq, int p0, int p1);
    void seq_cp(int src, int dst, int p0, int p1);
};

struct Sequence {
    std::vector<whisper_token_data> tokens;
    int    result_len = 0;
    double sum_logprobs_all = 0, sum_logprobs = 0, avg_logprobs = 0, entropy = 0, score = 0;
};

struct Decoder {
    Sequence sequence;
    int  i_batch = 0, seek_delta = 0;
    bool failed = false, completed = false, has_ts = false;
    std::vector<float> probs, logits, logprobs;
    std::vector<std::pair<double, int>> logits_id;
    std::mt19937 rng;
    Grammar grammar;                           // GBNF parse state of the tokens generated so far (params.grammar_rules)
    bool have_pending = false;                 // next token already chosen by the on-device sampler
    whisper_token_data pending;
    // beam search: the k categorical draws of the next step.  The uniforms are taken from `rng` when the decode is submitted (the same
    // numbers the reference consumes when it samples from those logits); the device returns the drawn tokens (pending_k), or -- when the
    // pass had to return full logits -- the host sampler uses the same uniforms (predrawn).
    bool have_pending_k = false;
    std::vector<whisper_token_data> pending_k;
    std::vector<double> predrawn;
};

struct Group;

struct Segment {
    int64_t t0 = 0, t1 = 0;
    std::string text;
    float no_speech_prob = 0;
    std::vector<whisper_token_data> tokens;
    bool speaker_turn_next = false;
};

} // namespace wb

struct whisper_state {
    whisper_state() : fe_own(new wb::FrontEnd()), fe(*fe_own) {}
    explicit whisper_state(std::unique_ptr<wb::FrontEnd> f) : fe_own(std::move(f)), fe(*fe_own) {}
    int64_t t_sample_us = 0, t_encode_us = 0, t_decode_us = 0, t_batchd_us = 0, t_prompt_us = 0, t_mel_us = 0;
    int32_t n_sample = 0, n_encode = 0, n_decode = 0, n_batchd = 0, n_prompt = 0, n_fail_p = 0, n_fail_h = 0;

    std::unique_ptr<wb::FrontEnd> fe_own;      // PCM + mel of this state (handed back to the context's pool by whisper_free_state)
    wb::FrontEnd & fe;                         // = *fe_own
    wb::Engine * eng = nullptr;                // the engine of the context's pool (null for result-only and engine-less test states)
    wb::Group * group = nullptr;               // non-null: this state lives in the context's pool; its encode/decode requests rendezvous
                                               // with those of the other states that are inside whisper_full* at the same time
    bool in_group_call = false;                // between Group::enter and Group::leave
    int cell_off = 0;                          // first self-KV cell of this state inside eng's pool
    wb::KvCells kv;
    int kv_self_n_dec = 1;
    wb::Decoder decoders[wb::MAX_DECODERS];
    std::vector<float> logits;                 // [n_tokens][n_vocab] of the last decode (rows flagged want_logits are valid)
    std::vector<wb::SampOut> samp_out;         // per row of the last decode when the on-device sampler was used: [rows][samp_stride]
    int samp_stride = 1;
    // What whisper.cpp:7190-7200 reads for the no-speech probability: ROW 0 of the logits buffer, log-sum-exp'ed against the maximum of
    // the WHOLE buffer (whisper_compute_logprobs takes max_element over all n_tokens rows, whisper.cpp:6160).  A decode resizes that
    // buffer to n_tokens rows (new rows are zero-filled) and refreshes only the rows it was asked logits for (whisper.cpp:2957-2963), so
    // row 0 is often stale.  `lrows` mirrors the buffer row by row as (max, sum exp(l - max), no-speech logit) so that the rule can be
    // followed on the device-sampler path too, where logits never reach the host; `row0_copy` holds row 0 itself when the host wrote it.
    struct LogitRow { float mx = 0.0f, sum = 0.0f, nosp = 0.0f; };
    std::vector<LogitRow> lrows;
    std::vector<float> row0_copy;
    bool row0_is_copy = false;
    std::vector<wb::Segment> result_all;
    std::vector<whisper_token> prompt_past0, prompt_past1;
    int   lang_id = 0;
    float no_speech_prob = 0.0f;
    int   exp_n_audio_ctx = 0;
    int   slot = 0;                            // cross-KV slot used by this state's decodes
    // experimental token-level timestamps (src/whisper.cpp:907-912, 8640-8820)
    int64_t t_beg = 0, t_last = 0; whisper_token tid_last = 0;
    std::vector<float> energy;                 // |PCM| averaged over +-32 samples
    // voice-activity detection in front of whisper_full (params.vad; src/whisper.cpp:923-934)
    struct VadFree { void operator()(whisper_vad_context * v) const { whisper_vad_free(v); } };
    std::unique_ptr<whisper_vad_context, VadFree> vad_context;
    wb::VadCut vad;                            // what the last whisper_full cut out, for mapping times back
    // TEST HOOK (wb200_dbg_scripted_context, tests/test_full_scripted_cpu.py): a state without an engine.  Mel / encode are no-ops and a
    // decode leaves all-zero logits, so the transcript is whatever the caller's logits_filter_callback scripts.  It computes nothing and
    // cannot be created through any whisper.h entry point.
    std::vector<float> dtw_qk_last;            // alignment-head weights of the last DTW pass [heads][n_audio_ctx][tokens] (wb200_dbg_last_dtw_qks)
    std::vector<int32_t> dtw_tok, dtw_time;    // its warping path, computed on the device from those weights (DtwPaths)
    int dtw_last_window[4] = {0, 0, 0, 0};     // its mel frames, sot_len, seek; DTW passes of the state so far (wb200_dbg_last_dtw_window)
    int dtw_last_shape[3] = {0, 0, 0};
    bool scripted = false;
    std::vector<int> dbg_tok, dbg_pos, dbg_seq; std::vector<int8_t> dbg_want;      // scripted states only: the last decode request (wb200_dbg_last_batch)
    std::vector<uint64_t> dbg_att;             // ... and per row a hash of the sorted positions it attends to (wb200_dbg_last_attended)
};

namespace wb {
// a further copy of the weights on another GPU of the box, with its own device pool (WB200_DEVICES, wb_api.cpp)
struct Replica { Model model; std::unique_ptr<Group> pool; };
}

struct whisper_context {
    int64_t t_load_us = 0, t_start_us = 0;
    whisper_context_params params;
    wb::Model model;
    wb::Vocab vocab;
    whisper_state * state = nullptr;
    std::string path_model;
    bool scripted = false;                     // TEST HOOK: see whisper_state::scripted
    std::vector<std::pair<int, int>> dtw_heads; // (text layer, head) of the alignment heads when params.dtw_token_timestamps survived init
    std::unique_ptr<wb::Group> pool;           // device pool shared by every state of this context (created with the first state)
    bool run_ahead = true;                     // TEST HOOK (wb200_dbg_run_ahead): Group::run_ahead of the pools created for this context
    // In-library multi-GPU: with WB200_DEVICES=all (or a list "0,1,..") a context loaded from a FILE keeps one replica of the weights per
    // listed GPU.  whisper_init_state places each new state on the GPU that holds the fewest, so whisper_full_parallel and concurrent
    // whisper_full_with_state callers spread over the box without any change on their side; every GPU batches its own states (no
    // collective, no data crosses GPUs: the chunks are independent -- src/whisper.cpp:7848-7869 semantics, N devices).
    std::vector<std::unique_ptr<wb::Replica>> replicas;
    std::mutex replicas_mu;
    ~whisper_context();
};

namespace wb {

// The device pool of a context and the lock-step batching of its states.  whisper.h allows concurrent whisper_full_with_state calls on
// DISTINCT states of one context (include/whisper.h:45-46), and whisper_full_parallel does exactly that (src/whisper.cpp:7848-7869).
// Every state created by whisper_init_state is a slot of this pool: one engine, one copy of the workspaces, a cross-KV slot and a range
// of self-KV cells per state.  Each calling thread runs the ordinary whisper_full_with_state control flow; its encode / decode requests
// block in submit() until all ACTIVE states (those inside a whisper_full* call) have one pending, then one of the threads executes them
// as a single batched device pass: one batched encoder pass for all windows, one decode launch for all live sequences (weights are read
// once per step).  A state that runs alone gets a 1-row pass immediately.
// request for the on-device logits filter + greedy pick of the rows of one decode call
struct SampReq { SampCfg cfg; uint64_t mask_key = 0; const std::vector<uint32_t> * mask_bits = nullptr; const int * rowinfo = nullptr;
                 const double * draws = nullptr; int stride = 1;      // beam search: [n_rows][stride] uniforms for the categorical draws; samp_out then holds `stride` entries per row
                 // run-ahead (Group::run): the member will submit the single-token step that follows the request's last row if the token
                 // sampled there is a text token, and that step's rowinfo will be next_rowinfo
                 bool next_step = false; int next_rowinfo[2] = { 0, 0 }; };

struct Group {
    Engine eng;
    bool scripted = false;                      // test hook: no engine, decodes leave zero logits
    const Model * model = nullptr;
    std::vector<std::pair<int, int>> dtw_heads; // alignment heads of the context (DTW token timestamps): the engine's capture table
    // ---- slots: one cross-KV slot + `cps` self-KV cells per state; the pool grows (contents preserved) while no pass is in flight
    int cap = 0, cps = 0;
    std::vector<uint8_t> slot_used;
    std::vector<std::unique_ptr<FrontEnd>> fe_cache;     // front ends of freed states (stream + PCM/mel buffers are reused)
    int n_registered = 0;                       // states attached
    std::unique_ptr<FrontEnd> take_fe();
    bool attach(whisper_state * st);            // whisper_init_state
    void detach(whisper_state * st);            // whisper_free_state
    bool ensure_cells(whisper_state * st, int cells);    // a state needs `cells` self-KV cells (n_decoders grew): kv.reset + pool relayout if needed
    // ---- rendezvous
    std::mutex mu;
    std::condition_variable cv;
    bool running = false;                       // a batch is executing (outside the lock)
    int n_active = 0;                           // states between enter() and leave()
    int64_t t_last_enter_us = 0;
    struct Req {
        int kind = 0;                           // 0 = encode, 1 = decode
        whisper_context * ctx = nullptr; whisper_state * st = nullptr;
        int seek = 0, n_ctx = 0;                // encode
        const int * tokens = nullptr, * pos = nullptr, * seq = nullptr; const int8_t * want = nullptr; int n = 0;   // decode
        const SampReq * samp = nullptr;
        int dtw_n_ctx = 0;                       // > 0: a DTW pass; capture its alignment-head queries and compute its weights over this many audio positions
        int dtw_sot_len = 0, dtw_n_frames = 0;   // DTW pass: tokens before the no-timestamps token, mel frames of the window (its path)
        const int * x_cells = nullptr, * x_idx = nullptr, * x_nkv = nullptr; int x_ld = 0;   // explicit self-KV cells / attended lists (relative to the state's range) instead of the KvCells bookkeeping: the ggml-backend plugin passes what the host's KQ_mask says
        bool taken = false;                      // (under mu) some thread took the batch that contains this request
        std::atomic<int> done{0};                // futex word: the member sleeps on its OWN request (no shared mutex to re-acquire on wake-up)
        bool ok = false; int64_t dt_us = 0;
    };
    std::vector<Req *> pending;
    // ---- run-ahead: after a pass of greedy, device-sampled rows the pool enqueues the next single-token step of every sequence that may
    // continue, with the token taken from the pass's sampler output on the device and every other input predicted on the host.  The next
    // batch takes the results of the rows whose real request equals the prediction; the others run in an ordinary pass.  A rejected row
    // is harmless: it wrote K/V only into the cell predicted for its own state, which no pass attends to before the pass that allocates
    // it writes it again, and that pass comes later in stream order.
    struct SpecRow {
        const whisper_state * st; int token, pos, seq, slot, cell, n_ctx, rowinfo[2];   // token: filled in when its source pass is waited for
        std::vector<int> idx;                    // attended cells
        int src_pass, src_row;                   // pass slot and row of the sampler output that holds the token
    };
    int spec_pass = -1;                         // engine pass slot of the queued run-ahead pass, -1: none
    uint64_t spec_mask_key = 0; SampCfg spec_cfg;
    std::vector<SpecRow> spec_rows;
    float spec_miss = 0.0f; int spec_idle = 0;  // share of recent run-ahead batches with a mispredicted row; batches since the last run-ahead pass
    bool run_ahead = true;                      // test hook (wb200_dbg_run_ahead): false keeps every batch on the lock-step path
    void spec_drop();                           // wait for the queued run-ahead pass and forget it (no batch is running)
    void enter(whisper_state * st);             // the state starts issuing requests (whisper_full_with_state, or one low-level call)
    void leave(whisper_state * st);
    void suspend(whisper_state * st);           // the state's thread is busy with a nested call on another state
    void resume(whisper_state * st);
    bool submit(Req & r);
    void run(std::vector<Req *> & batch);       // executes outside the lock
  private:
    void deactivate(whisper_state * st, bool clear_flag);
    bool grow_locked(std::unique_lock<std::mutex> & lk, int new_cap, int new_cps);
    int64_t grace_left_us() const;
};

// RAII around every whisper.h call that issues device work for a state: joins the rendezvous unless the state already has
// (whisper_full_parallel enters all its states up front).  A call made from INSIDE a callback of another active state on the same
// thread (legal with the reference: states are independent) suspends the outer state for its duration -- the outer state cannot
// submit anything while its thread is busy here, and the lock-step rendezvous must not wait for it.
struct GroupCall {
    whisper_state * st; bool entered = false; whisper_state * suspended = nullptr;
    explicit GroupCall(whisper_state * s);
    ~GroupCall();
    GroupCall(const GroupCall &) = delete; GroupCall & operator=(const GroupCall &) = delete;
};

int64_t time_us();
bool & tls_pcm_is_device();   // set by the batch driver: the next whisper_pcm_to_mel* `samples` pointer is a device pointer
// decode one batch through the engine with the reference's KV bookkeeping (whisper_decode_internal, whisper.cpp:2856-2986)
bool decode_batch(whisper_context & ctx, whisper_state & st, const int * tokens, const int * pos, const int * seq,
                  const int8_t * want, int n_tokens, const SampReq * samp = nullptr, int dtw_n_ctx = 0, int dtw_sot_len = 0, int dtw_n_frames = 0);
bool encode_window(whisper_context & ctx, whisper_state & st, int mel_offset);
}
