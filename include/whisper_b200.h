/*
 * whisper_b200.h -- C ABI of libwhisper_b200.so, the CUDA-native Whisper engine for the H100 (sm_90a).
 *
 * Binary-compatible with the reference interface `include/whisper.h` of ggml-org/whisper.cpp
 * @ 233fe1fc: same exported names, same by-value struct layouts, same return-code conventions,
 * so a program compiled against the reference header can be linked against this library
 * unchanged.  This file is an independent declaration of that ABI: each group below cites the
 * reference declaration it replaces (file:line in /root/reference) so parity can be checked.
 *
 * Only plain C types cross the boundary (pointers, sizes, POD structs, callbacks); no torch,
 * CUDA or ggml types appear here.  The three ggml typedefs the reference ABI leaks through
 * `#include "ggml.h"` (whisper.h:4) are re-declared with identical shapes in the first block.
 *
 * Implemented on the GPU hot path (SURVEY.md section 8): model load, log-mel, encode, decode,
 * whisper_full / _with_state / _parallel and all result getters.  Entry points of subsystems
 * that are out of scope for this engine (Silero VAD, OpenVINO, the ggml micro-benchmarks) are
 * exported and fail with the reference's own error codes -- see each comment.
 */
#ifndef WHISPER_B200_H
#define WHISPER_B200_H

#include <stdbool.h>
#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#  define WB_EXPORT __attribute__((visibility("default")))
#else
#  define WB_EXPORT
#endif

#ifdef __cplusplus
extern "C" {
#endif

/* ---- constants: whisper.h:33-36 ---------------------------------------------------------- */
enum {
    WB_SAMPLE_RATE = 16000, /* WHISPER_SAMPLE_RATE */
    WB_N_FFT       = 400,   /* WHISPER_N_FFT       */
    WB_HOP_LENGTH  = 160,   /* WHISPER_HOP_LENGTH  */
    WB_CHUNK_SIZE  = 30     /* WHISPER_CHUNK_SIZE  */
};

/* ---- types borrowed from ggml.h by the reference ABI --------------------------------------
 * ggml/include/ggml.h:640-647 (log levels), :712 (abort callback), :2840 (log callback)      */
#ifndef GGML_API /* when the real ggml.h is in scope its own definitions are used */
enum ggml_log_level {
    GGML_LOG_LEVEL_NONE = 0, GGML_LOG_LEVEL_DEBUG = 1, GGML_LOG_LEVEL_INFO = 2,
    GGML_LOG_LEVEL_WARN = 3, GGML_LOG_LEVEL_ERROR = 4, GGML_LOG_LEVEL_CONT = 5
};
typedef bool (*ggml_abort_callback)(void * data);
typedef void (*ggml_log_callback)(enum ggml_log_level level, const char * text, void * user_data);
#endif

/* ---- opaque handles and scalar typedefs: whisper.h:80-86 --------------------------------- */
struct whisper_context;   /* model weights (device resident, shared) + default state          */
struct whisper_state;     /* per-stream buffers: mel, KV caches, decoders, results            */
struct whisper_vad_context;
struct whisper_vad_segments;

typedef int32_t whisper_pos;
typedef int32_t whisper_token;
typedef int32_t whisper_seq_id;

/* ---- DTW alignment-head presets (accepted, unused: DTW is off under flash-attn,
 *      src/whisper.cpp:3720-3723): whisper.h:88-114 ------------------------------------------ */
enum whisper_alignment_heads_preset {
    WHISPER_AHEADS_NONE, WHISPER_AHEADS_N_TOP_MOST, WHISPER_AHEADS_CUSTOM,
    WHISPER_AHEADS_TINY_EN, WHISPER_AHEADS_TINY, WHISPER_AHEADS_BASE_EN, WHISPER_AHEADS_BASE,
    WHISPER_AHEADS_SMALL_EN, WHISPER_AHEADS_SMALL, WHISPER_AHEADS_MEDIUM_EN, WHISPER_AHEADS_MEDIUM,
    WHISPER_AHEADS_LARGE_V1, WHISPER_AHEADS_LARGE_V2, WHISPER_AHEADS_LARGE_V3,
    WHISPER_AHEADS_LARGE_V3_TURBO
};
typedef struct whisper_ahead  { int n_text_layer; int n_head; } whisper_ahead;
typedef struct whisper_aheads { size_t n_heads; const whisper_ahead * heads; } whisper_aheads;

/* ---- context creation parameters, passed BY VALUE: whisper.h:116-129 (48 bytes) ---------- */
struct whisper_context_params {
    bool  use_gpu;      /* must be true for this engine: there is no CPU fallback             */
    bool  flash_attn;   /* the fused attention layout (whisper.cpp:2147-2165) is the only one */
    int   gpu_device;   /* CUDA ordinal the weights and every state of this context live on   */
    bool  dtw_token_timestamps;
    enum whisper_alignment_heads_preset dtw_aheads_preset;
    int   dtw_n_top;
    struct whisper_aheads dtw_aheads;
    size_t dtw_mem_size;
};

/* ---- per-token result record: whisper.h:131-151 (56 bytes) ------------------------------- */
typedef struct whisper_token_data {
    whisper_token id;   /* sampled token                                                      */
    whisper_token tid;  /* most probable timestamp token at that step                         */
    float   p;          /* probability of `id`                                                */
    float   plog;       /* log-probability of `id`                                            */
    float   pt;         /* probability of `tid`                                               */
    float   ptsum;      /* total probability mass on timestamp tokens                         */
    int64_t t0, t1;     /* token-level times (only with token_timestamps)                     */
    int64_t t_dtw;      /* DTW time (unused here, kept -1)                                    */
    float   vlen;       /* voice length                                                       */
} whisper_token_data;

/* ---- custom model reader: whisper.h:153-159 ---------------------------------------------- */
typedef struct whisper_model_loader {
    void * context;
    size_t (*read )(void * ctx, void * output, size_t read_size);
    bool   (*eof  )(void * ctx);
    void   (*close)(void * ctx); /* always called once by init, on success and on failure     */
} whisper_model_loader;

/* ---- GBNF grammar elements (struct kept for layout; grammar sampling is out of scope and a
 *      non-empty grammar is ignored): whisper.h:162-190 -------------------------------------- */
enum whisper_gretype {
    WHISPER_GRETYPE_END = 0, WHISPER_GRETYPE_ALT = 1, WHISPER_GRETYPE_RULE_REF = 2,
    WHISPER_GRETYPE_CHAR = 3, WHISPER_GRETYPE_CHAR_NOT = 4, WHISPER_GRETYPE_CHAR_RNG_UPPER = 5,
    WHISPER_GRETYPE_CHAR_ALT = 6
};
typedef struct whisper_grammar_element { enum whisper_gretype type; uint32_t value; } whisper_grammar_element;

/* ---- VAD parameters (layout only): whisper.h:192-199 ------------------------------------- */
typedef struct whisper_vad_params {
    float threshold;
    int   min_speech_duration_ms;
    int   min_silence_duration_ms;
    float max_speech_duration_s;
    int   speech_pad_ms;
    float samples_overlap;
} whisper_vad_params;

/* ---- timing summary: whisper.h:438-444 --------------------------------------------------- */
struct whisper_timings { float sample_ms, encode_ms, decode_ms, batchd_ms, prompt_ms; };

/* ---- decoding strategy and callbacks: whisper.h:455-482 ---------------------------------- */
enum whisper_sampling_strategy { WHISPER_SAMPLING_GREEDY, WHISPER_SAMPLING_BEAM_SEARCH };

typedef void (*whisper_new_segment_callback)  (struct whisper_context *, struct whisper_state *, int n_new, void * user_data);
typedef void (*whisper_progress_callback)     (struct whisper_context *, struct whisper_state *, int progress, void * user_data);
typedef bool (*whisper_encoder_begin_callback)(struct whisper_context *, struct whisper_state *, void * user_data);
typedef void (*whisper_logits_filter_callback)(struct whisper_context *, struct whisper_state *,
                                               const whisper_token_data * tokens, int n_tokens,
                                               float * logits, void * user_data);

/* ---- whisper_full parameters, passed BY VALUE: whisper.h:487-591 (304 bytes).
 *      Field order is ABI; defaults follow src/whisper.cpp:5947-6053. ------------------------ */
struct whisper_full_params {
    enum whisper_sampling_strategy strategy;
    int  n_threads;
    int  n_max_text_ctx;
    int  offset_ms;
    int  duration_ms;

    bool translate;
    bool no_context;
    bool no_timestamps;
    bool single_segment;
    bool print_special;
    bool print_progress;
    bool print_realtime;
    bool print_timestamps;

    bool  token_timestamps;
    float thold_pt;
    float thold_ptsum;
    int   max_len;
    bool  split_on_word;
    int   max_tokens;

    bool debug_mode;
    int  audio_ctx;

    bool tdrz_enable;

    const char * suppress_regex;

    const char * initial_prompt;
    bool carry_initial_prompt;
    const whisper_token * prompt_tokens;
    int prompt_n_tokens;

    const char * language;
    bool detect_language;

    bool suppress_blank;
    bool suppress_nst;

    float temperature;
    float max_initial_ts;
    float length_penalty;

    float temperature_inc;
    float entropy_thold;
    float logprob_thold;
    float no_speech_thold;

    struct { int best_of; } greedy;
    struct { int beam_size; float patience; } beam_search;

    whisper_new_segment_callback   new_segment_callback;   void * new_segment_callback_user_data;
    whisper_progress_callback      progress_callback;      void * progress_callback_user_data;
    whisper_encoder_begin_callback encoder_begin_callback; void * encoder_begin_callback_user_data;
    ggml_abort_callback            abort_callback;         void * abort_callback_user_data;
    whisper_logits_filter_callback logits_filter_callback; void * logits_filter_callback_user_data;

    const whisper_grammar_element ** grammar_rules;
    size_t n_grammar_rules;
    size_t i_start_rule;
    float  grammar_penalty;

    bool         vad;
    const char * vad_model_path;
    whisper_vad_params vad_params;
};

struct whisper_vad_context_params { int n_threads; bool use_gpu; int gpu_device; }; /* whisper.h:703-707 */

/* =============================================================================================
 *  Lifecycle.  whisper.h:201-271.  Pointer-returning calls yield NULL on failure and never let
 *  a C++ exception escape (src/whisper.cpp:3735-3747).  The model file is the legacy "ggml"
 *  container (magic 0x67676d6c; src/whisper.cpp:1485-1962); weights are uploaded once to
 *  gpu_device and shared read-only by every state of the context.
 * ============================================================================================= */
WB_EXPORT const char * whisper_version(void);

WB_EXPORT struct whisper_context * whisper_init_from_file_with_params           (const char * path_model, struct whisper_context_params params);
WB_EXPORT struct whisper_context * whisper_init_from_buffer_with_params         (void * buffer, size_t buffer_size, struct whisper_context_params params);
WB_EXPORT struct whisper_context * whisper_init_with_params                     (struct whisper_model_loader * loader, struct whisper_context_params params);
WB_EXPORT struct whisper_context * whisper_init_from_file_with_params_no_state  (const char * path_model, struct whisper_context_params params);
WB_EXPORT struct whisper_context * whisper_init_from_buffer_with_params_no_state(void * buffer, size_t buffer_size, struct whisper_context_params params);
WB_EXPORT struct whisper_context * whisper_init_with_params_no_state            (struct whisper_model_loader * loader, struct whisper_context_params params);
/* deprecated default-parameter forms, whisper.h:216-239 */
WB_EXPORT struct whisper_context * whisper_init_from_file           (const char * path_model);
WB_EXPORT struct whisper_context * whisper_init_from_buffer         (void * buffer, size_t buffer_size);
WB_EXPORT struct whisper_context * whisper_init                     (struct whisper_model_loader * loader);
WB_EXPORT struct whisper_context * whisper_init_from_file_no_state  (const char * path_model);
WB_EXPORT struct whisper_context * whisper_init_from_buffer_no_state(void * buffer, size_t buffer_size);
WB_EXPORT struct whisper_context * whisper_init_no_state            (struct whisper_model_loader * loader);

WB_EXPORT struct whisper_state * whisper_init_state(struct whisper_context * ctx);

/* OpenVINO is not part of this engine: both return 1 exactly like a reference build without
 * WHISPER_USE_OPENVINO (src/whisper.cpp:3559-3616). */
WB_EXPORT int whisper_ctx_init_openvino_encoder_with_state(struct whisper_context * ctx, struct whisper_state * state,
                                                           const char * model_path, const char * device, const char * cache_dir);
WB_EXPORT int whisper_ctx_init_openvino_encoder(struct whisper_context * ctx, const char * model_path,
                                                const char * device, const char * cache_dir);

WB_EXPORT void whisper_free               (struct whisper_context * ctx);
WB_EXPORT void whisper_free_state         (struct whisper_state * state);
WB_EXPORT void whisper_free_params        (struct whisper_full_params * params);
WB_EXPORT void whisper_free_context_params(struct whisper_context_params * params);

/* =============================================================================================
 *  Low-level pipeline: PCM -> log-mel -> encoder -> decoder.  whisper.h:276-340.
 *  Return 0 on success.  whisper_decode* returns +1 on failure (src/whisper.cpp:3968).
 * ============================================================================================= */
WB_EXPORT int whisper_pcm_to_mel           (struct whisper_context * ctx, const float * samples, int n_samples, int n_threads);
WB_EXPORT int whisper_pcm_to_mel_with_state(struct whisper_context * ctx, struct whisper_state * state, const float * samples, int n_samples, int n_threads);
WB_EXPORT int whisper_set_mel              (struct whisper_context * ctx, const float * data, int n_len, int n_mel);
WB_EXPORT int whisper_set_mel_with_state   (struct whisper_context * ctx, struct whisper_state * state, const float * data, int n_len, int n_mel);
WB_EXPORT int whisper_encode               (struct whisper_context * ctx, int offset, int n_threads);
WB_EXPORT int whisper_encode_with_state    (struct whisper_context * ctx, struct whisper_state * state, int offset, int n_threads);
WB_EXPORT int whisper_decode               (struct whisper_context * ctx, const whisper_token * tokens, int n_tokens, int n_past, int n_threads);
WB_EXPORT int whisper_decode_with_state    (struct whisper_context * ctx, struct whisper_state * state, const whisper_token * tokens, int n_tokens, int n_past, int n_threads);

/* Logits of the last whisper_decode: [n_tokens][n_vocab] f32, owned by the state.  whisper.h:411-416 */
WB_EXPORT float * whisper_get_logits           (struct whisper_context * ctx);
WB_EXPORT float * whisper_get_logits_from_state(struct whisper_state * state);

/* =============================================================================================
 *  Tokenizer, languages, vocabulary and model getters.  whisper.h:347-435.
 * ============================================================================================= */
WB_EXPORT int whisper_tokenize   (struct whisper_context * ctx, const char * text, whisper_token * tokens, int n_max_tokens); /* <0: -needed */
WB_EXPORT int whisper_token_count(struct whisper_context * ctx, const char * text);

WB_EXPORT int          whisper_lang_max_id  (void);
WB_EXPORT int          whisper_lang_id      (const char * lang);   /* -1 when unknown */
WB_EXPORT const char * whisper_lang_str     (int id);
WB_EXPORT const char * whisper_lang_str_full(int id);
WB_EXPORT int whisper_lang_auto_detect           (struct whisper_context * ctx, int offset_ms, int n_threads, float * lang_probs);
WB_EXPORT int whisper_lang_auto_detect_with_state(struct whisper_context * ctx, struct whisper_state * state, int offset_ms, int n_threads, float * lang_probs);

WB_EXPORT int whisper_n_len           (struct whisper_context * ctx);
WB_EXPORT int whisper_n_len_from_state(struct whisper_state * state);
WB_EXPORT int whisper_n_vocab         (struct whisper_context * ctx);
WB_EXPORT int whisper_n_text_ctx      (struct whisper_context * ctx);
WB_EXPORT int whisper_n_audio_ctx     (struct whisper_context * ctx);
WB_EXPORT int whisper_is_multilingual (struct whisper_context * ctx);

WB_EXPORT int whisper_model_n_vocab      (struct whisper_context * ctx);
WB_EXPORT int whisper_model_n_audio_ctx  (struct whisper_context * ctx);
WB_EXPORT int whisper_model_n_audio_state(struct whisper_context * ctx);
WB_EXPORT int whisper_model_n_audio_head (struct whisper_context * ctx);
WB_EXPORT int whisper_model_n_audio_layer(struct whisper_context * ctx);
WB_EXPORT int whisper_model_n_text_ctx   (struct whisper_context * ctx);
WB_EXPORT int whisper_model_n_text_state (struct whisper_context * ctx);
WB_EXPORT int whisper_model_n_text_head  (struct whisper_context * ctx);
WB_EXPORT int whisper_model_n_text_layer (struct whisper_context * ctx);
WB_EXPORT int whisper_model_n_mels       (struct whisper_context * ctx);
WB_EXPORT int whisper_model_ftype        (struct whisper_context * ctx);
WB_EXPORT int whisper_model_type         (struct whisper_context * ctx);
WB_EXPORT const char * whisper_model_type_readable(struct whisper_context * ctx);

WB_EXPORT const char * whisper_token_to_str(struct whisper_context * ctx, whisper_token token);
WB_EXPORT whisper_token whisper_token_eot (struct whisper_context * ctx);
WB_EXPORT whisper_token whisper_token_sot (struct whisper_context * ctx);
WB_EXPORT whisper_token whisper_token_solm(struct whisper_context * ctx);
WB_EXPORT whisper_token whisper_token_prev(struct whisper_context * ctx);
WB_EXPORT whisper_token whisper_token_nosp(struct whisper_context * ctx);
WB_EXPORT whisper_token whisper_token_not (struct whisper_context * ctx);
WB_EXPORT whisper_token whisper_token_beg (struct whisper_context * ctx);
WB_EXPORT whisper_token whisper_token_lang(struct whisper_context * ctx, int lang_id);
WB_EXPORT whisper_token whisper_token_translate (struct whisper_context * ctx);
WB_EXPORT whisper_token whisper_token_transcribe(struct whisper_context * ctx);

/* =============================================================================================
 *  Timings / diagnostics.  whisper.h:445-450, 756-763.
 *  whisper_get_timings returns a heap object the caller owns (src/whisper.cpp:4271-4282).
 * ============================================================================================= */
WB_EXPORT struct whisper_timings * whisper_get_timings(struct whisper_context * ctx);
WB_EXPORT void whisper_print_timings(struct whisper_context * ctx);
WB_EXPORT void whisper_reset_timings(struct whisper_context * ctx);
WB_EXPORT const char * whisper_print_system_info(void);
WB_EXPORT void whisper_log_set(ggml_log_callback log_callback, void * user_data);
/* ggml CPU micro-benchmarks have no counterpart here: they report "not supported" and return 0 */
WB_EXPORT int          whisper_bench_memcpy          (int n_threads);
WB_EXPORT const char * whisper_bench_memcpy_str      (int n_threads);
WB_EXPORT int          whisper_bench_ggml_mul_mat    (int n_threads);
WB_EXPORT const char * whisper_bench_ggml_mul_mat_str(int n_threads);

/* =============================================================================================
 *  Full transcription.  whisper.h:594-626.  Return codes (src/whisper.cpp:6831-7788):
 *  0 ok, -1 VAD requested (unsupported here), -2 mel, -3 language detect, -4 too many decoders,
 *  -5 audio_ctx too large, -6 encode failed, -7 KV allocation, -8/-9 decode failed.
 *  whisper_full_parallel runs n_processors independent slices (src/whisper.cpp:7813-7941), each
 *  on its own state and CUDA stream, and merges the segments in slice order.
 * ============================================================================================= */
WB_EXPORT struct whisper_context_params * whisper_context_default_params_by_ref(void);
WB_EXPORT struct whisper_context_params   whisper_context_default_params       (void);
WB_EXPORT struct whisper_full_params * whisper_full_default_params_by_ref(enum whisper_sampling_strategy strategy);
WB_EXPORT struct whisper_full_params   whisper_full_default_params       (enum whisper_sampling_strategy strategy);

WB_EXPORT int whisper_full           (struct whisper_context * ctx, struct whisper_full_params params, const float * samples, int n_samples);
WB_EXPORT int whisper_full_with_state(struct whisper_context * ctx, struct whisper_state * state, struct whisper_full_params params, const float * samples, int n_samples);
WB_EXPORT int whisper_full_parallel  (struct whisper_context * ctx, struct whisper_full_params params, const float * samples, int n_samples, int n_processors);

/* ---- results: whisper.h:630-693, 766-767.  Strings stay valid until the next whisper_full*
 *      on the same state. ------------------------------------------------------------------- */
WB_EXPORT int whisper_full_n_segments           (struct whisper_context * ctx);
WB_EXPORT int whisper_full_n_segments_from_state(struct whisper_state * state);
WB_EXPORT int whisper_full_lang_id              (struct whisper_context * ctx);
WB_EXPORT int whisper_full_lang_id_from_state   (struct whisper_state * state);

WB_EXPORT int64_t whisper_full_get_segment_t0           (struct whisper_context * ctx, int i_segment);
WB_EXPORT int64_t whisper_full_get_segment_t0_from_state(struct whisper_state * state, int i_segment);
WB_EXPORT int64_t whisper_full_get_segment_t1           (struct whisper_context * ctx, int i_segment);
WB_EXPORT int64_t whisper_full_get_segment_t1_from_state(struct whisper_state * state, int i_segment);
WB_EXPORT bool whisper_full_get_segment_speaker_turn_next           (struct whisper_context * ctx, int i_segment);
WB_EXPORT bool whisper_full_get_segment_speaker_turn_next_from_state(struct whisper_state * state, int i_segment);
WB_EXPORT const char * whisper_full_get_segment_text           (struct whisper_context * ctx, int i_segment);
WB_EXPORT const char * whisper_full_get_segment_text_from_state(struct whisper_state * state, int i_segment);
WB_EXPORT float whisper_full_get_segment_no_speech_prob           (struct whisper_context * ctx, int i_segment);
WB_EXPORT float whisper_full_get_segment_no_speech_prob_from_state(struct whisper_state * state, int i_segment);

WB_EXPORT int whisper_full_n_tokens           (struct whisper_context * ctx, int i_segment);
WB_EXPORT int whisper_full_n_tokens_from_state(struct whisper_state * state, int i_segment);
WB_EXPORT const char * whisper_full_get_token_text           (struct whisper_context * ctx, int i_segment, int i_token);
WB_EXPORT const char * whisper_full_get_token_text_from_state(struct whisper_context * ctx, struct whisper_state * state, int i_segment, int i_token);
WB_EXPORT whisper_token whisper_full_get_token_id           (struct whisper_context * ctx, int i_segment, int i_token);
WB_EXPORT whisper_token whisper_full_get_token_id_from_state(struct whisper_state * state, int i_segment, int i_token);
WB_EXPORT whisper_token_data whisper_full_get_token_data           (struct whisper_context * ctx, int i_segment, int i_token);
WB_EXPORT whisper_token_data whisper_full_get_token_data_from_state(struct whisper_state * state, int i_segment, int i_token);
WB_EXPORT int64_t whisper_full_get_token_t0           (struct whisper_context * ctx, int i_segment, int i_token);
WB_EXPORT int64_t whisper_full_get_token_t0_from_state(struct whisper_state * state, int i_segment, int i_token);
WB_EXPORT int64_t whisper_full_get_token_t1           (struct whisper_context * ctx, int i_segment, int i_token);
WB_EXPORT int64_t whisper_full_get_token_t1_from_state(struct whisper_state * state, int i_segment, int i_token);
WB_EXPORT float whisper_full_get_token_p           (struct whisper_context * ctx, int i_segment, int i_token);
WB_EXPORT float whisper_full_get_token_p_from_state(struct whisper_state * state, int i_segment, int i_token);

/* VAD segment accessors: VAD never runs here, so the count is always 0 (whisper.h:688-693) */
WB_EXPORT int     whisper_full_n_vad_segments               (struct whisper_context * ctx);
WB_EXPORT int     whisper_full_n_vad_segments_from_state    (struct whisper_state * state);
WB_EXPORT int64_t whisper_full_get_vad_segment_t0           (struct whisper_context * ctx, int i);
WB_EXPORT int64_t whisper_full_get_vad_segment_t0_from_state(struct whisper_state * state, int i);
WB_EXPORT int64_t whisper_full_get_vad_segment_t1           (struct whisper_context * ctx, int i);
WB_EXPORT int64_t whisper_full_get_vad_segment_t1_from_state(struct whisper_state * state, int i);

/* =============================================================================================
 *  Silero VAD (whisper.h:699-750): OUT OF SCOPE (SURVEY.md section 2.1).  The symbols exist so
 *  that callers link; init returns NULL, detection returns false, accessors return 0.
 * ============================================================================================= */
WB_EXPORT struct whisper_vad_params         whisper_vad_default_params(void);
WB_EXPORT struct whisper_vad_context_params whisper_vad_default_context_params(void);
WB_EXPORT struct whisper_vad_context * whisper_vad_init_from_file_with_params(const char * path_model, struct whisper_vad_context_params params);
WB_EXPORT struct whisper_vad_context * whisper_vad_init_with_params(struct whisper_model_loader * loader, struct whisper_vad_context_params params);
WB_EXPORT bool    whisper_vad_detect_speech         (struct whisper_vad_context * vctx, const float * samples, int n_samples);
WB_EXPORT bool    whisper_vad_detect_speech_no_reset(struct whisper_vad_context * vctx, const float * samples, int n_samples);
WB_EXPORT void    whisper_vad_reset_state(struct whisper_vad_context * vctx);
WB_EXPORT int     whisper_vad_n_probs(struct whisper_vad_context * vctx);
WB_EXPORT float * whisper_vad_probs  (struct whisper_vad_context * vctx);
WB_EXPORT struct whisper_vad_segments * whisper_vad_segments_from_probs  (struct whisper_vad_context * vctx, struct whisper_vad_params params);
WB_EXPORT struct whisper_vad_segments * whisper_vad_segments_from_samples(struct whisper_vad_context * vctx, struct whisper_vad_params params, const float * samples, int n_samples);
WB_EXPORT int   whisper_vad_segments_n_segments    (struct whisper_vad_segments * segments);
WB_EXPORT float whisper_vad_segments_get_segment_t0(struct whisper_vad_segments * segments, int i_segment);
WB_EXPORT float whisper_vad_segments_get_segment_t1(struct whisper_vad_segments * segments, int i_segment);
WB_EXPORT void  whisper_vad_free_segments(struct whisper_vad_segments * segments);
WB_EXPORT void  whisper_vad_free         (struct whisper_vad_context * ctx);

/* =============================================================================================
 *  Engine extensions (no reference counterpart; prefix wb200_).  They expose device-side
 *  intermediates to the parity tests and the batched multi-chunk driver used by bench.py.
 * ============================================================================================= */
/* copy an intermediate of the last encode to host; returns element count, <0 on error.
 * which: 0 = mel [n_mel][n_len] f32, 1 = conv-stem output [n_ctx][n_state] f32 (token-major),
 *        2 = encoder output [n_ctx][n_state] f32, 3/4 = cross K/V [n_text_layer][1536][n_state] as f32 */
WB_EXPORT int64_t wb200_read_tensor(struct whisper_state * state, int which, float * out, int64_t cap);
/* run `n_chunks` independent PCM buffers through whisper_full_with_state semantics on ONE device in LOCK-STEP:
 * up to 64 member states share one engine, so every encoder pass / decode step serves all live chunks at once
 * (weights are read once per step).  Chunk i's segments land in the result-only state states_out[i] (free with
 * whisper_free_state).  _ex flags bit 0: samples[i] are DEVICE pointers (PCM already in HBM).  Returns 0 ok. */
WB_EXPORT int wb200_full_batch(struct whisper_context * ctx, struct whisper_full_params params,
                               const float * const * samples, const int * n_samples, int n_chunks,
                               struct whisper_state ** states_out);
WB_EXPORT int wb200_full_batch_ex(struct whisper_context * ctx, struct whisper_full_params params,
                                  const float * const * samples, const int * n_samples, int n_chunks,
                                  struct whisper_state ** states_out, int flags);
/* the default state owned by a context created with a *_with_params (non-_no_state) call; NULL otherwise */
WB_EXPORT struct whisper_state * wb200_ctx_state(struct whisper_context * ctx);
/* Decode with the self-attention KV cells spelled out by the caller (entry point of the ggml-backend plugin, plugin/ggml_b200_backend.cpp):
 * row j is stored in cell cells[j] of the state's range and attends to the cells idx[j*ld .. j*ld + nkv[j]); this is the information
 * whisper_build_graph_decoder puts into kv_head and KQ_mask (reference src/whisper.cpp:2580-2599, 2928-2938).  logits: [n_tokens][n_vocab]. */
WB_EXPORT int wb200_decode_explicit(struct whisper_context * ctx, struct whisper_state * state, const whisper_token * tokens, const int * pos, int n_tokens,
                                    const int * cells, const int * idx, int ld, const int * nkv, int n_cells_needed, float * logits);
/* In-library multi-GPU (environment WB200_DEVICES = "all" | "0,1,.." at whisper_init_from_file*): number of GPUs that hold a replica of
   the weights, and the GPU a state was placed on by whisper_init_state (the one with the fewest states). */
WB_EXPORT int wb200_n_devices(struct whisper_context * ctx);
WB_EXPORT int wb200_state_device(struct whisper_state * state);
/* stage PCM in HBM ahead of time: a following whisper_full_with_state(ctx, state, params, NULL, n_samples) (or
 * whisper_pcm_to_mel_with_state with samples == NULL) then starts from the device-resident samples (bench.py `value`) */
WB_EXPORT int wb200_pcm_upload(struct whisper_state * state, const float * samples, int n_samples);
/* per-kernel-class CUDA-event timing (classes: 0 wgmma GEMM, 1 decode GEMV, 2 decode attention, 3 other).
 * enable(1) clears the accumulators; collect() synchronises the device and fills four arrays of 4 entries:
 * summed duration [ms], launches, algorithmic bytes, algorithmic flops. */
WB_EXPORT void wb200_profile_enable(int on);
WB_EXPORT void wb200_profile_collect(double * ms4, uint64_t * launches4, double * bytes4, double * flops4);
/* coarse engine counters since load: [0] decode passes [1] decode rows [2] decode GPU ms [3] decode host ms [4] encode calls
 * [5] encode windows [6] encode GPU ms [7] CUDA-graph replays [8] alignment-weight (k_dtw_qk) GPU ms [9] DTW passes
 * [10] host DTW ms [11] device DTW path GPU ms [12] run-ahead decode rows launched [13] run-ahead rows whose results were taken */
WB_EXPORT void wb200_counters(double * out, int n);
/* bytes this library has copied host->device / device->host since load */
WB_EXPORT void wb200_traffic(uint64_t * h2d, uint64_t * d2h);
/* last CUDA error text for this thread ("" when none) */
WB_EXPORT const char * wb200_last_error(void);
/* number of CUDA kernels this library has launched since load (bench.py's gpu_launches) */
WB_EXPORT uint64_t wb200_launch_count(void);
/* device-event timers of the last encode on `state`, in ms: [0]=mel [1]=conv [2]=encoder [3]=cross */
WB_EXPORT int wb200_last_encode_ms(struct whisper_state * state, float * out4);

#ifdef __cplusplus
}
#endif
#endif /* WHISPER_B200_H */
