// wb_dtw.h -- DTW token timestamps (whisper_context_params.dtw_token_timestamps; src/whisper.cpp:8856-9167).
// The cross-attention weights of the alignment heads come from the device (one extra decoder pass over the window's text, batched with the
// other states of the pool, whose rows capture the alignment-head queries; k_dtw_qk), and so does the warping path (normalisation over
// the tokens, 7-tap median filter over time, mean over heads, dynamic time warping, backtrace; DtwPaths, wb_dtw_kernel.cuh).  dtw_path
// below is the host reference those kernels reproduce bit for bit; the assignment of the path to the tokens (dtw_assign) is host code.
#pragma once
#include <cstdint>
#include <utility>
#include <vector>
#include "../../include/whisper_b200.h"

namespace wb {

struct Segment;

// the (text layer, head) pairs of a context, in the order the reference concatenates them: by layer, inside a layer in table order
// (aheads_masks_init / get_alignment_heads_by_layer, src/whisper.cpp:1160-1273, 8856-8875).  false + last_error on invalid parameters.
bool dtw_resolve_heads(const whisper_context_params & cp, int n_text_layer, int n_head, std::vector<std::pair<int, int>> & out);

// qk: [n_heads][n_audio_ctx][n_tokens] softmax weights (tokens fastest).  Uses audio positions < n_audio_tokens and the tokens
// [sot_len, n_tokens - 1).  Returns the warping path as (token index, time index) pairs in path order.
void dtw_path(const float * qk, int n_tokens, int n_audio_ctx, int n_heads, int n_audio_tokens, int sot_len, int medfilt_width,
              std::vector<int32_t> & tok_idx, std::vector<int32_t> & time_idx);

// walk the path and stamp t_dtw on the text tokens (id < eot) of segments [i_segment, i_segment + n_segments) (src/whisper.cpp:9128-9153)
void dtw_assign(const std::vector<int32_t> & tok_idx, const std::vector<int32_t> & time_idx, int seek, int token_eot,
                std::vector<Segment> & segments, int i_segment, int n_segments);

} // namespace wb
