// wb_model.h -- the Whisper model as it lives on one GPU: hyper-parameters, vocabulary (host) and weights (HBM).
//
// File format: the legacy "ggml" container written by models/convert-pt-to-ggml.py:268-339 and read by
// whisper_model_load (src/whisper.cpp:1485-1962): magic, 11 x i32 hparams, mel filters, vocabulary, then a stream
// of { n_dims, name_len, ttype, ne[n_dims], name, raw data } records without padding.  Tensor names follow
// src/whisper-arch.h:42-109.
//
// HBM layout decisions (DESIGN.md section 3):
//   * 2-D weights keep their file quantisation; 32-value blocks are re-laid "planar" (wb_quant.cuh) so every access
//     is a 16-byte aligned vector load; K-quant super-blocks and F16 rows are kept verbatim.
//   * Matrices that consume the same activation are stacked along the output dimension so one launch covers them:
//     encoder/decoder self-attention [Wq;Wk] and Wv, decoder cross [Wk(l);...;Wv(l)...] over all text layers.
//   * conv weights (F16, ne = [3, ic, oc]) are re-ordered tap-major [3][oc][ic] so each tap is a K-major GEMM operand.
#pragma once
#include <map>
#include <string>
#include <vector>
#include "wb_common.h"
#include "wb_quant.cuh"

struct whisper_model_loader; // include/whisper_b200.h

namespace wb {

struct HParams {
    int32_t n_vocab = 51864, n_audio_ctx = 1500, n_audio_state = 384, n_audio_head = 6, n_audio_layer = 4;
    int32_t n_text_ctx = 448, n_text_state = 384, n_text_head = 6, n_text_layer = 4, n_mels = 80, ftype = 1;
    float eps = 1e-5f;
};

struct Vocab {                      // src/whisper.cpp:429-458
    int n_vocab = 51864;
    std::map<std::string, int32_t> token_to_id;
    std::map<int32_t, std::string> id_to_token;
    int32_t token_eot = 50256, token_sot = 50257, token_translate = 50357, token_transcribe = 50358,
            token_solm = 50359, token_prev = 50360, token_nosp = 50361, token_not = 50362, token_beg = 50363;
    bool is_multilingual() const { return n_vocab >= 51865; }
    int  num_languages()   const { return n_vocab - 51765 - (is_multilingual() ? 1 : 0); }
};

struct LNorm { const float * w = nullptr; const float * b = nullptr; };

struct EncLayerW {
    LNorm ln0, ln1;
    QMat  qk;  const float * qk_bias = nullptr;   // rows [0,d)=Wq (+bq), [d,2d)=Wk (no bias -> zeros)
    QMat  v;   const float * v_bias  = nullptr;
    QMat  o;   const float * o_bias  = nullptr;
    QMat  fc1; const float * fc1_bias = nullptr;
    QMat  fc2; const float * fc2_bias = nullptr;
};

struct DecLayerW {
    LNorm ln0, lnc, lnm;
    QMat  qkv; const float * qkv_bias = nullptr; const float * qkv_scale = nullptr; // [3d]: q,k scaled by 64^-1/4 (whisper.cpp:2558,2565)
    QMat  o;   const float * o_bias  = nullptr;
    QMat  cq;  const float * cq_bias = nullptr;
    QMat  co;  const float * co_bias = nullptr;
    QMat  fc1; const float * fc1_bias = nullptr;
    QMat  fc2; const float * fc2_bias = nullptr;
};

struct Model {
    HParams hp;
    int     wtype = WT_F16;          // type of every 2-D weight (src/whisper.cpp:1549-1559)
    int     mtype = 0;               // e_model (1 tiny .. 5 large)
    int     n_loaded = 0;            // 0 => weight-less test stub (src/whisper.cpp:1947-1948)
    int     device = 0;
    bool    dec_tm = false;          // decoder matrices + token embedding are in the tile-major layout (persistent decode kernel)
    int64_t t_load_us = 0;

    int n_filt_mel = 0, n_filt_fft = 0;
    std::vector<float> filters_host; // [n_mel][n_fft]
    const float * filters = nullptr; // device copy

    const float  * e_pe = nullptr;           // [n_audio_ctx][d] f32
    const __half * conv1_w = nullptr;        // [3][d][n_mels]
    const __half * conv2_w = nullptr;        // [3][d][d]
    const float  * conv1_b = nullptr, * conv2_b = nullptr;
    LNorm e_ln;
    const float * d_pe = nullptr;            // [n_text_ctx][d]
    QMat  d_te;                              // [n_vocab][d]  (embedding rows AND logits matrix, whisper.cpp:2525,2827)
    LNorm d_ln;
    std::vector<EncLayerW> enc;
    std::vector<DecLayerW> dec;
    QMat  cross_kv;                          // rows: [K(l=0..L-1) ; V(l=0..L-1)] each d rows
    const float * cross_bias = nullptr;      // [2*L*d]: zeros for K rows, bv for V rows
    const float * cross_scale = nullptr;     // [2*L*d]: 64^-1/4 for K rows (whisper.cpp:2304-2314), 1 for V rows

    std::vector<void *> allocs;              // every cudaMalloc owned by the model
    size_t bytes_weights = 0;

    ~Model();
};

// Parse + upload.  Returns false with set_error() text on failure; never throws.
bool model_load(whisper_model_loader * loader, Model & m, Vocab & v, int device);

} // namespace wb
