"""ctypes binding of the whisper.h C ABI (include/whisper_b200.h == reference include/whisper.h).

Host-side mirror of the reference interface for Python callers: the same by-value structs and entry points a
cgo / JNA / Ruby binding of whisper.cpp uses (bindings/go/whisper.go, bindings/java/.../WhisperCppJnaLibrary.java),
bound to libwhisper_b200.so.  `bind_whisper_api` works on ANY library exporting the whisper.h ABI, which is how the
tests drive the reference build and this engine through identical calls.
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("WB200_LIB") or os.path.join(HERE, "libwhisper_b200.so")      # WB200_LIB: A/B builds of the same ABI


# by-value ABI structs (whisper.h:116-151, 487-591)
class Aheads(C.Structure):
    _fields_ = [("n_heads", C.c_size_t), ("heads", C.c_void_p)]


class ContextParams(C.Structure):
    _fields_ = [("use_gpu", C.c_bool), ("flash_attn", C.c_bool), ("gpu_device", C.c_int),
                ("dtw_token_timestamps", C.c_bool), ("dtw_aheads_preset", C.c_int), ("dtw_n_top", C.c_int),
                ("dtw_aheads", Aheads), ("dtw_mem_size", C.c_size_t)]


class TokenData(C.Structure):
    _fields_ = [("id", C.c_int32), ("tid", C.c_int32), ("p", C.c_float), ("plog", C.c_float), ("pt", C.c_float),
                ("ptsum", C.c_float), ("t0", C.c_int64), ("t1", C.c_int64), ("t_dtw", C.c_int64), ("vlen", C.c_float)]


class VadParams(C.Structure):
    _fields_ = [("threshold", C.c_float), ("min_speech_duration_ms", C.c_int), ("min_silence_duration_ms", C.c_int),
                ("max_speech_duration_s", C.c_float), ("speech_pad_ms", C.c_int), ("samples_overlap", C.c_float)]


class Greedy(C.Structure):
    _fields_ = [("best_of", C.c_int)]


class BeamSearch(C.Structure):
    _fields_ = [("beam_size", C.c_int), ("patience", C.c_float)]


class FullParams(C.Structure):
    _fields_ = [("strategy", C.c_int), ("n_threads", C.c_int), ("n_max_text_ctx", C.c_int), ("offset_ms", C.c_int),
                ("duration_ms", C.c_int), ("translate", C.c_bool), ("no_context", C.c_bool), ("no_timestamps", C.c_bool),
                ("single_segment", C.c_bool), ("print_special", C.c_bool), ("print_progress", C.c_bool),
                ("print_realtime", C.c_bool), ("print_timestamps", C.c_bool), ("token_timestamps", C.c_bool),
                ("thold_pt", C.c_float), ("thold_ptsum", C.c_float), ("max_len", C.c_int), ("split_on_word", C.c_bool),
                ("max_tokens", C.c_int), ("debug_mode", C.c_bool), ("audio_ctx", C.c_int), ("tdrz_enable", C.c_bool),
                ("suppress_regex", C.c_char_p), ("initial_prompt", C.c_char_p), ("carry_initial_prompt", C.c_bool),
                ("prompt_tokens", C.POINTER(C.c_int32)), ("prompt_n_tokens", C.c_int), ("language", C.c_char_p),
                ("detect_language", C.c_bool), ("suppress_blank", C.c_bool), ("suppress_nst", C.c_bool),
                ("temperature", C.c_float), ("max_initial_ts", C.c_float), ("length_penalty", C.c_float),
                ("temperature_inc", C.c_float), ("entropy_thold", C.c_float), ("logprob_thold", C.c_float),
                ("no_speech_thold", C.c_float), ("greedy", Greedy), ("beam_search", BeamSearch),
                ("new_segment_callback", C.c_void_p), ("new_segment_callback_user_data", C.c_void_p),
                ("progress_callback", C.c_void_p), ("progress_callback_user_data", C.c_void_p),
                ("encoder_begin_callback", C.c_void_p), ("encoder_begin_callback_user_data", C.c_void_p),
                ("abort_callback", C.c_void_p), ("abort_callback_user_data", C.c_void_p),
                ("logits_filter_callback", C.c_void_p), ("logits_filter_callback_user_data", C.c_void_p),
                ("grammar_rules", C.c_void_p), ("n_grammar_rules", C.c_size_t), ("i_start_rule", C.c_size_t),
                ("grammar_penalty", C.c_float), ("vad", C.c_bool), ("vad_model_path", C.c_char_p),
                ("vad_params", VadParams)]


def bind_whisper_api(L):
    """declare the signatures of the whisper.h entry points used by the tests on either library"""
    vp = C.c_void_p
    L.whisper_context_default_params.restype = ContextParams
    L.whisper_full_default_params.restype = FullParams
    L.whisper_full_default_params.argtypes = [C.c_int]
    L.whisper_init_from_file_with_params.restype = vp
    L.whisper_init_from_file_with_params.argtypes = [C.c_char_p, ContextParams]
    L.whisper_init_from_file_with_params_no_state.restype = vp
    L.whisper_init_from_file_with_params_no_state.argtypes = [C.c_char_p, ContextParams]
    L.whisper_init_state.restype = vp
    L.whisper_init_state.argtypes = [vp]
    L.whisper_free.argtypes = [vp]
    L.whisper_free_state.argtypes = [vp]
    L.whisper_pcm_to_mel.argtypes = [vp, vp, C.c_int, C.c_int]
    L.whisper_set_mel.argtypes = [vp, vp, C.c_int, C.c_int]
    L.whisper_encode.argtypes = [vp, C.c_int, C.c_int]
    L.whisper_decode.argtypes = [vp, vp, C.c_int, C.c_int, C.c_int]
    L.whisper_get_logits.restype = C.POINTER(C.c_float)
    L.whisper_get_logits.argtypes = [vp]
    L.whisper_full.argtypes = [vp, FullParams, vp, C.c_int]
    L.whisper_full_with_state.argtypes = [vp, vp, FullParams, vp, C.c_int]
    L.whisper_full_parallel.argtypes = [vp, FullParams, vp, C.c_int, C.c_int]
    L.whisper_full_n_segments.argtypes = [vp]
    L.whisper_full_n_segments_from_state.argtypes = [vp]
    L.whisper_full_n_tokens.argtypes = [vp, C.c_int]
    L.whisper_full_n_tokens_from_state.argtypes = [vp, C.c_int]
    L.whisper_full_get_token_id.argtypes = [vp, C.c_int, C.c_int]
    L.whisper_full_get_token_id_from_state.argtypes = [vp, C.c_int, C.c_int]
    L.whisper_full_get_token_data.restype = TokenData
    L.whisper_full_get_token_data.argtypes = [vp, C.c_int, C.c_int]
    L.whisper_full_get_token_p.restype = C.c_float
    L.whisper_full_get_token_p.argtypes = [vp, C.c_int, C.c_int]
    L.whisper_full_get_segment_text.restype = C.c_char_p
    L.whisper_full_get_segment_text.argtypes = [vp, C.c_int]
    L.whisper_full_get_segment_text_from_state.restype = C.c_char_p
    L.whisper_full_get_segment_text_from_state.argtypes = [vp, C.c_int]
    for n in ("whisper_full_get_segment_t0", "whisper_full_get_segment_t1"):
        getattr(L, n).restype = C.c_int64
        getattr(L, n).argtypes = [vp, C.c_int]
        getattr(L, n + "_from_state").restype = C.c_int64
        getattr(L, n + "_from_state").argtypes = [vp, C.c_int]
    L.whisper_full_get_segment_no_speech_prob.restype = C.c_float
    L.whisper_full_get_segment_no_speech_prob.argtypes = [vp, C.c_int]
    L.whisper_tokenize.argtypes = [vp, C.c_char_p, C.POINTER(C.c_int32), C.c_int]
    L.whisper_token_to_str.restype = C.c_char_p
    L.whisper_token_to_str.argtypes = [vp, C.c_int32]
    L.whisper_lang_str.restype = C.c_char_p
    L.whisper_lang_str_full.restype = C.c_char_p
    L.whisper_lang_id.argtypes = [C.c_char_p]
    L.whisper_print_system_info.restype = C.c_char_p
    L.whisper_version.restype = C.c_char_p
    L.whisper_model_type_readable.restype = C.c_char_p
    L.whisper_model_type_readable.argtypes = [vp]
    L.whisper_get_timings.restype = C.POINTER(C.c_float * 5)
    L.whisper_get_timings.argtypes = [vp]
    for n in ("whisper_n_len", "whisper_n_vocab", "whisper_n_text_ctx", "whisper_n_audio_ctx", "whisper_is_multilingual",
              "whisper_model_n_vocab", "whisper_model_n_audio_ctx", "whisper_model_n_audio_state", "whisper_model_n_audio_head",
              "whisper_model_n_audio_layer", "whisper_model_n_text_ctx", "whisper_model_n_text_state", "whisper_model_n_text_head",
              "whisper_model_n_text_layer", "whisper_model_n_mels", "whisper_model_ftype", "whisper_model_type",
              "whisper_token_eot", "whisper_token_sot", "whisper_token_solm", "whisper_token_prev", "whisper_token_nosp",
              "whisper_token_not", "whisper_token_beg", "whisper_token_translate", "whisper_token_transcribe",
              "whisper_full_lang_id", "whisper_print_timings", "whisper_reset_timings"):
        getattr(L, n).argtypes = [vp]
    L.whisper_token_lang.argtypes = [vp, C.c_int]
    return L




class WhisperB200:
    """Minimal object wrapper: one context (weights on `gpu_device`) + its default state."""

    def __init__(self, model_path, gpu_device=0, lib_path=LIB_PATH, dtw_aheads_preset=None, dtw_n_top=-1):
        """dtw_aheads_preset: a whisper_alignment_heads_preset value (1 = the dtw_n_top last layers, 3.. = the tables of the released
        models) turns on DTW token timestamps (flash_attn off, as whisper.h requires): every text token gets a t_dtw, see tokens()"""
        if not os.path.exists(lib_path):
            raise RuntimeError(f"{lib_path} is missing: build it with __graft_entry__.build() (nvcc, sm_90a); there is no CPU fallback")
        self.L = bind_whisper_api(C.CDLL(lib_path))
        self.L.wb200_last_error.restype = C.c_char_p
        self.L.wb200_launch_count.restype = C.c_uint64
        self.L.wb200_ctx_state.restype = C.c_void_p
        self.L.wb200_ctx_state.argtypes = [C.c_void_p]
        cp = self.L.whisper_context_default_params()
        cp.gpu_device = gpu_device
        if dtw_aheads_preset is not None:
            cp.flash_attn = False; cp.dtw_token_timestamps = True; cp.dtw_aheads_preset = int(dtw_aheads_preset); cp.dtw_n_top = int(dtw_n_top)
        self.ctx = self.L.whisper_init_from_file_with_params(os.fsencode(model_path), cp)
        if not self.ctx:
            raise RuntimeError("whisper_init_from_file_with_params failed: " + self.L.wb200_last_error().decode())

    def close(self):
        if self.ctx:
            self.L.whisper_free(self.ctx)
            self.ctx = None

    def default_params(self, strategy=0):
        p = self.L.whisper_full_default_params(strategy)
        p.print_progress = False
        return p

    def full(self, pcm, params=None):
        """pcm: float32 mono 16 kHz (host).  Returns (rc, [(t0, t1, text, [token ids])...])"""
        pcm = np.ascontiguousarray(pcm, dtype=np.float32)
        p = params if params is not None else self.default_params()
        rc = self.L.whisper_full(self.ctx, p, pcm.ctypes.data_as(C.c_void_p), len(pcm))
        return rc, self.segments()

    def segments(self):
        L, ctx = self.L, self.ctx
        out = []
        for i in range(L.whisper_full_n_segments(ctx)):
            toks = [L.whisper_full_get_token_id(ctx, i, j) for j in range(L.whisper_full_n_tokens(ctx, i))]
            out.append((L.whisper_full_get_segment_t0(ctx, i), L.whisper_full_get_segment_t1(ctx, i),
                        L.whisper_full_get_segment_text(ctx, i).decode("utf-8", "replace"), toks))
        return out

    def tokens(self):
        """per segment, per token: (id, t0, t1, t_dtw) in centiseconds; t_dtw is -1 unless the context has DTW token timestamps"""
        L, ctx = self.L, self.ctx
        return [[(t.id, t.t0, t.t1, t.t_dtw) for t in (L.whisper_full_get_token_data(ctx, i, j) for j in range(L.whisper_full_n_tokens(ctx, i)))]
                for i in range(L.whisper_full_n_segments(ctx))]

    def launch_count(self):
        return int(self.L.wb200_launch_count())
