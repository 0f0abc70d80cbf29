"""ctypes binding of the C ABI in ``include/masr_b200.h`` (libmasr_b200.so, built in-tree by
``__graft_entry__.build()`` / ``masr_b200/build.py``).

There is deliberately no fallback: if the shared library is missing or a call fails, an
exception is raised (BASELINE.json north_star: "no CPU fallback")."""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmasr_b200.so")

OK = 0
EPI_BIAS, EPI_BIAS_SILU, EPI_BIAS_RELU, EPI_BIAS_GLU, EPI_BIAS_SCALE, EPI_RESIDUAL = range(6)
STATUS_GAIN_EXCEEDED = 1

_vp, _i, _i64, _f = C.c_void_p, C.c_int, C.c_int64, C.c_float


class LmTables(C.Structure):
    """``masr_lm_tables`` of include/masr_b200.h."""
    _fields_ = [("keys", _vp), ("vals", _vp), ("tok2lm", _vp), ("order", _i), ("bos", _i), ("eos", _i), ("vocab", _i),
                ("off", _i64 * 8), ("mask", _i64 * 8)]


_lmp = C.POINTER(LmTables)


class WordLmTables(C.Structure):
    """``masr_word_lm_tables`` of include/masr_b200.h."""
    _fields_ = [("keys", _vp), ("vals", _vp), ("lex_off", _vp), ("lex_tok", _vp), ("lex_next", _vp), ("lex_word", _vp),
                ("order", _i), ("bos", _i), ("eos", _i), ("vocab", _i), ("space", _i), ("root", _i), ("nodes", _i),
                ("dict_size", _i), ("off", _i64 * 8), ("mask", _i64 * 8)]


_wlmp = C.POINTER(WordLmTables)


class HotwordGraph(C.Structure):
    """``masr_hotword_graph`` of include/masr_b200.h."""
    _fields_ = [("arc_off", _vp), ("arc_tok", _vp), ("arc_next", _vp), ("fail", _vp), ("tail", _vp), ("leaf", _vp),
                ("acc", _vp), ("ta_acc", _vp), ("fin", _vp), ("nodes", _i)]


_hgp = C.POINTER(HotwordGraph)
LM_INFO_ORDER, LM_INFO_CHAR_BASED, LM_INFO_DICT_SIZE, LM_INFO_VOCAB, LM_INFO_KEY_WORDS, LM_INFO_VAL_FLOATS = range(6)
LM_INFO_READ, LM_INFO_KEPT, LM_INFO_SLOTS, LM_INFO_TABLE_BYTES = 8, 14, 20, 26
WORD_LM_INFO_NODES, WORD_LM_INFO_ARCS, WORD_LM_INFO_SPACE = 27, 28, 29

# name -> argtypes, exactly the declarations of include/masr_b200.h
SIGNATURES = {
    "masr_abi_version": [],
    "masr_check_device": [],
    "masr_stage_waves_f32": [_vp, _vp, _i, _vp, _vp, _i, _vp],
    "masr_resample_f32": [_vp, _vp, _vp, _i, _i, _vp, _i, _vp, _vp, _i64, _i, _vp],
    "masr_silero_vad_layout": [C.POINTER(_i64)],
    "masr_silero_vad_encode_f32": [_vp, _i64, _i, _vp, _vp, _vp, _vp],
    "masr_silero_vad_recur_f32": [_vp, _i64, _i, _vp, _vp, _vp, _vp],
    "masr_silero_vad_recur_slots_f32": [_vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp],
    "masr_fbank_workspace_bytes": [_i, _i64, C.POINTER(_i64)],
    "masr_wave_gain_f32": [_vp, _vp, _i, _i64, _f, _f, _vp, _vp, _vp, _vp],
    "masr_fbank_f32": [_vp, _vp, _vp, _i, _i, _vp, _vp, _vp],
    "masr_conv1_cmvn_relu_f32": [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp],
    "masr_conv2_s2_relu_f32": [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp],
    "masr_gemm_f32": [_vp, _i64, _vp, _vp, _vp, _i64, _vp, _i64, _i, _i, _i, _i, _f, _vp],
    "masr_gemm_tc_f16x2": [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _i64, _i, _i, _i, _i, _f, _vp],
    "masr_ffn_tc_f16x2": [_vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _i, _f, _vp],
    "masr_ctc_head_argmax_tc_f16x2": [_vp, _vp, _i64, _vp, _vp, _vp, _i, _i, _i, _vp, _i64, _vp, _vp, _vp],
    "masr_split_f16": [_vp, _vp, _vp, _i64, _vp],
    "masr_conv1_cmvn_relu_planes_f16": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp],
    "masr_conv2_tc_f16x2": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp],
    "masr_layernorm_f32": [_vp, _i64, _vp, _vp, _vp, _i64, _i, _i, _f, _vp],
    "masr_layernorm_split_f16": [_vp, _i64, _vp, _vp, _vp, _vp, _i64, _i, _i, _f, _vp],
    "masr_layernorm2_split_f16": [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _f, _vp],
    "masr_layernorm_ada_split_f16": [_vp, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _i, _f, _vp],
    "masr_affine_split_f16": [_vp, _vp, _vp, _vp, _vp, _i64, _i, _vp],
    "masr_dwconv_bn_silu_f32": [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _i, _i, _i, _i, _i, _vp],
    "masr_time_reduce_dw_split_f16": [_vp, _i64, _vp, _vp, _vp, _vp, _i64, _vp, _i, _i, _i, _i, _i, _vp],
    "masr_upsample2_add_f32": [_vp, _vp, _vp, _i64, _i64, _i, _i, _i, _vp],
    "masr_relpos_attention_f32": [_vp, _i64, _i64, _vp, _vp, _i64, _i64, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _i64, _i64,
                                  _vp, _vp, _i, _i, _i, _i, _vp],
    "masr_relpos_attention_tc": [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp, _i64,
                                 _i64, _vp, _vp, _i, _i, _i, _i, _vp],
    "masr_relpos_attention_tc5": [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp,
                                  _i64, _i64, _vp, _vp, _i, _i, _i, _i, _vp],
    "masr_dwconv_ln_silu_f32": [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _i, _i, _i, _i,
                                _i, _f, _vp],
    "masr_dwconv_ln_silu_strided_f32": [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _vp, _i, _i, _i,
                                        _i, _i, _i, _f, _vp],
    "masr_grouped_attention_f32": [_vp, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp],
    "masr_grouped_attention_cache_f32": [_vp, _i64, _i64, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i,
                                         _i, _i, _vp],
    "masr_avgpool2_time_f32": [_vp, _i64, _vp, _i64, _vp, _i, _i, _i, _vp],
    "masr_lstm_step_f32": [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _vp, _i, _i, _i, _i, _vp],
    "masr_lstm_seq_workspace_bytes": [_i, _i, C.POINTER(_i64)],
    "masr_lstm_seq_f32": [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _vp, _i, _i, _i, _i, _vp, _i64, _vp],
    "masr_gru_step_f32": [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _vp, _i, _i, _i, _i, _vp],
    "masr_gru_seq_f32": [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _vp, _i, _i, _i, _i, _vp, _i64, _vp],
    "masr_rnn_seq_tc_workspace_bytes": [_i, _i, C.POINTER(_i64)],
    "masr_rnn_tc_pack_f16x2": [_vp, _vp, _i, _i, _vp],
    "masr_lstm_seq_tc_f16x2": [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _vp, _i, _i, _i, _i, _vp, _i64, _vp],
    "masr_gru_seq_tc_f16x2": [_vp, _i64, _i64, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i, _vp, _i, _i, _i, _i, _vp, _i64, _vp],
    "masr_stream_append_rows": [_vp, _vp, _i64, _i64, _i, _vp, _vp, _i64, _i64, _vp, _vp, _i, _i, _vp],
    "masr_stream_shift_cache": [_vp, _vp, _i64, _i, _i, _vp, _i, _vp],
    "masr_ctc_frame_argmax_f32": [_vp, _i64, _i, _i, _vp, _vp, _vp, _i64, _vp],
    "masr_ctc_topk_f32": [_vp, _i64, _i, _i, _i, _f, _vp, _vp, _vp, _vp],
    "masr_ctc_prefix_beam_workspace": [_i, _i, C.POINTER(_i64), C.POINTER(_i64)],
    "masr_ctc_prefix_beam": [_vp, _vp, _vp, _i64, _vp, _i, _i, _i, _vp, _vp, _vp, _i64, _vp, _i64, _vp, _vp, _vp],
    "masr_ctc_prefix_beam_state_size": [C.POINTER(_i64), C.POINTER(_i64)],
    "masr_ctc_prefix_beam_frames": [_vp, _vp, _i64, _vp, _i64, _vp, _i, _vp, _i64, _vp],
    "masr_ctc_prefix_beam_stream": [_vp, _vp, _vp, _i64, _vp, _i, _i, _i, _vp, _vp, _vp, _i64, _vp, _vp, _i, _vp, _i64, _vp, _vp, _vp],
    "masr_ctc_greedy_collapse": [_vp, _vp, _i64, _vp, _i, _i, _vp, _i64, _vp, _vp, _vp, _vp],
    "masr_lm_load_arpa": [_vp, _vp, _i, C.POINTER(_vp)],
    "masr_lm_info": [_vp, C.POINTER(_i64)],
    "masr_lm_export": [_vp, _vp, _vp, _vp, _lmp],
    "masr_lm_free": [_vp],
    "masr_lm_score_f32": [_lmp, _vp, _vp, _i, _vp, _vp],
    "masr_ctc_topk_blank_f32": [_vp, _i64, _i, _i, _i, _f, _i, _vp, _vp, _vp, _vp, _vp],
    "masr_ctc_prefix_beam_lm": [_vp, _vp, _vp, _vp, _i64, _vp, _i, _i, _i, _lmp, _f, _f, _vp, _vp, _vp, _i64, _vp, _i64, _vp, _vp,
                                _vp, _vp],
    "masr_ctc_prefix_beam_lm_state_size": [C.POINTER(_i64), C.POINTER(_i64)],
    "masr_ctc_prefix_beam_lm_stream": [_vp, _vp, _vp, _vp, _i64, _vp, _i, _i, _i, _lmp, _f, _f, _vp, _vp, _vp, _i64, _vp, _vp, _i,
                                       _vp, _i64, _vp, _vp, _vp, _vp],
    "masr_ctc_prefix_beam_pool": [_vp, _vp, _vp, _i64, _vp, _i, _i, _i, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _i64, _vp, _vp,
                                  _vp],
    "masr_ctc_prefix_beam_lm_pool": [_vp, _vp, _vp, _vp, _i64, _vp, _i, _i, _i, _lmp, _f, _f, _vp, _vp, _vp, _i64, _vp, _vp, _vp,
                                     _vp, _i64, _vp, _vp, _vp, _vp],
    "masr_word_lm_load_arpa": [_vp, _vp, _i, C.POINTER(_vp)],
    "masr_word_lm_info": [_vp, C.POINTER(_i64)],
    "masr_word_lm_export": [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _wlmp],
    "masr_word_lm_score_f32": [_wlmp, _vp, _vp, _i, _vp, _vp],
    "masr_ctc_prefix_beam_wordlm": [_vp, _vp, _vp, _vp, _i64, _vp, _i, _i, _i, _wlmp, _f, _f, _vp, _vp, _vp, _i64, _vp, _i64, _vp,
                                    _vp, _vp, _vp],
    "masr_ctc_prefix_beam_wordlm_state_size": [C.POINTER(_i64), C.POINTER(_i64)],
    "masr_ctc_prefix_beam_wordlm_stream": [_vp, _vp, _vp, _vp, _i64, _vp, _i, _i, _i, _wlmp, _f, _f, _vp, _vp, _vp, _i64, _vp, _vp,
                                           _i, _vp, _i64, _vp, _vp, _vp, _vp],
    "masr_ctc_prefix_beam_wordlm_pool": [_vp, _vp, _vp, _vp, _i64, _vp, _i, _i, _i, _wlmp, _f, _f, _vp, _vp, _vp, _i64, _vp, _vp,
                                         _vp, _vp, _i64, _vp, _vp, _vp, _vp],
    "masr_ctc_prefix_beam_hot_state_size": [C.POINTER(_i64), C.POINTER(_i64)],
    "masr_ctc_prefix_beam_lm_hot_state_size": [C.POINTER(_i64), C.POINTER(_i64)],
    "masr_ctc_prefix_beam_wordlm_hot_state_size": [C.POINTER(_i64), C.POINTER(_i64)],
    "masr_ctc_prefix_beam_hot": [_vp, _vp, _vp, _i64, _vp, _i, _i, _i, _vp, _vp, _vp, _i64, _vp, _i64, _vp, _vp, _hgp, _vp, _vp],
    "masr_ctc_prefix_beam_hot_stream": [_vp, _vp, _vp, _i64, _vp, _i, _i, _i, _vp, _vp, _vp, _i64, _vp, _vp, _i, _vp, _i64, _vp,
                                        _vp, _hgp, _vp, _vp],
    "masr_ctc_prefix_beam_hot_pool": [_vp, _vp, _vp, _i64, _vp, _i, _i, _i, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _i64, _vp,
                                      _vp, _hgp, _vp, _vp],
    "masr_ctc_prefix_beam_lm_hot": [_vp, _vp, _vp, _vp, _i64, _vp, _i, _i, _i, _lmp, _f, _f, _vp, _vp, _vp, _i64, _vp, _i64, _vp,
                                    _vp, _vp, _hgp, _vp, _vp],
    "masr_ctc_prefix_beam_lm_hot_stream": [_vp, _vp, _vp, _vp, _i64, _vp, _i, _i, _i, _lmp, _f, _f, _vp, _vp, _vp, _i64, _vp, _vp,
                                           _i, _vp, _i64, _vp, _vp, _vp, _hgp, _vp, _vp],
    "masr_ctc_prefix_beam_lm_hot_pool": [_vp, _vp, _vp, _vp, _i64, _vp, _i, _i, _i, _lmp, _f, _f, _vp, _vp, _vp, _i64, _vp, _vp,
                                         _vp, _vp, _i64, _vp, _vp, _vp, _hgp, _vp, _vp],
    "masr_ctc_prefix_beam_wordlm_hot": [_vp, _vp, _vp, _vp, _i64, _vp, _i, _i, _i, _wlmp, _f, _f, _vp, _vp, _vp, _i64, _vp, _i64,
                                        _vp, _vp, _vp, _hgp, _vp, _vp],
    "masr_ctc_prefix_beam_wordlm_hot_stream": [_vp, _vp, _vp, _vp, _i64, _vp, _i, _i, _i, _wlmp, _f, _f, _vp, _vp, _vp, _i64, _vp,
                                               _vp, _i, _vp, _i64, _vp, _vp, _vp, _hgp, _vp, _vp],
    "masr_ctc_prefix_beam_wordlm_hot_pool": [_vp, _vp, _vp, _vp, _i64, _vp, _i, _i, _i, _wlmp, _f, _f, _vp, _vp, _vp, _i64, _vp,
                                             _vp, _vp, _vp, _i64, _vp, _vp, _vp, _hgp, _vp, _vp],
    "masr_ctc_prefix_beam_nbest": [_vp, _vp, _i64, _vp, _vp, _vp, _i, _i, _vp, _i64, _vp, _vp, _vp, _vp],
    "masr_ctc_prefix_beam_lm_nbest": [_vp, _vp, _i64, _vp, _vp, _vp, _i, _i, _lmp, _f, _f, _vp, _i64, _vp, _vp, _vp, _vp,
                                      _vp],
    "masr_ctc_prefix_beam_wordlm_nbest": [_vp, _vp, _i64, _vp, _vp, _vp, _i, _i, _wlmp, _f, _f, _vp, _i64, _vp, _vp, _vp,
                                          _vp, _vp],
    "masr_ctc_prefix_beam_hot_nbest": [_vp, _vp, _i64, _vp, _vp, _vp, _i, _i, _vp, _i64, _vp, _vp, _vp, _hgp, _vp, _vp],
    "masr_ctc_prefix_beam_lm_hot_nbest": [_vp, _vp, _i64, _vp, _vp, _vp, _i, _i, _lmp, _f, _f, _vp, _i64, _vp, _vp, _vp,
                                          _vp, _hgp, _vp, _vp],
    "masr_ctc_prefix_beam_wordlm_hot_nbest": [_vp, _vp, _i64, _vp, _vp, _vp, _i, _i, _wlmp, _f, _f, _vp, _i64, _vp, _vp,
                                              _vp, _vp, _hgp, _vp, _vp],
}


class MasrB200Error(RuntimeError):
    pass


_lib: Optional[C.CDLL] = None


def load() -> C.CDLL:
    """Load the shared library and declare every prototype.  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise MasrB200Error(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). masr_b200 has no CPU or PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    lib.masr_last_error.restype = C.c_char_p
    lib.masr_last_error.argtypes = []
    for name, argtypes in SIGNATURES.items():
        fn = getattr(lib, name)            # AttributeError here == header/library mismatch
        fn.argtypes = argtypes
        fn.restype = C.c_int
    _lib = lib
    return lib


def last_error() -> str:
    return load().masr_last_error().decode("utf-8", "replace")


def check(rc: int, what: str):
    if rc != OK:
        raise MasrB200Error(f"{what} failed (code {rc}): {last_error()}")


def call(name: str, *args):
    """Invoke an ABI function and raise on a non-zero status."""
    check(getattr(load(), name)(*args), name)
