"""ctypes binding of libspeech_b200.so (the C ABI declared in include/speech_b200.h).

There is NO fallback: if the shared library is missing, or a call returns a non-zero status, a
RuntimeError is raised.  The product path never routes through oracle/ or a CPU implementation.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libspeech_b200.so")

_c_int = ctypes.c_int
_c_ll = ctypes.c_longlong
_c_sz = ctypes.c_size_t
_vp = ctypes.c_void_p
_fl = ctypes.c_float


class SbNgramLm(ctypes.Structure):
    """struct SbNgramLm of include/speech_b200.h: device tables of an n-gram LM"""
    _fields_ = [("keys", _vp), ("vals", _vp), ("logp", _vp), ("bow", _vp), ("tok", _vp),
                ("cap", _c_int), ("order", _c_int), ("num_classes", _c_int), ("bos", _c_int),
                ("blank", _c_int),
                ("lm_upper", ctypes.c_double), ("lm_abs", ctypes.c_double)]


class SbWordLm(ctypes.Structure):
    """struct SbWordLm of include/speech_b200.h: device tables of a word n-gram LM and lexicon"""
    _fields_ = [("ngram", SbNgramLm), ("lex_keys", _vp), ("lex_vals", _vp), ("lex_word", _vp),
                ("lex_cap", _c_int), ("num_words", _c_int), ("has_unk", _c_int),
                ("num_classes", _c_int), ("blank", _c_int), ("delimiter", _c_int)]


_lmp = ctypes.POINTER(SbNgramLm)
_wlmp = ctypes.POINTER(SbWordLm)
_db = ctypes.c_double

# name -> (restype, argtypes): every symbol include/speech_b200.h declares
SIGNATURES = {
    "sb_version": (_c_int, []),
    "sb_status_string": (ctypes.c_char_p, [_c_int]),
    "sb_device_info": (_c_int, [_vp, _vp, _vp, _vp]),
    "sb_ctc_workspace_size": (_c_int, [_c_int, _c_int, _c_int, _c_int, ctypes.POINTER(_c_sz)]),
    "sb_ctc_fwd_bwd": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _c_int, _c_int, _c_int, _c_int,
                                _c_int, _vp, _vp, _c_sz, _vp]),
    "sb_ctc_compact_workspace_size": (_c_int, [_c_int, _c_int, _c_int, _c_int,
                                               ctypes.POINTER(_c_sz)]),
    "sb_ctc_fwd_bwd_compact": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _c_int, _c_int, _c_int,
                                        _c_int, _c_int, _vp, _vp, _c_sz, _vp]),
    "sb_ctc_viterbi_workspace_size": (_c_int, [_c_int, _c_int, _c_int, _c_int,
                                               ctypes.POINTER(_c_sz)]),
    "sb_ctc_viterbi": (_c_int, [_vp, _vp, _vp, _vp, _vp, _c_int, _c_int, _c_int, _c_int, _c_int,
                                _vp, _vp, _vp, _c_sz, _vp]),
    "sb_gemm_bf16_tn": (_c_int, [_vp, _c_ll, _vp, _c_ll, _vp, _c_ll, _vp, _c_int, _c_int, _c_int,
                                 _c_int, _c_int, _c_int, _c_int, _c_int, _vp]),
    "sb_ctc_prefix_beam_workspace_size": (_c_int, [_c_int, _c_int, _c_int, ctypes.POINTER(_c_sz)]),
    "sb_ctc_prefix_beam": (_c_int, [_vp, _vp, _c_int, _c_int, _c_int, _c_int, _c_int, _vp, _vp, _vp,
                                    _vp, _c_sz, _vp]),
    "sb_ctc_prefix_beam_shortlist": (_c_int, [_vp, _vp, _c_int, _c_int, _c_int, _c_int, _c_int,
                                              _vp, _vp, _vp, _vp, _c_sz, _vp]),
    "sb_ctc_prefix_beam_lm_workspace_size": (_c_int, [_c_int, _c_int, _c_int, _c_int,
                                                      ctypes.POINTER(_c_sz)]),
    "sb_ctc_prefix_beam_lm": (_c_int, [_vp, _vp, _c_int, _c_int, _c_int, _c_int, _c_int, _lmp, _db,
                                       _db, _vp, _vp, _vp, _vp, _c_sz, _vp]),
    "sb_ctc_prefix_beam_lm_shortlist": (_c_int, [_vp, _vp, _c_int, _c_int, _c_int, _c_int, _c_int,
                                                 _lmp, _db, _db, _vp, _vp, _vp, _vp, _c_sz, _vp]),
    "sb_debug_ctc_lm_rescans": (_c_int, [ctypes.POINTER(ctypes.c_ulonglong)]),
    "sb_ctc_stream_state_size": (_c_int, [_c_int, _c_int, _c_int, _c_int, ctypes.POINTER(_c_sz)]),
    "sb_ctc_stream_workspace_size": (_c_int, [_c_int, _c_int, _c_int, ctypes.POINTER(_c_sz)]),
    "sb_ctc_stream_reset": (_c_int, [_vp, _c_int, _c_int, _c_int, _c_int, _c_int, _vp]),
    "sb_ctc_stream_step": (_c_int, [_vp, _vp, _c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _vp,
                                    _vp, _c_sz, _vp]),
    "sb_ctc_stream_step_shortlist": (_c_int, [_vp, _vp, _c_int, _c_int, _c_int, _c_int, _c_int,
                                              _c_int, _vp, _vp, _c_sz, _vp]),
    "sb_ctc_stream_step_lm": (_c_int, [_vp, _vp, _c_int, _c_int, _c_int, _c_int, _c_int, _lmp, _db,
                                       _db, _c_int, _vp, _vp, _c_sz, _vp]),
    "sb_ctc_stream_step_lm_shortlist": (_c_int, [_vp, _vp, _c_int, _c_int, _c_int, _c_int, _c_int,
                                                 _lmp, _db, _db, _c_int, _vp, _vp, _c_sz, _vp]),
    "sb_ctc_stream_best": (_c_int, [_vp, _c_int, _c_int, _c_int, _vp, _vp, _vp, _vp, _vp]),
    "sb_ctc_stream_nbest": (_c_int, [_vp, _c_int, _c_int, _c_int, _vp, _vp, _vp, _vp, _vp]),
    "sb_ctc_prefix_beam_wordlm": (_c_int, [_vp, _vp, _c_int, _c_int, _c_int, _c_int, _c_int,
                                           _wlmp, _db, _db, _db, _vp, _vp, _vp, _vp, _c_sz, _vp]),
    "sb_ctc_prefix_beam_wordlm_shortlist": (_c_int, [_vp, _vp, _c_int, _c_int, _c_int, _c_int,
                                                     _c_int, _wlmp, _db, _db, _db, _vp, _vp, _vp,
                                                     _vp, _c_sz, _vp]),
    "sb_ctc_stream_step_wordlm": (_c_int, [_vp, _vp, _c_int, _c_int, _c_int, _c_int, _c_int,
                                           _wlmp, _db, _db, _db, _c_int, _vp, _vp, _c_sz, _vp]),
    "sb_ctc_stream_step_wordlm_shortlist": (_c_int, [_vp, _vp, _c_int, _c_int, _c_int, _c_int,
                                                     _c_int, _wlmp, _db, _db, _db, _c_int, _vp,
                                                     _vp, _c_sz, _vp]),
    "sb_ctc_stream_best_wordlm": (_c_int, [_vp, _c_int, _c_int, _c_int, _wlmp, _db, _db, _db,
                                           _vp, _vp, _vp, _vp, _vp]),
    "sb_conv_im2col": (_c_int, [_vp, _vp, _fl, _vp, _c_int, _c_int, _c_int, _c_int, _c_int, _c_int,
                                _c_int, _c_int, _c_int, _vp]),
    "sb_conv_relu_to_bct": (_c_int, [_vp, _vp, _fl, _vp, _c_int, _c_int, _c_int, _c_int, _vp]),
    "sb_conv_dtop": (_c_int, [_vp, _vp, _vp, _fl, _vp, _vp, _c_int, _c_int, _c_int, _c_int, _vp]),
    "sb_conv_col2im_relu": (_c_int, [_vp, _c_ll, _vp, _vp, _fl, _vp, _vp, _c_int, _c_int, _c_int,
                                     _c_int, _c_int, _c_int, _c_int, _vp]),
    "sb_conv_direct_ok": (_c_int, [_c_int] * 6),
    "sb_conv_fwd_direct": (_c_int, [_vp, _vp, _fl, _vp, _c_int, _vp, _vp] + [_c_int] * 8 + [_vp]),
    "sb_conv_dgrad_direct": (_c_int, [_vp, _vp, _c_int, _vp, _vp, _fl, _vp, _vp] + [_c_int] * 8
                             + [_vp]),
    "sb_conv_wgrad_direct": (_c_int, [_vp, _vp, _fl, _vp, _vp] + [_c_int] * 8 + [_vp]),
    "sb_sumsq_workspace_size": (_c_int, [ctypes.POINTER(_c_sz)]),
    "sb_sumsq": (_c_int, [_vp, _c_ll, _vp, _vp, _vp]),
    "sb_sgd_clip_step": (_c_int, [_vp, _vp, _vp, _vp, _c_ll, _vp, _fl, _fl, _fl, _vp]),
    "sb_s2s_workspace_size": (_c_int, [_c_int, _c_int, _c_int, ctypes.POINTER(_c_sz)]),
    "sb_s2s_cell_fwd": (_c_int, [_vp, _vp, _c_int, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                 _c_int, _c_int, _vp]),
    "sb_s2s_attn_fwd": (_c_int, [_vp, _c_int, _vp, _vp, _vp, _vp, _vp, _fl, _c_int, _c_int, _c_int,
                                 _c_int, _c_int, _vp, _vp, _vp, _vp, _c_int, _vp, _c_ll, _vp, _vp,
                                 _vp, _c_int, _c_int, _vp, _c_int, _vp, _vp, _vp, _c_sz, _vp]),
    "sb_s2s_dout": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _c_ll, _c_int, _c_int, _vp]),
    "sb_s2s_attn_bwd": (_c_int, [_vp] * 22 + [_c_int] * 5 + [_vp, _vp, _c_sz, _vp]),
    "sb_s2s_cell_bwd": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _c_int, _c_int, _vp]),
    "sb_s2s_check_done": (_c_int, [_vp, _c_int, _vp, _vp, _c_int, _vp]),
    "sb_s2s_score_tokens": (_c_int, [_vp, _c_ll, _c_int, _vp, _c_int, _vp, _c_int, _c_int, _vp,
                                     _vp]),
    "sb_s2s_beam_state_size": (_c_int, [ctypes.POINTER(_c_sz)]),
    "sb_s2s_beam_init": (_c_int, [_vp, _vp, _vp, _c_int, _vp]),
    "sb_s2s_beam_select": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _c_int, _c_int, _c_int,
                                    _c_int, _c_int, _c_int, _c_int, _vp]),
    "sb_s2s_beam_gather": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _c_int, _c_int, _c_int,
                                    _vp]),
    "sb_s2s_beam_init_batch": (_c_int, [_vp, _vp, _c_int, _vp, _c_int, _c_int, _vp, _c_int, _vp]),
    "sb_s2s_beam_select_batch": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _c_int, _c_int,
                                          _c_int, _c_int, _c_int, _c_int, _c_int, _vp, _c_int,
                                          _vp]),
    "sb_s2s_beam_gather_batch": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _c_int, _c_int,
                                          _c_int, _c_int, _vp]),
    "sb_s2s_fc_fused": (_c_int, [_c_int, _c_int]),
    "sb_s2s_fc_workspace_size": (_c_int, [_c_ll, _c_int, ctypes.POINTER(_c_sz)]),
    "sb_s2s_fc_rows": (_c_int, [_vp, _vp, _vp, _vp, _c_ll, _c_int, _c_int, _vp, _c_int, _c_ll,
                                _c_ll, _vp, _vp, _c_int, _c_int, _vp, _c_int, _vp, _vp, _c_sz,
                                _vp]),
    "sb_s2s_fc_logp": (_c_int, [_vp, _c_int, _c_ll, _c_ll, _vp, _c_ll, _c_int, _vp, _vp, _c_sz,
                                _vp]),
    "sb_s2s_beam_select_fits": (_c_int, [_c_int, _c_int]),
    "sb_s2s_beam_split_workspace_size": (_c_int, [_c_int, _c_int, ctypes.POINTER(_c_sz)]),
    "sb_s2s_beam_select_split": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _c_int, _c_int,
                                          _c_int, _c_int, _c_int, _c_int, _c_int, _vp, _c_sz,
                                          _vp]),
    "sb_s2s_beam_split_workspace_size_batch": (_c_int, [_c_int, _c_int, _c_int,
                                                        ctypes.POINTER(_c_sz)]),
    "sb_s2s_beam_select_split_batch": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _c_int, _c_int,
                                                _c_int, _c_int, _c_int, _c_int, _c_int, _vp,
                                                _c_int, _vp, _c_sz, _vp]),
    "sb_s2s_beam_select_lm_batch": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _c_int, _c_int,
                                             _c_int, _c_int, _c_int, _c_int, _c_int, _vp, _c_int,
                                             _lmp, _db, _db, _vp]),
    "sb_s2s_beam_select_split_lm_batch": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _c_int,
                                                   _c_int, _c_int, _c_int, _c_int, _c_int, _c_int,
                                                   _vp, _c_int, _vp, _c_sz, _lmp, _db, _db, _vp]),
    "sb_s2s_beam_select_wordlm_batch": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _c_int,
                                                 _c_int, _c_int, _c_int, _c_int, _c_int, _c_int,
                                                 _vp, _c_int, _wlmp, _db, _db, _db, _vp, _vp]),
    "sb_s2s_beam_select_split_wordlm_batch": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _c_int,
                                                       _c_int, _c_int, _c_int, _c_int, _c_int,
                                                       _c_int, _vp, _c_int, _vp, _c_sz, _wlmp,
                                                       _db, _db, _db, _vp, _vp]),
    "sb_s2s_ctc_state_size": (_c_int, [_c_int, _c_int, _c_int, _c_int, ctypes.POINTER(_c_sz)]),
    "sb_s2s_ctc_init": (_c_int, [_vp, _vp, _vp, _c_sz, _c_int, _c_int, _c_int, _c_int, _c_int,
                                 _c_int, _db, _c_int, _vp]),
    "sb_s2s_ctc_candidates": (_c_int, [_vp, _vp, _vp, _vp, _vp, _c_int, _vp, _c_sz, _c_int,
                                       _c_int, _c_int, _c_int, _c_int, _c_int, _db, _c_int, _vp,
                                       _c_int, _lmp, _db, _db, _vp]),
    "sb_s2s_ctc_candidates_wordlm": (_c_int, [_vp, _vp, _vp, _vp, _vp, _c_int, _vp, _c_sz,
                                              _c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _db,
                                              _c_int, _vp, _c_int, _wlmp, _db, _db, _db, _vp,
                                              _vp]),
    "sb_s2s_ctc_select_batch": (_c_int, [_vp, _vp, _vp, _c_sz, _vp, _vp, _vp, _vp, _vp, _vp,
                                         _c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _db,
                                         _c_int, _c_int, _c_int, _c_int, _vp, _c_int, _vp]),
    "sb_rnnt_workspace_size": (_c_int, [_c_int, _c_int, _c_int, ctypes.POINTER(_c_sz)]),
    "sb_rnnt_fwd_bwd": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _c_int, _c_int, _c_int, _c_int, _c_int,
                                 _vp, _vp, _c_sz, _vp]),
    "sb_rnnt_fwd_bwd_compact": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _c_int, _c_int, _c_int, _c_int,
                                         _vp, _vp, _c_sz, _vp]),
    "sb_rnnt_viterbi_workspace_size": (_c_int, [_c_int, _c_int, _c_int, ctypes.POINTER(_c_sz)]),
    "sb_rnnt_viterbi": (_c_int, [_vp, _vp, _vp, _vp, _vp, _c_int, _c_int, _c_int, _vp, _vp, _vp,
                                 _c_sz, _vp]),
    "sb_rnnt_joint_fwd": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _c_int, _c_int, _c_int, _c_int,
                                   _c_int, _c_int, _vp]),
    "sb_rnnt_joint_dlogits": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _c_int, _c_int,
                                       _c_int, _c_int, _c_int, _c_int, _vp]),
    "sb_rnnt_joint_build_slab": (_c_int, [_vp, _vp, _vp, _c_int, _c_int, _c_int, _c_int, _c_int,
                                          _c_int, _vp]),
    "sb_rnnt_joint_reduce_slab": (_c_int, [_vp, _vp, _vp, _vp, _c_int, _c_int, _c_int, _c_int,
                                           _c_int, _c_int, _vp]),
    "sb_rnnt_joint_vocab_fwd_rows": (_c_int, [_vp, _c_ll, _vp, _vp, _vp, _vp, _c_int, _c_int, _c_int,
                                              _c_int, _c_int, _c_int, _c_int, _vp]),
    "sb_rnnt_joint_vocab_bwd_rows": (_c_int, [_vp, _c_ll, _vp, _vp, _vp, _vp, _c_ll, _vp, _c_int,
                                              _c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _vp]),
    "sb_rnnt_decode_static_workspace_size": (_c_int, [_c_int, _c_int, _c_int, _c_int,
                                                      ctypes.POINTER(_c_sz)]),
    "sb_rnnt_decode_static": (_c_int, [_vp, _vp, _vp, _c_int, _c_int, _c_int, _c_int, _c_int, _c_int,
                                       _vp, _vp, _vp, _vp, _c_sz, _vp]),
    "sb_rnnt_decode_static_fits": (_c_int, [_c_int, _c_int]),
    "sb_rnnt_shortlist_rows": (_c_int, [_vp, _c_ll, _vp, _c_int, _c_int, _c_int, _c_int, _c_int,
                                        _c_int, _c_int, _c_int, _c_int, _vp, _vp, _vp, _vp]),
    "sb_rnnt_decode_static_shortlist": (_c_int, [_vp, _vp, _vp, _c_int, _vp, _vp, _c_int, _c_int,
                                                 _c_int, _c_int, _c_int, _c_int, _vp, _vp, _vp, _vp,
                                                 _vp, _c_sz, _vp]),
    "sb_rnnt_search_workspace_size": (_c_int, [_c_int, _c_int, _c_int, _c_int,
                                               ctypes.POINTER(_c_sz)]),
    "sb_rnnt_search_init": (_c_int, [_vp, _c_int, _c_int, _c_int, _c_int, _vp, _c_sz, _vp]),
    "sb_rnnt_search_reset": (_c_int, [_vp, _c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _vp,
                                      _c_sz, _vp]),
    "sb_rnnt_search_round": (_c_int, [_vp, _vp, _vp, _vp, _c_int, _vp, _c_int, _c_int, _c_int, _vp,
                                      _vp, _vp, _c_int, _c_int, _c_int, _c_int, _c_int, _c_int,
                                      _vp, _c_sz, _vp]),
    "sb_rnnt_search_frame_end": (_c_int, [_vp, _c_int, _vp, _vp, _c_int, _c_int, _vp, _c_int,
                                          _c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _vp,
                                          _c_sz, _vp]),
    "sb_rnnt_search_final": (_c_int, [_vp, _c_int, _vp, _vp, _vp, _c_int, _c_int, _c_int, _c_int,
                                      _vp, _c_sz, _vp]),
    "sb_rnnt_pred_step": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _c_int,
                                   _c_int, _c_int, _c_int, _c_int, _vp]),
    "sb_rnnt_search_lm_rows": (_c_int, [_vp, _vp, _vp, _vp, _vp, _c_int, _vp, _c_int, _c_int,
                                        _c_int, _c_int, _c_int, _c_int, _c_int, _c_int, _lmp, _db,
                                        _db, _vp, _c_sz, _vp]),
    "sb_rnnt_search_round_lm": (_c_int, [_vp, _vp, _vp, _vp, _c_int, _vp, _c_int, _c_int, _c_int,
                                         _vp, _vp, _vp, _c_int, _c_int, _c_int, _c_int, _c_int,
                                         _c_int, _vp, _c_sz, _vp]),
    "sb_debug_gru_timeline": (_c_int, [_vp]),
    "sb_debug_gru_cluster": (_c_int, [_c_int]),
    "sb_debug_gru_ksplit": (_c_int, [_c_int]),
    "sb_debug_gru_flags": (_c_int, [_c_int]),
    "sb_debug_gru_fwd_kernel": (ctypes.c_char_p, []),
    "sb_debug_gru_bwd_kernel": (ctypes.c_char_p, []),
    "sb_debug_gru_plan": (_c_int, [_c_int, ctypes.POINTER(_c_int)]),
    "sb_debug_gru_wide_ring": (_c_int, [_c_int]),
    "sb_debug_gemm_flags": (_c_int, [_c_int]),
    "sb_debug_gemm_kernel": (ctypes.c_char_p, []),
    "sb_debug_gemm_epilogue": (ctypes.c_char_p, []),
    "sb_edit_distance": (_c_ll, [_vp, _c_ll, _vp, _c_ll]),
    "sb_log_specgram": (_c_int, [_vp, _vp, _vp, _c_int, _c_int, _c_int, ctypes.c_double, _fl, _vp,
                                 _vp, _vp, _c_int, _vp]),
    "sb_gru_fwd_workspace_size": (_c_int, [_c_int, _c_int, _c_int, ctypes.POINTER(_c_sz)]),
    "sb_gru_fwd": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _c_sz, _c_int, _c_int, _c_int,
                            _c_int, _vp]),
    "sb_gru_fwd_h0": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _c_sz, _c_int, _c_int,
                               _c_int, _c_int, _vp]),
    "sb_gru_fwd_f32": (_c_int, [_vp, _vp, _vp, _vp, _vp, _c_int, _c_int, _c_int, _c_int, _vp]),
    "sb_time_align": (_c_int, [_vp, _c_ll, _vp, _c_ll, _vp, _c_int, _c_int, _c_int, _c_int, _c_int,
                               _vp]),
    "sb_lookahead_fwd": (_c_int, [_vp, _vp, _vp, _vp, _vp, _c_int, _c_int, _c_int, _c_int, _vp]),
    "sb_lookahead_bwd_workspace_size": (_c_int, [_c_int, _c_int, _c_int, _c_int,
                                                 ctypes.POINTER(_c_sz)]),
    "sb_lookahead_bwd": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _c_sz, _c_int, _c_int, _c_int,
                                  _c_int, _vp]),
    "sb_gru_bwd_workspace_size": (_c_int, [_c_int, _c_int, _c_int, ctypes.POINTER(_c_sz)]),
    "sb_gru_bwd": (_c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _c_sz, _c_int, _c_int,
                            _c_int, _c_int, _vp]),
    "sb_gru_plan": (_c_int, [_c_int, _c_int, _c_int, ctypes.POINTER(_c_int)]),
    "sb_rnnt_joint_resident": (_c_int, [_c_int, _c_int]),
}

_lib = None
launch_count = 0   # C-ABI kernel launches issued by this process (bench.py: gpu_launches)


class SpeechB200Error(RuntimeError):
    pass


def load():
    """Load the CUDA library; raises if it has not been built (python -m speech_b200.csrc.build)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise SpeechB200Error(
            "speech_b200: %s is missing - build it with `python -m speech_b200.csrc.build` "
            "(there is no CPU fallback)" % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status, what):
    if status != 0:
        msg = load().sb_status_string(status).decode()
        raise SpeechB200Error("speech_b200: %s failed: %s (status %d)" % (what, msg, status))


def workspace_size(query, *args):
    """Bytes a `sb_*_workspace_size` / `sb_s2s_beam_state_size` query asks for: query(*args,
    &bytes); raises through check."""
    n = _c_sz(0)
    check(query(*args, ctypes.byref(n)), query.__name__)
    return n.value


def pack_labels(labels, label_lens, act_lens, B, dev, num_classes=None, lattice_rows=None):
    """The flat label format sb_ctc_fwd_bwd and sb_rnnt_fwd_bwd(_compact) share, moved to `dev` in
    one pinned host->device copy of [labels | offsets | label_lens | act_lens] (int32).
    Raises ValueError unless label_lens / act_lens hold one entry per utterance and label_lens sums
    to the number of labels; num_classes (CTC): every label lies in [0, num_classes);
    lattice_rows (Transducer, U+1): no label sequence is longer than lattice_rows - 1.
    -> (labels, offsets, label_lens, act_lens) device views, longest label sequence (0 if B = 0)."""
    import torch
    lab = labels.detach().to("cpu", torch.int32).reshape(-1)
    llen = label_lens.detach().to("cpu", torch.int32).reshape(-1)
    alen = act_lens.detach().to("cpu", torch.int32).reshape(-1)
    if llen.numel() != B or alen.numel() != B:
        raise ValueError("act_lens / label_lens must have one entry per utterance")
    n = lab.numel()
    if int(llen.sum()) != n:
        if lattice_rows is not None:
            raise ValueError("labels / y_lens mismatch")
        raise ValueError("labels has %d entries but label_lens sums to %d" % (n, int(llen.sum())))
    if num_classes is not None and n and (int(lab.min()) < 0 or int(lab.max()) >= num_classes):
        raise ValueError("label out of range")
    max_len = int(llen.max()) if B else 0
    if lattice_rows is not None and max_len > lattice_rows - 1:
        raise ValueError("a label sequence is longer than the lattice (U+1 = %d)" % lattice_rows)
    offs = torch.zeros(B, dtype=torch.int32)
    if B > 1:
        offs[1:] = torch.cumsum(llen[:-1], 0)
    packed = torch.cat([lab, offs, llen, alen]).pin_memory().to(dev, non_blocking=True)
    return (packed[:n], packed[n:n + B], packed[n + B:n + 2 * B], packed[n + 2 * B:]), max_len


def ptr(t):
    """Raw device/host pointer of a tensor (None -> NULL)."""
    return None if t is None else t.data_ptr()


def stream_ptr():
    import torch
    return torch.cuda.current_stream().cuda_stream


def require_cuda(t, name):
    if not t.is_cuda:
        raise SpeechB200Error(
            "speech_b200: %s must live on a CUDA device - this package has no CPU path" % name)
