"""ctypes binding of libfsn_b200.so (C ABI: include/fsn_b200.h).  PyTorch is used only for
device memory and streams; every pointer handed to the library is ``tensor.data_ptr()``."""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "csrc", "libfsn_b200.so")

FSN_OK, FSN_ERR_SHAPE, FSN_ERR_UNSUPPORTED, FSN_ERR_CUDA, FSN_ERR_WORKSPACE = 0, 1, 2, 3, 4
ACT = {None: 0, False: 0, "": 0, "ReLU": 1, "Tanh": 2, "ReLU6": 3}
CELL = {"LSTM": 0, "GRU": 1}
PREC = {"fp32": 0, "f16_tc": 1, "tf32_tc": 2, "f16x3_tc": 3}


class ModelDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "num_freqs", "look_ahead", "fb_num_neighbors", "sb_num_neighbors", "fb_hidden", "sb_hidden",
        "fb_activation", "sb_activation", "norm_type", "num_groups_in_drop_band", "precision", "cell_type")]


class SeqWeights(C.Structure):
    _fields_ = [("w_ih", C.c_void_p * 2), ("w_hh", C.c_void_p * 2), ("b_ih", C.c_void_p * 2),
                ("b_hh", C.c_void_p * 2), ("fc_w", C.c_void_p), ("fc_b", C.c_void_p)]


class LstmLayer(C.Structure):
    _fields_ = [("w_ih", C.c_void_p), ("w_hh", C.c_void_p), ("b_ih", C.c_void_p), ("b_hh", C.c_void_p)]


class FastDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in (
        "num_freqs", "look_ahead", "shrink_size", "num_mels", "enc1_hidden", "enc2_hidden", "bn_hidden", "bn_layers",
        "dec_hidden", "noisy_num_neighbors", "enc_num_neighbors", "precision", "cell_type", "norm_type")]


class FastWeights(C.Structure):
    _fields_ = [("mel_fb", C.c_void_p), ("enc1", LstmLayer), ("enc2", LstmLayer), ("enc_fc_w", C.c_void_p),
                ("enc_fc_b", C.c_void_p), ("bn", LstmLayer * 2), ("bn_fc_w", C.c_void_p), ("bn_fc_b", C.c_void_p),
                ("dec1", LstmLayer), ("dec2", LstmLayer), ("dec_fc_w", C.c_void_p), ("dec_fc_b", C.c_void_p),
                ("bn_packed", C.c_void_p)]


class SeqGrads(C.Structure):
    _fields_ = [("w_ih", C.c_void_p * 2), ("w_hh", C.c_void_p * 2), ("b_ih", C.c_void_p * 2),
                ("b_hh", C.c_void_p * 2), ("fc_w", C.c_void_p), ("fc_b", C.c_void_p)]


class LstmGrads(C.Structure):
    _fields_ = [("w_ih", C.c_void_p), ("w_hh", C.c_void_p), ("b_ih", C.c_void_p), ("b_hh", C.c_void_p)]


class FastGrads(C.Structure):
    _fields_ = [("enc1", LstmGrads), ("enc2", LstmGrads), ("enc_fc_w", C.c_void_p), ("enc_fc_b", C.c_void_p),
                ("bn", LstmGrads * 2), ("bn_fc_w", C.c_void_p), ("bn_fc_b", C.c_void_p),
                ("dec1", LstmGrads), ("dec2", LstmGrads), ("dec_fc_w", C.c_void_p), ("dec_fc_b", C.c_void_p)]


MAX_PARAM_TENSORS = 64
SB_PROBE_FIELDS, SB_PROBE_SLOTS = 16, 4  # fsn_debug_sb_lstm_tc_probe records (FSN_SB_PROBE_FIELDS / _SLOTS)


class ParamList(C.Structure):
    _fields_ = [("n", C.c_int), ("param", C.c_void_p * MAX_PARAM_TENSORS), ("grad", C.c_void_p * MAX_PARAM_TENSORS),
                ("exp_avg", C.c_void_p * MAX_PARAM_TENSORS), ("exp_avg_sq", C.c_void_p * MAX_PARAM_TENSORS),
                ("numel", C.c_int64 * MAX_PARAM_TENSORS)]


class FullbandDesc(C.Structure):
    _fields_ = [("num_freqs", C.c_int32), ("hidden", C.c_int32), ("num_layers", C.c_int32), ("look_ahead", C.c_int32),
                ("activation", C.c_int32), ("norm_type", C.c_int32), ("precision", C.c_int32), ("cell_type", C.c_int32)]


class FullbandGrads(C.Structure):
    _fields_ = [("layer", LstmGrads * 8), ("fc_w", C.c_void_p), ("fc_b", C.c_void_p)]


IMP_MAX_SECTIONS = 8


class ImprovedDesc(C.Structure):
    _fields_ = [("n_fft", C.c_int32), ("hop_length", C.c_int32), ("win_length", C.c_int32), ("num_freqs", C.c_int32),
                ("fdrc", C.c_float), ("num_sections", C.c_int32), ("freq_cutoffs", C.c_int32 * IMP_MAX_SECTIONS),
                ("sb_num_center", C.c_int32 * IMP_MAX_SECTIONS), ("sb_num_neighbor", C.c_int32 * IMP_MAX_SECTIONS),
                ("fb_num_center", C.c_int32 * IMP_MAX_SECTIONS), ("fb_num_neighbor", C.c_int32 * IMP_MAX_SECTIONS),
                ("fb_hidden", C.c_int32), ("sb_hidden", C.c_int32), ("fb_activation", C.c_int32),
                ("sb_activation", C.c_int32), ("precision", C.c_int32), ("cell_type", C.c_int32)]


class ImprovedWeights(C.Structure):
    _fields_ = [("fb", SeqWeights), ("sb", SeqWeights * IMP_MAX_SECTIONS), ("sb_packed", C.c_void_p * IMP_MAX_SECTIONS)]


class ImprovedGrads(C.Structure):
    _fields_ = [("fb", SeqGrads), ("sb", SeqGrads * IMP_MAX_SECTIONS)]


_P, _I, _L, _F, _S = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_size_t
_SIGNATURES = {
    "fsn_version": (C.c_int, []),
    "fsn_last_error": (C.c_char_p, []),
    "fsn_built_arch": (C.c_int, []),
    "fsn_stft": (C.c_int, [_P, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _I, _P]),
    "fsn_istft": (C.c_int, [_P, _P, _I, _P, _I, _I, _I, _I, _I, _I, _P, _P]),
    "fsn_decompress_cirm": (C.c_int, [_P, _P, _L, _F, _F, _P]),
    "fsn_compress_cirm": (C.c_int, [_P, _P, _L, _F, _F, _P]),
    "fsn_build_cirm": (C.c_int, [_P, _P, _P, _P, _P, _L, _P]),
    "fsn_drop_band": (C.c_int, [_P, _P, _I, _I, _I, _I, _I, _P]),
    "fsn_model_workspace_bytes": (_S, [C.POINTER(ModelDesc), _I, _I]),
    "fsn_sb_packed_bytes": (_S, [C.POINTER(ModelDesc)]),
    "fsn_pack_sb_weights": (C.c_int, [C.POINTER(ModelDesc), C.POINTER(SeqWeights), _P, _P]),
    "fsn_model_forward": (C.c_int, [C.POINTER(ModelDesc), C.POINTER(SeqWeights), C.POINTER(SeqWeights), _P, _P,
                                    _I, _I, _P, _P, _S, _P]),
    "fsn_enhance_workspace_bytes": (_S, [C.POINTER(ModelDesc), _I, _I, _I, _I]),
    "fsn_enhance": (C.c_int, [C.POINTER(ModelDesc), C.POINTER(SeqWeights), C.POINTER(SeqWeights), _P, _P, _P, _I, _I,
                              _I, _I, _I, _P, _P, _P, _F, _P, _S, _P]),
    "fsn_fast_workspace_bytes": (_S, [C.POINTER(FastDesc), _I, _I]),
    "fsn_fast_packed_bytes": (_S, [C.POINTER(FastDesc)]),
    "fsn_fast_pack_bn_weights": (C.c_int, [C.POINTER(FastDesc), C.POINTER(FastWeights), _P, _P]),
    "fsn_fast_model_forward": (C.c_int, [C.POINTER(FastDesc), C.POINTER(FastWeights), _P, _I, _I, _P, _P, _S, _P]),
    "fsn_improved_workspace_bytes": (_S, [C.POINTER(ImprovedDesc), _I, _I]),
    "fsn_improved_forward": (C.c_int, [C.POINTER(ImprovedDesc), C.POINTER(ImprovedWeights), _P, _I, _I, _P, _P, _P, _S,
                                       _P]),
    "fsn_improved_enhance_workspace_bytes": (_S, [C.POINTER(ImprovedDesc), _I, _I]),
    "fsn_improved_enhance": (C.c_int, [C.POINTER(ImprovedDesc), C.POINTER(ImprovedWeights), _P, _P, _I, _I, _P, _P, _P, _F,
                                       _P, _S, _P]),
    "fsn_improved_packed_bytes": (_S, [C.POINTER(ImprovedDesc), _I]),
    "fsn_improved_pack_sb_weights": (C.c_int, [C.POINTER(ImprovedDesc), C.POINTER(ImprovedWeights), _I, _P, _P]),
    "fsn_improved_train_workspace_bytes": (_S, [C.POINTER(ImprovedDesc), _I, _I]),
    "fsn_improved_train_forward": (C.c_int, [C.POINTER(ImprovedDesc), C.POINTER(ImprovedWeights), _P, _I, _I, _P, _P, _S,
                                             _P]),
    "fsn_improved_train_backward": (C.c_int, [C.POINTER(ImprovedDesc), C.POINTER(ImprovedWeights), _P, _I, _I,
                                              C.POINTER(ImprovedGrads), _P, _S, _P]),
    "fsn_train_workspace_bytes": (_S, [C.POINTER(ModelDesc), _I, _I]),
    "fsn_train_forward": (C.c_int, [C.POINTER(ModelDesc), C.POINTER(SeqWeights), C.POINTER(SeqWeights), _P, _I, _I, _P,
                                    _P, _S, _P]),
    "fsn_train_backward": (C.c_int, [C.POINTER(ModelDesc), C.POINTER(SeqWeights), C.POINTER(SeqWeights), _P, _I, _I,
                                     C.POINTER(SeqGrads), C.POINTER(SeqGrads), _P, _S, _P]),
    "fsn_fast_train_workspace_bytes": (_S, [C.POINTER(FastDesc), _I, _I]),
    "fsn_fast_train_forward": (C.c_int, [C.POINTER(FastDesc), C.POINTER(FastWeights), _P, _I, _I, _P, _P, _S, _P]),
    "fsn_fast_train_backward": (C.c_int, [C.POINTER(FastDesc), C.POINTER(FastWeights), _P, _I, _I, C.POINTER(FastGrads), _P,
                                          _S, _P]),
    "fsn_mse_loss_scratch_bytes": (_S, []),
    "fsn_mse_loss": (C.c_int, [_P, _P, _I, _I, _I, _P, _P, _P, _S, _P]),
    "fsn_cirm_mse_per_clip_workspace_bytes": (_S, [_I, _I, _I, _I]),
    "fsn_cirm_mse_per_clip": (C.c_int, [_P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _S, _P]),
    "fsn_clip_adam_scratch_bytes": (_S, []),
    "fsn_clip_adam": (C.c_int, [C.POINTER(ParamList), _F, _F, _F, _F, _F, _F, _I, _P, _P, _S, _P]),
    "fsn_clip_adam_steps": (C.c_int, [C.POINTER(ParamList), _F, _F, _F, _F, _F, _F, _P, _P, _P, _S, _P]),
    "fsn_fullband_workspace_bytes": (_S, [C.POINTER(FullbandDesc), _I, _I]),
    "fsn_fullband_forward": (C.c_int, [C.POINTER(FullbandDesc), _P, _P, _P, _P, _I, _I, _P, _P, _S, _P]),
    "fsn_fullband_enhance_workspace_bytes": (_S, [C.POINTER(FullbandDesc), _I, _I, _I, _I]),
    "fsn_fullband_enhance": (C.c_int, [C.POINTER(FullbandDesc), _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _F, _P,
                                       _S, _P]),
    "fsn_fullband_stream_state_bytes": (_S, [C.POINTER(FullbandDesc), _I, _I, _I]),
    "fsn_fullband_stream_workspace_bytes": (_S, [C.POINTER(FullbandDesc), _I, _I, _I, _I]),
    "fsn_fullband_stream_delay": (C.c_int, [C.POINTER(FullbandDesc), _I, _I]),
    "fsn_fullband_stream_step": (C.c_int, [C.POINTER(FullbandDesc), _P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _S,
                                           _P, _S, _P]),
    "fsn_fast_stream_state_bytes": (_S, [C.POINTER(FastDesc), _I, _I, _I]),
    "fsn_fast_stream_workspace_bytes": (_S, [C.POINTER(FastDesc), _I, _I, _I, _I]),
    "fsn_fast_stream_delay": (C.c_int, [C.POINTER(FastDesc), _I, _I]),
    "fsn_fast_stream_step": (C.c_int, [C.POINTER(FastDesc), C.POINTER(FastWeights), _P, _P, _P, _I, _I, _I, _I, _I, _P, _P,
                                       _S, _P, _S, _P]),
    "fsn_fast_stream_tc_state_bytes": (_S, [C.POINTER(FastDesc), _I, _I, _I]),
    "fsn_fast_stream_tc_workspace_bytes": (_S, [C.POINTER(FastDesc), _I, _I, _I, _I]),
    "fsn_fast_stream_tc_delay": (C.c_int, [C.POINTER(FastDesc), _I, _I]),
    "fsn_fast_stream_tc_step": (C.c_int, [C.POINTER(FastDesc), C.POINTER(FastWeights), _P, _P, _P, _I, _I, _I, _I, _I, _P,
                                          _P, _S, _P, _S, _P]),
    "fsn_stream_state_bytes": (_S, [C.POINTER(ModelDesc), _I, _I, _I]),
    "fsn_stream_workspace_bytes": (_S, [C.POINTER(ModelDesc), _I, _I, _I, _I]),
    "fsn_stream_delay": (C.c_int, [C.POINTER(ModelDesc), _I, _I]),
    "fsn_stream_step": (C.c_int, [C.POINTER(ModelDesc), C.POINTER(SeqWeights), C.POINTER(SeqWeights), _P, _P, _P, _I, _I,
                                  _I, _I, _I, _P, _P, _S, _P, _S, _P]),
    "fsn_stream_tc_state_bytes": (_S, [C.POINTER(ModelDesc), _I, _I, _I]),
    "fsn_stream_tc_workspace_bytes": (_S, [C.POINTER(ModelDesc), _I, _I, _I, _I]),
    "fsn_stream_tc_delay": (C.c_int, [C.POINTER(ModelDesc), _I, _I]),
    "fsn_stream_tc_step": (C.c_int, [C.POINTER(ModelDesc), C.POINTER(SeqWeights), C.POINTER(SeqWeights), _P, _P, _P, _P,
                                     _I, _I, _I, _I, _I, _P, _P, _S, _P, _S, _P]),
    "fsn_fullband_train_workspace_bytes": (_S, [C.POINTER(FullbandDesc), _I, _I]),
    "fsn_fullband_train_forward": (C.c_int, [C.POINTER(FullbandDesc), _P, _P, _P, _P, _I, _I, _P, _P, _S, _P]),
    "fsn_fullband_train_backward": (C.c_int, [C.POINTER(FullbandDesc), _P, _P, _P, _P, _I, _I, C.POINTER(FullbandGrads), _P,
                                              _S, _P]),
    "fsn_peak_normalize_int16": (C.c_int, [_P, _I, _I, _F, _P, _P]),
    "fsn_si_sdr": (C.c_int, [_P, _P, _I, _I, _P, _P]),
    "fsn_si_sdr_lengths": (C.c_int, [_P, _P, _P, _I, _I, _P, _P]),
    "fsn_stoi_workspace_bytes": (_S, [_I, _I, _I]),
    "fsn_stoi": (C.c_int, [_P, _P, _P, _I, _I, _I, _P, _P, _S, _P]),
    "fsn_resample_workspace_bytes": (_S, [_I, _I, _I, _I, _I]),
    "fsn_resample": (C.c_int, [_P, _P, _I, _I, _I, _I, _I, _P, _I, _P, _S, _P]),
    "fsn_rir_convolve": (C.c_int, [_P, _P, _P, _I, _I, _I, _P, _P]),
    "fsn_snr_mix": (C.c_int, [_P, _P, _P, _P, _F, _F, _I, _I, _P, _P, _P]),
    "fsn_debug_row_to_unit": (C.c_int, [_I, _I, _I, _I, C.POINTER(C.c_int), C.POINTER(C.c_int)]),
    "fsn_debug_unit_to_row": (C.c_int, [_I, _I, _I, _I, _I]),
    "fsn_debug_reflect_count": (C.c_int, [_I, _I, _I]),
    "fsn_debug_lstm_tc_workspace_bytes": (_S, [_I, _I, _I, _I, _I]),
    "fsn_debug_lstm_layer_tc": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _S, _P]),
    "fsn_debug_lstm_tc_carry": (C.c_int, [_P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _P, _P, _P, _I, _P, _P, _S, _P]),
    "fsn_debug_linear_tc": (C.c_int, [_P, _I, _I, _P, _P, _I, _I, _I, _P, _P, _S, _P]),
    "fsn_debug_lstm_rec_tc_scratch_bytes": (_S, [_I, _I]),
    "fsn_debug_lstm_rec_tc": (C.c_int, [_P, _P, _P, _P, _L, _L, _P, _L, _L, _I, _I, _I, _I, _P, _P, _P, _L, _P, _I, _P, _P,
                                        _S, _P]),
    "fsn_debug_sb_lstm_tc_packed_bytes": (_S, [_I, _I]),
    "fsn_debug_sb_lstm_tc_max_clusters": (C.c_int, [_I, _I, _I, _I, C.POINTER(C.c_int)]),
    "fsn_debug_sb_lstm_tc": (C.c_int, [C.POINTER(SeqWeights), _I, _I, _I, _I, _I, _I, _P, _P, _I, _I, _I, _I, _P, _P, _I,
                                       _I, _I, _I, _I, _P, _P, _P]),
    "fsn_debug_sb_lstm_tc2_ws_bytes": (_S, [_I, _I, _I, _I, _I]),
    "fsn_debug_sb_lstm_tc2": (C.c_int, [C.POINTER(SeqWeights), _I, _I, _I, _I, _I, _P, _P, _I, _I, _I, _I, _P, _P, _I, _I,
                                        _I, _I, _P, _P, _P, _P]),
    "fsn_debug_sb_tc2_pass": (C.c_int, [C.POINTER(SeqWeights), _I, _I, _I, _I, _I, _P, _P, _I, _I, _I, _I, _P, _P, _I, _I,
                                        _I, _I, _I, _I, _P, _P, _S, _P, _P]),
    "fsn_debug_sb_lstm_tc_carry": (C.c_int, [C.POINTER(SeqWeights), _I, _I, _I, _I, _I, _P, _P, _I, _I, _I, _P, _I, _P,
                                             _I, _P, _P, _P, _P, _P]),
    "fsn_debug_sb_lstm_tc_phased": (C.c_int, [C.POINTER(SeqWeights), _I, _I, _I, _I, _P, _P, _I, _I, _I, _I, _P, _P, _P,
                                              _P, _P, _P, _P, _P, _P, _P]),
    "fsn_debug_sb_lstm_tc_probe": (C.c_int, [C.POINTER(SeqWeights), _I, _I, _I, _I, _I, _I, _P, _P, _I, _I, _I, _I, _P, _P,
                                             _I, _I, _I, _I, _I, _P, _P, _P, _I, _I, _P]),
    "fsn_debug_tgemm": (C.c_int, [_P, _L, _P, _L, _P, _L, _I, _I, _I, _I, _P, _L, _P]),
    "fsn_debug_tgemm_blocked": (C.c_int, [_P, _P, _P, _I, _I, _I, _I, _I, _P, _L, _P]),
    "fsn_debug_lstm_fwd_step": (C.c_int, [_P, _P, _P, _P, _I, _P, _P, _P, _P, _P, _P, _I, _I, _I, _P, _L, _P]),
    "fsn_debug_fc_gemm": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _P]),
    "fsn_debug_sgemm": (C.c_int, [_I, _P, _L, _P, _L, _P, _L, _I, _I, _I, _I, _P, _L, _P]),
    "fsn_debug_colsum": (C.c_int, [_P, _L, _I, _L, _P, _P, _P, _L, _P]),
    "fsn_debug_small_out_wgrad": (C.c_int, [_P, _P, _L, _I, _P, _P, _L, _P]),
    "fsn_debug_transpose": (C.c_int, [_P, _L, _I, _P, _P]),
    "fsn_debug_transpose_blocked": (C.c_int, [_P, _L, _I, _L, _P, _P, _I, C.POINTER(C.c_int), _P, _P]),
    "fsn_debug_gemm_tc": (C.c_int, [_P, _L, _I, _P, _I, _I, _P, _I, _P, _I, _I, _P, _L, _L, _P, _S, _P]),
    "fsn_debug_lstm_train_workspace_bytes": (_S, [_I, _I, _I, _I, _I, _I]),
    "fsn_debug_lstm_train": (C.c_int, [C.POINTER(LstmLayer), _I, _I, _I, _I, _I, _I, _P, _P, _P, _P, _I, _P, _P,
                                       C.POINTER(LstmGrads), _P, _P, _S, _P]),
    "fsn_debug_seq_stack_workspace_bytes": (_S, [_I, C.POINTER(C.c_int), _I, _I, _I, _I, _I, _I, _I, _I]),
    "fsn_debug_seq_stack": (C.c_int, [C.POINTER(LstmLayer), _I, C.POINTER(C.c_int), _I, _I, _I, _I, _I, _I, _I, _I, _P, _P,
                                      _P, _P, _I, _I, _P, _P, _S, C.POINTER(C.c_int), _P]),
    "fsn_debug_stft": (C.c_int, [_P, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _I, _P]),
    "fsn_debug_istft": (C.c_int, [_P, _P, _I, _P, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P, _P, _F, _P, _P]),
    "fsn_debug_istft_mask_adjoint": (C.c_int, [_P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P]),
    "fsn_debug_wav_epilogue": (C.c_int, [_P, _P, _I, _I, _P, _P, _F, _P, _P, _I, _I, _I, _P]),
    "fsn_debug_norm_unfold_bwd": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _F, _I, _P, _P, _P]),
    "fsn_debug_fast_norm_unfold_bwd": (C.c_int, [_P, _P, _P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _F, _P, _P, _P, _P]),
    "fsn_debug_imp_unfold_bwd": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P]),
    "fsn_debug_imp_section_input": (C.c_int, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _I, _P, _P, _P]),
    "fsn_debug_imp_section_lstm_tc_workspace_bytes": (_S, [_I, _I, _I, _I, _I]),
    "fsn_debug_imp_section_lstm_tc": (C.c_int, [C.POINTER(SeqWeights), _I, _I, _I, _P, _I, _I, _I, _I, _P, _P, _P, _S, _P]),
    "fsn_debug_norm_stats": (C.c_int, [_P, _I, _I, _I, _I, _L, _L, _P, _P, _I, _I, _P, _F, _F, _F, _P, _P, _P, _P, _P]),
    "fsn_debug_train_stats": (C.c_int, [_P, _I, _I, _I, _I, _I, _P, _P]),
    "fsn_debug_forgetting_scale": (C.c_int, [_P, _I, _P, _I, _I, _I, _I, _L, _L, _F, _P, _P, _I, _I, _P, _P, _P, _P, _P]),
    "fsn_debug_forgetting_bwd": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P]),
    "fsn_debug_stoi_stages": (C.c_int, [_P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _S, _P]),
    "fsn_debug_cum_clip_scale": (C.c_int, [_P, _I, _I, _I, _L, _L, _F, _P, _P, _P]),
    "fsn_debug_cum_unit_scale": (C.c_int, [_P, _P, _I, _I, _I, _I, _I, _I, _F, _I, _P, _P]),
    "fsn_debug_forget_unit_broadcast": (C.c_int, [_P, _I, _I, _I, _I, _P, _P]),
    "fsn_debug_fast_bn": (C.c_int, [_P, _P, _L, _L, _I, _I, _I, _I, _I, _I, _I, _F, _P, _P, _P, _P, _P]),
    "fsn_debug_fast_dec_input": (C.c_int, [_P, _P, _L, _L, _L, _I, _I, _I, _I, _I, _L, _L, _P, _P]),
    "fsn_debug_transpose_mag": (C.c_int, [_P, _I, _I, _I, _I, _L, _L, _P, _P, _P, _P]),
    "fsn_debug_crm_output": (C.c_int, [_P, _L, _L, _I, _I, _I, _I, _P, _P]),
    "fsn_debug_scale_rows": (C.c_int, [_P, _P, _L, _I, _I, _I, _P, _P]),
    "fsn_debug_imp_compress": (C.c_int, [_P, _I, _I, _I, _F, _I, _P, _P]),
    "fsn_debug_train_gather": (C.c_int, [_P, _P, _P, _P, _I, _I, _I, _I, _I, _I, _P, _P]),
    "fsn_debug_sb_head": (C.c_int, [_P, _I, _I, _I, _P, _P, _I, _I, _I, _I, _I, _I, _L, _L, _I, _P, _P]),
    "fsn_debug_sb_head_bwd": (C.c_int, [_P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I, _L, _L, _P, _P]),
    "fsn_debug_train_dy": (C.c_int, [_P, _P, _I, _I, _I, _I, _I, _I, _P, _P]),
    "fsn_last_error_code": (C.c_int, []),
    "fsn_last_launch_count": (C.c_int64, []),
    "fsn_total_launch_count": (C.c_int64, []),
    "fsn_set_profiling": (C.c_int, [_I]),
    "fsn_last_stage_ms": (C.c_float, [_I]),
}
EXPORTED_SYMBOLS = tuple(_SIGNATURES)

_lib: Optional[C.CDLL] = None


def load() -> C.CDLL:
    """Load the CUDA library; fail loudly if it has not been built (no fallback path exists)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"fullsubnet_b200: {LIB_PATH} is missing. Build it with `python -c 'import __graft_entry__ as g; "
                "g.build()'` (nvcc, sm_90a). There is no CPU/PyTorch fallback for this path.")
        lib = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError if the ABI is incomplete
            fn.restype, fn.argtypes = res, args
        _lib = lib
    return _lib


def check(rc: int) -> None:
    """Map C-ABI status codes to the exception types the reference raises."""
    if rc == FSN_OK:
        return
    msg = load().fsn_last_error().decode()
    if rc == FSN_ERR_SHAPE:
        raise AssertionError(msg)
    if rc == FSN_ERR_UNSUPPORTED:
        raise NotImplementedError(msg)
    raise RuntimeError(f"libfsn_b200 error {rc}: {msg}")


def check_workspace(nbytes: int) -> int:
    """*_workspace_bytes() return 0 on failure: raise what the failed shape / configuration check asked for."""
    if nbytes == 0:
        check(load().fsn_last_error_code() or FSN_ERR_SHAPE)
    return nbytes


def require_cuda(t: torch.Tensor, what: str) -> torch.Tensor:
    if not t.is_cuda:
        raise RuntimeError(
            f"fullsubnet_b200: {what} must be a CUDA tensor (got {t.device}); this package has no CPU path.")
    if t.dtype != torch.float32:
        t = t.float()
    return t.contiguous()


def lengths_table(lengths, B: int, L: int) -> np.ndarray:
    """Per-clip lengths (sequence of B ints or a CPU integer tensor) -> contiguous int32 host array; the library checks
    the rest (n_fft/2 < length, max == L) before any CUDA call."""
    if isinstance(lengths, torch.Tensor):
        if lengths.is_cuda or lengths.is_floating_point() or lengths.is_complex() or lengths.dim() != 1:
            raise ValueError("lengths must be a 1-D CPU integer tensor or a sequence of ints")
        lengths = lengths.tolist()
    lens = np.ascontiguousarray([int(v) for v in lengths], dtype=np.int32)
    if lens.shape != (B,):
        raise ValueError(f"lengths has {lens.size} entries for a batch of {B} clips")
    if lens.size and int(lens.max()) > L:
        b = int(lens.argmax())
        raise ValueError(f"lengths[{b}] = {int(lens[b])} exceeds the {L} samples of a row")
    return lens


def stream_ptr(device) -> int:
    return torch.cuda.current_stream(device).cuda_stream


def ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()
