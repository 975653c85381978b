"""ctypes binding of libb200tts.so (C ABI declared in include/b200tts.h).

The library is the product: if it is missing or fails to load, every op raises -- there is no
eager-PyTorch or CPU fallback (north_star: "no CPU fallback").
"""
import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_double, c_float, c_int, c_int32, c_longlong, c_size_t, c_uint8, c_uint64, c_ulonglong, c_void_p

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, 'libb200tts.so')

CELL_DROPOUT, CELL_ZONEOUT = 0, 1
ATT_LOCATION, ATT_FORWARD = 0, 1


class B200TTSError(RuntimeError):
    pass


class DecoderShape(Structure):
    _fields_ = [(n, c_int) for n in ('B', 'L', 'T', 'M', 'D', 'P', 'A', 'C', 'K', 'N', 'cell_kind', 'training')] + \
               [('rate_h', c_float), ('rate_c', c_float), ('prenet_rate', c_float), ('att_kind', c_int), ('att_extent', c_int), ('R', c_int),
                                                                     ('att_window_back', c_int), ('att_window_ahead', c_int)]


DECODER_PARAM_FIELDS = ('prenet_w0', 'prenet_b0', 'prenet_w1', 'prenet_b1', 'att_w_ih', 'att_w_hh', 'att_b_ih', 'att_b_hh',
                        'gen_w_ih', 'gen_w_hh', 'gen_b_ih', 'gen_b_hh', 'attn_query', 'attn_memory', 'attn_location',
                        'attn_loc_features', 'attn_bias', 'attn_energy', 'frame_w', 'frame_b', 'stop_w', 'stop_b')


class DecoderParams(Structure):
    _fields_ = [(n, c_void_p) for n in DECODER_PARAM_FIELDS]


class DecoderInputs(Structure):
    _fields_ = [(n, c_void_p) for n in ('memory', 'text_lengths', 'target', 'teacher', 'mask_prenet0', 'mask_prenet1',
                                        'mask_att_h', 'mask_att_c', 'mask_gen_h', 'mask_gen_c', 'mask_step_prenet0',
                                        'mask_step_prenet1', 'forced_rows')] + \
        [('forced_count', c_int), ('forced_alignment', c_void_p)]


class DecoderOutputs(Structure):
    _fields_ = [(n, c_void_p) for n in ('spectrogram', 'stop', 'alignments')]


class DecoderState(Structure):
    _fields_ = [(n, c_void_p) for n in ('att_h', 'att_c', 'gen_h', 'gen_c', 'context', 'cum_weights', 'frame', 'attended')]


class DecoderOutputGrads(Structure):
    _fields_ = [(n, c_void_p) for n in ('d_spectrogram', 'd_stop', 'd_alignments')]


class ConvBlockShape(Structure):
    _fields_ = [(n, c_int) for n in ('NB', 'G', 'Cin', 'Cout', 'L', 'k', 'dilation', 'activation', 'highway', 'training')] + \
               [('eps', c_float), ('momentum', c_float), ('dropout', c_float), ('stage', c_int)]


class LossShape(Structure):
    _fields_ = [(n, c_int) for n in ('B', 'N', 'T', 'L', 'guided')] + [('guided_g', c_float), ('stop_pos_weight', c_float), ('R', c_int)]


class BiLSTMShape(Structure):
    _fields_ = [(n, c_int) for n in ('B', 'L', 'E', 'H')]


BILSTM_PARAM_FIELDS = ('w_ih', 'w_hh', 'b_ih', 'b_hh', 'w_ih_reverse', 'w_hh_reverse', 'b_ih_reverse', 'b_hh_reverse')


class BiLSTMParams(Structure):
    _fields_ = [(n, c_void_p) for n in BILSTM_PARAM_FIELDS]


class VocoderShape(Structure):
    _fields_ = [(n, c_int) for n in ('B', 'total_frames', 'N', 'hop', 'win', 'n_mels')] + \
               [(n, c_float) for n in ('power', 'momentum', 'preemphasis')] + [('nnls_iters', c_int)]


class GLStreamShape(Structure):
    _fields_ = [(n, c_int) for n in ('N', 'hop', 'win', 'lookahead', 'iters', 'slots')] + [('preemphasis', c_float)]


class GLStreamRow(Structure):
    _fields_ = [(n, c_int) for n in ('slot', 'frames', 'ended')] + [(n, c_longlong) for n in ('s_off', 'wave_off')]


# include/b200tts.h: B200TTS_GL_STREAM_MAX_LOOKAHEAD
GL_STREAM_MAX_LOOKAHEAD = 7


class AnalysisShape(Structure):
    _fields_ = [(n, c_int) for n in ('B', 'total_samples', 'total_frames', 'N', 'hop', 'win', 'n_mels')] + [('preemphasis', c_double)]


class GemmDesc(Structure):
    """b200tts_gemm_desc: the library's whole GEMM descriptor (csrc/common.cuh GemmDesc), for b200tts_debug_gemm."""
    _fields_ = [('A', c_void_p), ('B', c_void_p), ('C', c_void_p), ('bias', c_void_p)] + \
               [(n, c_int) for n in ('M', 'N', 'K', 'lda', 'ldb', 'ldc', 'transA', 'transB')] + \
               [('alpha', c_float), ('beta', c_float), ('batch', c_int)] + \
               [(n, c_longlong) for n in ('strideA', 'strideB', 'strideC')] + \
               [('a_batch_mod', c_int), ('splitk', c_int), ('partial', c_void_p), ('keep_partials', c_int),
                ('A16', c_void_p), ('lda16', c_int), ('B16', c_void_p), ('ldb16', c_int), ('kin', c_int),
                ('kosA', c_longlong), ('kosB', c_longlong)]


class WaveRNNFoldShape(Structure):
    _fields_ = [(n, c_int) for n in ('B', 'rows', 'n_mels', 'aux_dims', 'hop', 'pad', 'scale', 'target', 'overlap', 'max_frames')]


class WaveRNNWindowShape(Structure):
    _fields_ = [(n, c_int) for n in ('n_mels', 'aux_dims', 'hop', 'pad', 'scale', 'frames')] + [('m0', c_longlong)] + \
               [(n, c_int) for n in ('mel_len', 'a0', 'aux_len')]


class WaveRNNWindowRow(Structure):
    _fields_ = [('w', WaveRNNWindowShape), ('s0', c_longlong), ('mel_off', c_longlong), ('aux_off', c_longlong), ('n', c_int)]


class WaveRNNUnfoldStream(Structure):
    _fields_ = [(n, c_longlong) for n in ('q0', 'q1', 'wave_off')] + [(n, c_int) for n in ('frames', 'fold0', 'nfolds', 'src')]


WAVERNN_MAX_STREAMS = 64

# include/b200tts.h: the stream ids of the draws under one request seed (b200tts_fill_keep_mask_rows, b200tts_fill_uniform_rows)
SEED_STREAMS = {'step_prenet0': 0x5EED000000000001, 'step_prenet1': 0x5EED000000000002, 'vocoder': 0x5EED000000000003}


class WaveRNNShape(Structure):
    _fields_ = [(n, c_int) for n in ('rows', 'rnn_dims', 'fc_dims', 'n_out', 'mode', 'fold_len')]


WAVERNN_PARAM_FIELDS = ('w_hh1', 'b_hh1', 'u1', 'w_prev', 'w_ih2x', 'w_hh2', 'b_hh2', 'w_fc1x', 'w_fc2x', 'w_fc3', 'b_fc3')


class WaveRNNParams(Structure):
    _fields_ = [(n, c_void_p) for n in WAVERNN_PARAM_FIELDS]


class WaveRNNCond(Structure):
    _fields_ = [(n, c_void_p) for n in ('c', 'g1', 'c2', 'p1', 'p2')]


class GRUSeqShape(Structure):
    _fields_ = [(n, c_int) for n in ('B', 'T', 'R')]


# include/b200tts.h: B200TTS_WAVERNN_RAW / _MOL
WAVERNN_MODES = {'RAW': 0, 'MOL': 1}

# include/b200tts.h: B200TTS_MCD_CUT / _STRETCH / _DTW and B200TTS_DTW_MAX_FRAMES
MCD_MODES = {'cut': 0, 'stretch': 1, 'dtw': 2}
DTW_MAX_FRAMES = 6455


class AlignShape(Structure):
    _fields_ = [(n, c_int) for n in ('B', 'S', 'L')] + [(n, c_longlong) for n in ('ld', 'batch_stride')]


# include/b200tts.h: B200TTS_ALIGN_MAX_SYMBOLS and B200TTS_ALIGN_MAX_CELLS
ALIGN_MAX_SYMBOLS = 1024
ALIGN_MAX_CELLS = 1728512

# include/b200tts.h: B200TTS_PITCH_THRESHOLDS, B200TTS_PITCH_MAX_BINS and B200TTS_PITCH_MAX_FRAME_LENGTH
PITCH_THRESHOLDS = 100
PITCH_MAX_BINS = 1201
PITCH_MAX_FRAME_LENGTH = 2048


class PitchShape(Structure):
    _fields_ = [(n, c_int) for n in ('B', 'total_samples', 'total_frames', 'frame_length', 'win_length', 'hop', 'min_period', 'max_period',
                                     'n_bins', 'transition_width')] + \
               [(n, c_double) for n in ('sr', 'fmin', 'log_tiny', 'log_init')] + \
               [('thresholds', c_double * PITCH_THRESHOLDS), ('beta_probs', c_double * PITCH_THRESHOLDS)]


# include/b200tts.h: B200TTS_PSOLA_MAX_PERIOD
PSOLA_MAX_PERIOD = 1024


class PsolaShape(Structure):
    _fields_ = [(n, c_int) for n in ('B', 'total_samples', 'total_frames', 'hop', 'unvoiced_spacing')] + [('sr', c_double)]


# include/b200tts.h: B200TTS_WSOLA_MAX_HOP, B200TTS_WSOLA_MAX_TOLERANCE
WSOLA_MAX_HOP = 1024
WSOLA_MAX_TOLERANCE = 1024


class WsolaShape(Structure):
    _fields_ = [(n, c_int) for n in ('B', 'total_samples', 'total_out_samples', 'total_frames', 'hop', 'tolerance')]


# include/b200tts.h: B200TTS_RESAMPLE_MAX_FACTOR
RESAMPLE_MAX_FACTOR = 2048


class ResampleShape(Structure):
    _fields_ = [(n, c_int) for n in ('B', 'total_samples', 'total_out_samples', 'total_taps', 'max_factor')]


class TrimShape(Structure):
    _fields_ = [(n, c_int) for n in ('B', 'total_samples', 'total_frames', 'frame_length', 'hop')] + [('top_db', c_double)]


# name -> (restype, argtypes); the "-m not gpu" suite checks every symbol of the header resolves
SIGNATURES = {
    'b200tts_last_error': (c_char_p, []),
    'b200tts_version': (c_int, []),
    'b200tts_launch_count': (c_ulonglong, []),
    'b200tts_set_precision': (c_int, [c_int]),
    'b200tts_get_precision': (c_int, []),
    'b200tts_kernel_timing': (c_int, [c_int]),
    'b200tts_kernel_timing_read': (c_int, [c_int, c_char_p, c_int, POINTER(c_float), POINTER(c_int)]),
    'b200tts_set_scratch': (c_int, [c_void_p, c_size_t]),
    'b200tts_set_tensor_core_gemm': (c_int, [c_int]),
    'b200tts_debug_persist_profile_offset': (c_size_t, [POINTER(DecoderShape)]),
    'b200tts_debug_persist_bwd_profile_offset': (c_size_t, [POINTER(DecoderShape), c_int]),
    'b200tts_debug_decoder_views': (c_int, [POINTER(DecoderShape), POINTER(c_size_t), c_int]),
    'b200tts_debug_decoder_geometry': (c_int, [POINTER(DecoderShape), POINTER(c_int), c_int]),
    'b200tts_gemm_f32': (c_int, [c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_int, c_void_p, c_int, c_float,
                                 c_void_p, c_int, c_void_p, c_int, c_longlong, c_longlong, c_longlong, c_int, c_void_p,
                                 c_void_p]),
    'b200tts_debug_gemm': (c_int, [POINTER(GemmDesc), c_int, c_void_p, c_size_t, c_void_p]),
    'b200tts_debug_gemm_pack_cache': (c_int, [c_int]),
    'b200tts_decoder_workspace_bytes': (c_size_t, [POINTER(DecoderShape)]),
    'b200tts_decoder_bwd_workspace_bytes': (c_size_t, [POINTER(DecoderShape)]),
    'b200tts_decoder_path': (c_int, [POINTER(DecoderShape)]),
    'b200tts_decoder_forward': (c_int, [POINTER(DecoderShape), POINTER(DecoderParams), POINTER(DecoderInputs),
                                        POINTER(DecoderOutputs), c_void_p, c_size_t, c_void_p]),
    'b200tts_decoder_forward_chunk': (c_int, [POINTER(DecoderShape), POINTER(DecoderParams), POINTER(DecoderInputs),
                                              POINTER(DecoderOutputs), POINTER(DecoderState), c_int, c_void_p, c_size_t, c_void_p]),
    'b200tts_decoder_state_reset_rows': (c_int, [POINTER(DecoderShape), POINTER(DecoderState), POINTER(c_int), c_int, c_void_p]),
    'b200tts_decoder_backward': (c_int, [POINTER(DecoderShape), POINTER(DecoderParams), POINTER(DecoderInputs),
                                         POINTER(DecoderOutputs), POINTER(DecoderOutputGrads), c_void_p, c_void_p,
                                         c_size_t, POINTER(DecoderParams), c_void_p, c_void_p]),
    'b200tts_attention_step_workspace_elems': (c_size_t, [c_int, c_int, c_int]),
    'b200tts_attention_step': (c_int, [c_int] * 7 + [c_void_p] * 14),
    'b200tts_attention_step_backward_workspace_elems': (c_size_t, [c_int] * 5),
    'b200tts_attention_step_backward': (c_int, [c_int] * 6 + [c_void_p] * 20),
    'b200tts_debug_attention_backward_chunk': (c_int, [c_int] * 5),
    'b200tts_forward_attention_step_workspace_elems': (c_size_t, [c_int, c_int, c_int]),
    'b200tts_forward_attention_step': (c_int, [c_int] * 5 + [c_void_p] * 12),
    'b200tts_forward_attention_step_backward_workspace_elems': (c_size_t, [c_int] * 3),
    'b200tts_forward_attention_step_backward': (c_int, [c_int] * 4 + [c_void_p] * 16),
    'b200tts_convblock_saved_bytes': (c_size_t, [POINTER(ConvBlockShape)]),
    'b200tts_convblock_workspace_bytes': (c_size_t, [POINTER(ConvBlockShape)]),
    'b200tts_convblock_forward': (c_int, [POINTER(ConvBlockShape), c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                          c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'b200tts_convblock_forward_masked': (c_int, [POINTER(ConvBlockShape), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                                                 c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'b200tts_convblock_backward': (c_int, [POINTER(ConvBlockShape), c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                           c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'b200tts_convblock_forward_counts': (c_int, [POINTER(ConvBlockShape), c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                                 c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'b200tts_convblock_backward_counts': (c_int, [POINTER(ConvBlockShape), c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                                  c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                                  c_void_p]),
    'b200tts_lstm_cell_forward': (c_int, [c_int, c_int, c_int, c_int, c_float, c_float] + [c_void_p] * 8),
    'b200tts_lstm_cell_backward': (c_int, [c_int, c_int, c_int, c_int, c_float, c_float] + [c_void_p] * 9),
    'b200tts_generator_workspace_bytes': (c_size_t, [c_int, c_int]),
    'b200tts_generator_forward': (c_int, [c_int, c_int, c_int, c_longlong] + [c_void_p] * 8),
    'b200tts_generator_backward': (c_int, [c_int, c_int, c_int, c_longlong] + [c_void_p] * 12),
    'b200tts_embedding_forward': (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_longlong, c_int, c_void_p]),
    'b200tts_embedding_backward': (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_longlong, c_int, c_int, c_void_p]),
    'b200tts_adam_clip_scratch_floats': (c_size_t, []),
    'b200tts_adam_clip_step': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_float, c_float, c_float, c_float, c_float, c_float,
                                       c_int, c_void_p, c_void_p]),
    'b200tts_bilstm_saved_bytes': (c_size_t, [POINTER(BiLSTMShape)]),
    'b200tts_bilstm_workspace_bytes': (c_size_t, [POINTER(BiLSTMShape)]),
    'b200tts_bilstm_forward': (c_int, [POINTER(BiLSTMShape), POINTER(BiLSTMParams), c_void_p, c_void_p, c_void_p, c_void_p,
                                       c_void_p, c_void_p]),
    'b200tts_bilstm_backward': (c_int, [POINTER(BiLSTMShape), POINTER(BiLSTMParams), c_void_p, c_void_p, c_void_p, c_void_p,
                                        POINTER(BiLSTMParams), c_void_p, c_void_p]),
    'b200tts_debug_bilstm_layout': (c_int, [POINTER(BiLSTMShape), POINTER(c_size_t), c_int]),
    'b200tts_loss_workspace_bytes': (c_size_t, []),
    'b200tts_tacotron_loss_forward': (c_int, [POINTER(LossShape)] + [c_void_p] * 12),
    'b200tts_tacotron_loss_backward': (c_int, [POINTER(LossShape)] + [c_void_p] * 14),
    'b200tts_set_mask_epoch': (c_int, [c_void_p]),
    'b200tts_fill_keep_mask': (c_int, [c_void_p, c_size_t, c_float, c_uint64, c_uint64, c_void_p]),
    'b200tts_fill_keep_mask_rows': (c_int, [c_void_p, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_uint64, c_void_p]),
    'b200tts_fill_uniform_rows': (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_uint64, c_void_p]),
    'b200tts_vocoder_workspace_bytes': (c_size_t, [POINTER(VocoderShape)]),
    'b200tts_vocoder_fft_plan': (c_int, [c_int, POINTER(c_int), c_int]),
    'b200tts_spectrogram_magnitude': (c_int, [POINTER(VocoderShape), c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p]),
    'b200tts_griffinlim': (c_int, [POINTER(VocoderShape), c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_size_t,
                                   c_void_p]),
    'b200tts_deemphasis_normalize': (c_int, [POINTER(VocoderShape), c_void_p, c_void_p, c_void_p]),
    'b200tts_gl_stream_workspace_bytes': (c_size_t, [POINTER(GLStreamShape)]),
    'b200tts_gl_stream_reset': (c_int, [POINTER(GLStreamShape), c_void_p, c_size_t, POINTER(c_int), c_int, c_void_p]),
    'b200tts_gl_stream_run': (c_int, [POINTER(GLStreamShape), POINTER(GLStreamRow), c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    'b200tts_analysis_workspace_bytes': (c_size_t, [POINTER(AnalysisShape)]),
    'b200tts_stft_magnitude': (c_int, [POINTER(AnalysisShape), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    'b200tts_amplitude_to_db': (c_int, [POINTER(AnalysisShape), c_void_p, c_void_p, c_void_p, c_void_p]),
    'b200tts_mel_cepstrum': (c_int, [c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    'b200tts_mel_cepstral_distortion': (c_int, [c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'b200tts_monotonic_alignment': (c_int, [POINTER(AlignShape)] + [c_void_p] * 7),
    'b200tts_alignment_scores': (c_int, [POINTER(AlignShape)] + [c_void_p] * 8),
    'b200tts_pitch_workspace_bytes': (c_size_t, [POINTER(PitchShape)]),
    'b200tts_pitch_cmnd': (c_int, [POINTER(PitchShape)] + [c_void_p] * 5),
    'b200tts_pitch_observations': (c_int, [POINTER(PitchShape)] + [c_void_p] * 4),
    'b200tts_pitch_viterbi': (c_int, [POINTER(PitchShape)] + [c_void_p] * 6 + [c_size_t, c_void_p]),
    'b200tts_psola_workspace_bytes': (c_size_t, [POINTER(PsolaShape)]),
    'b200tts_psola_marks': (c_int, [POINTER(PsolaShape)] + [c_void_p] * 6 + [c_size_t, c_void_p]),
    'b200tts_psola_overlap_add': (c_int, [POINTER(PsolaShape)] + [c_void_p] * 3 + [c_size_t, c_void_p, c_void_p]),
    'b200tts_wsola_positions': (c_int, [POINTER(WsolaShape)] + [c_void_p] * 6),
    'b200tts_wsola_overlap_add': (c_int, [POINTER(WsolaShape)] + [c_void_p] * 7),
    'b200tts_resample': (c_int, [POINTER(ResampleShape)] + [c_void_p] * 7),
    'b200tts_trim_silence': (c_int, [POINTER(TrimShape)] + [c_void_p] * 6),
    'b200tts_wavernn_upsample_layer': (c_int, [c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    'b200tts_wavernn_fold': (c_int, [POINTER(WaveRNNFoldShape)] + [c_void_p] * 7 + [c_int, c_int, c_void_p, c_void_p]),
    'b200tts_wavernn_workspace_bytes': (c_size_t, [POINTER(WaveRNNShape)]),
    'b200tts_wavernn_prepare': (c_int, [POINTER(WaveRNNShape), POINTER(WaveRNNParams), c_void_p, c_size_t, c_void_p]),
    'b200tts_wavernn_run': (c_int, [POINTER(WaveRNNShape), POINTER(WaveRNNParams), POINTER(WaveRNNCond), c_int, c_int, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_size_t, c_void_p]),
    'b200tts_wavernn_run_stream': (c_int, [POINTER(WaveRNNShape), POINTER(WaveRNNParams), POINTER(WaveRNNCond), c_longlong, c_int, c_void_p,
                                           c_void_p, c_void_p, c_size_t, c_void_p]),
    'b200tts_wavernn_run_rows': (c_int, [POINTER(WaveRNNShape), POINTER(WaveRNNParams), POINTER(WaveRNNCond), c_void_p, c_void_p, c_int, c_int,
                                         c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    'b200tts_wavernn_reset_rows': (c_int, [POINTER(WaveRNNShape), c_void_p, c_size_t, POINTER(c_int), c_int, c_void_p]),
    'b200tts_wavernn_window_rows': (c_int, [POINTER(WaveRNNWindowRow), c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'b200tts_wavernn_upsample_segments': (c_int, [c_int, c_int, POINTER(c_int), c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    'b200tts_wavernn_aborted': (c_int, [POINTER(WaveRNNShape), c_void_p, c_size_t, POINTER(c_int), c_void_p]),
    'b200tts_wavernn_deemphasis': (c_int, [c_int, c_int, c_int, c_float, c_void_p, c_void_p]),
    'b200tts_wavernn_unfold': (c_int, [c_int] * 5 + [c_void_p] * 3 + [c_longlong, c_void_p, c_void_p, c_void_p]),
    'b200tts_wavernn_unfold_streams': (c_int, [c_int] * 5 + [POINTER(WaveRNNUnfoldStream), c_void_p, c_void_p, c_int, c_longlong, c_void_p,
                                                          c_void_p, c_void_p]),
    'b200tts_gru_seq_saved_bytes': (c_size_t, [POINTER(GRUSeqShape)]),
    'b200tts_gru_seq_workspace_bytes': (c_size_t, [POINTER(GRUSeqShape)]),
    'b200tts_gru_seq_forward': (c_int, [POINTER(GRUSeqShape)] + [c_void_p] * 6 + [c_size_t, c_void_p]),
    'b200tts_gru_seq_backward': (c_int, [POINTER(GRUSeqShape)] + [c_void_p] * 8 + [c_size_t, c_void_p]),
    'b200tts_gru_seq_aborted': (c_int, [POINTER(GRUSeqShape), c_void_p, c_size_t, POINTER(c_int), c_void_p]),
    'b200tts_gru_seq_abort_flag_copy': (c_int, [POINTER(GRUSeqShape), c_void_p, c_size_t, c_void_p, c_void_p]),
    'b200tts_wavernn_cut_windows': (c_int, [c_int] * 7 + [c_void_p, c_longlong] + [c_void_p] * 8),
    'b200tts_wavernn_upsample_layer_backward_workspace_bytes': (c_size_t, [c_int, c_int, c_int]),
    'b200tts_wavernn_upsample_layer_backward': (c_int, [c_int] * 3 + [c_void_p] * 6 + [c_size_t, c_void_p]),
    'b200tts_wavernn_stretch_backward': (c_int, [c_int] * 4 + [c_void_p] * 3),
    'b200tts_wavernn_loss_workspace_bytes': (c_size_t, [c_longlong]),
    'b200tts_column_sum_workspace_bytes': (c_size_t, [c_int]),
    'b200tts_column_sum': (c_int, [c_longlong, c_int, c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    'b200tts_wavernn_loss': (c_int, [c_int, c_longlong, c_int] + [c_void_p] * 5 + [c_size_t, c_void_p]),
}

_lib = None


def load():
    """Load (once) and return the shared library; raise B200TTSError if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise B200TTSError(f'{LIB_PATH} is missing: run `python -m multilingual_text_to_speech_b200.build` '
                           '(or __graft_entry__.build()); there is no fallback path')
    try:
        lib = ctypes.CDLL(LIB_PATH)
    except OSError as exc:
        raise B200TTSError(f'cannot load {LIB_PATH}: {exc}') from exc
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(lib, name)      # AttributeError if the symbol is absent
        fn.restype, fn.argtypes = restype, argtypes
    _lib = lib
    return lib


def check(status, what):
    if status != 0:
        msg = load().b200tts_last_error()
        raise B200TTSError(f'{what} failed with status {status}: {msg.decode() if msg else ""}')


def ptr(t):
    """Device/host pointer of a torch tensor (None -> NULL)."""
    return None if t is None else c_void_p(t.data_ptr())


PRECISIONS = {'fp32': 0, 'bf16': 1}


_scratch = None


def ensure_scratch(nbytes=3 << 29):
    """Device scratch for the wgmma GEMM's packed bf16 operands (owned here, handed to the library)."""
    global _scratch
    import torch
    if _scratch is None or _scratch.numel() < nbytes:
        _scratch = torch.empty(nbytes + 1024, dtype=torch.uint8, device='cuda')
        base = (_scratch.data_ptr() + 1023) // 1024 * 1024
        check(load().b200tts_set_scratch(c_void_p(base), nbytes), 'b200tts_set_scratch')
    return _scratch


def set_precision(name):
    check(load().b200tts_set_precision(PRECISIONS[name]), 'b200tts_set_precision')
    if name == 'bf16':
        import torch
        if torch.cuda.is_available():
            ensure_scratch()


def set_tensor_core_gemm(enabled):
    check(load().b200tts_set_tensor_core_gemm(int(bool(enabled))), 'b200tts_set_tensor_core_gemm')


def get_precision():
    return {v: k for k, v in PRECISIONS.items()}[load().b200tts_get_precision()]


def kernel_timing(enable):
    check(load().b200tts_kernel_timing(int(bool(enable))), 'b200tts_kernel_timing')


def kernel_timing_read():
    """{kernel name: (total ms, launches)} collected since kernel_timing(True); synchronize the device first."""
    import ctypes
    lib, out, i = load(), {}, 0
    while True:
        name = ctypes.create_string_buffer(128)
        ms, cnt = c_float(0), c_int(0)
        st = lib.b200tts_kernel_timing_read(i, name, 128, ctypes.byref(ms), ctypes.byref(cnt))
        if st == 1:
            return out
        check(st, 'b200tts_kernel_timing_read')
        out[name.value.decode()] = (ms.value, cnt.value)
        i += 1


def launch_count():
    return int(load().b200tts_launch_count())
