"""ctypes binding of libcapb200.so (C ABI: include/capb200.h).  There is no CPU fallback: if the library is missing
or a call fails the error surfaces as a RuntimeError, which the reference's training loop already turns into a
checkpoint-and-exit (tools/train.py:287-292)."""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_double, c_float, c_int, c_long, c_longlong, c_ulonglong, c_void_p

PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(PKG, 'libcapb200.so')

MODE_SIMT_FP32, MODE_TC_F16X3, MODE_TC_F16X1 = 0, 1, 2
MODES = {'simt_fp32': MODE_SIMT_FP32, 'tc_f16x3': MODE_TC_F16X3, 'tc_f16x1': MODE_TC_F16X1}
# capb200_linear additionally exposes the training step's split-K GEMM variants
OP_MODES = dict(MODES, skinny_tf32x3=3, skinny_fp32=4, tf32x3_tc=5, tf32x3_tc_dgrad=6, tf32x3_tc_wgrad=7)
FAMILY_UPDOWN, FAMILY_NEWFC, FAMILY_ATT2IN2 = 0, 1, 2
FAMILY_AOA = 3                    # ensemble members only (capb200_ensemble_member)
ENSEMBLE_MAX_MEMBERS = 8
SAMPLE_GREEDY, SAMPLE_MULTINOMIAL, SAMPLE_FORCED, SAMPLE_TEACHER, SAMPLE_TOPK, SAMPLE_TOPP = 0, 1, 2, 3, 4, 5


class ModelCfg(Structure):
    _fields_ = [('family', c_int), ('vocab_size', c_int), ('input_encoding_size', c_int), ('rnn_size', c_int), ('att_hid_size', c_int),
                ('fc_feat_size', c_int), ('att_feat_size', c_int), ('seq_length', c_int), ('numeric_mode', c_int)]


WEIGHT_FIELDS = ['embed', 'fc_embed_w', 'fc_embed_b', 'att_embed_w', 'att_embed_b', 'ctx2att_w', 'ctx2att_b', 'logit_w', 'logit_b',
                 'att_lstm_w_ih', 'att_lstm_w_hh', 'att_lstm_b_ih', 'att_lstm_b_hh', 'lang_lstm_w_ih', 'lang_lstm_w_hh', 'lang_lstm_b_ih',
                 'lang_lstm_b_hh', 'h2att_w', 'h2att_b', 'alpha_w', 'alpha_b', 'i2h_w', 'i2h_b', 'h2h_w', 'h2h_b', 'a2c_w', 'a2c_b']


class Weights(Structure):
    _fields_ = [(f, c_void_p) for f in WEIGHT_FIELDS]


class DecodeEdits(Structure):
    _fields_ = [('decoding_constraint', c_int), ('unk_col', c_int), ('n_bad_endings', c_int), ('bad_endings', c_void_p), ('block_trigrams', c_int),
                ('trigram_rows', c_int)]

    @classmethod
    def none(cls):
        return cls(0, -1, 0, None, 0, 0)


class BeamOpts(Structure):
    _fields_ = [('beam_size', c_int), ('sample_n', c_int), ('penalty_kind', c_int), ('penalty_alpha', c_float), ('temperature', c_float),
                ('edits', DecodeEdits)]

    def __init__(self, beam_size, sample_n, penalty_kind=0, penalty_alpha=0.0, temperature=1.0, edits=None):
        super().__init__(beam_size, sample_n, penalty_kind, penalty_alpha, temperature, edits if edits is not None else DecodeEdits.none())


class DiverseOpts(Structure):
    _fields_ = [('base', BeamOpts), ('group_size', c_int), ('diversity_lambda', c_float)]

    def __init__(self, base, group_size, diversity_lambda):
        super().__init__(base, group_size, diversity_lambda)


class SampleOpts(Structure):
    _fields_ = [('sample_n', c_int), ('method', c_int), ('temperature', c_float), ('seed', c_ulonglong), ('steps', c_int), ('top', c_float),
                ('edits', DecodeEdits)]

    def __init__(self, sample_n, method, temperature=1.0, seed=0, steps=0, top=0.0, edits=None):
        super().__init__(sample_n, method, temperature, seed, steps, top, edits if edits is not None else DecodeEdits.none())


class EnsembleMember(Structure):
    _fields_ = [('family', c_int), ('engine', c_void_p), ('weight', c_float)]


class RewardWeights(Structure):
    _fields_ = [('cider', c_double), ('bleu', c_double)]


class SamplerOpts(Structure):
    _fields_ = [('train_method', c_int), ('train_top', c_float), ('baseline_method', c_int), ('baseline_top', c_float), ('forced_baseline', c_void_p)]


class ScstOpts(Structure):
    _fields_ = [('sample_n', c_int), ('temperature', c_float), ('seed', c_ulonglong), ('drop_prob', c_float), ('upstream', c_float), ('baseline', c_int),
                ('forced_tokens', c_void_p), ('att_masks', c_void_p), ('keep_rows', c_int), ('row_loss', c_void_p),
                ('sampler', POINTER(SamplerOpts)), ('reward_weights', POINTER(RewardWeights))]


BASELINE_GREEDY, BASELINE_LEAVE_ONE_OUT = 0, 1


class PpoOpts(Structure):
    _fields_ = [('cliprange', c_float), ('kl_coef', c_float)]


class AoaScstOpts(Structure):
    _fields_ = [('sample_n', c_int), ('temperature', c_float), ('seed', c_ulonglong), ('upstream', c_float), ('baseline', c_int),
                ('drop_prob_lm', c_float), ('drop_attn', c_float), ('drop_aoa', c_float), ('drop_sublayer', c_float), ('ctx_drop', c_int),
                ('forced_tokens', c_void_p), ('att_masks', c_void_p), ('keep_rows', c_int), ('row_loss', c_void_p),
                ('sampler', POINTER(SamplerOpts)), ('reward_weights', POINTER(RewardWeights))]


class AoaXeOpts(Structure):
    _fields_ = [('seq_per_img', c_int), ('steps', c_int), ('seed', c_ulonglong), ('label_smoothing', c_float), ('upstream', c_float),
                ('drop_prob_lm', c_float), ('drop_attn', c_float), ('drop_aoa', c_float), ('drop_sublayer', c_float), ('ctx_drop', c_int),
                ('att_masks', c_void_p), ('ss_prob', c_float), ('tokens_used', c_void_p), ('keep_rows', c_int), ('row_loss', c_void_p)]


class XeOpts(Structure):
    _fields_ = [('seq_per_img', c_int), ('steps', c_int), ('seed', c_ulonglong), ('drop_prob', c_float), ('label_smoothing', c_float),
                ('upstream', c_float), ('att_masks', c_void_p), ('ss_prob', c_float), ('tokens_used', c_void_p), ('keep_rows', c_int), ('row_loss', c_void_p)]


GRAD_FIELDS = ['embed', 'fc_embed_w', 'fc_embed_b', 'att_embed_w', 'att_embed_b', 'ctx2att_w', 'ctx2att_b', 'logit_w', 'logit_b',
               'att_lstm_w_ih', 'att_lstm_w_hh', 'att_lstm_b_ih', 'att_lstm_b_hh', 'lang_lstm_w_ih', 'lang_lstm_w_hh', 'lang_lstm_b_ih',
               'lang_lstm_b_hh', 'h2att_w', 'h2att_b', 'alpha_w', 'alpha_b']


class UpdownGrads(Structure):
    _fields_ = [(f, c_void_p) for f in GRAD_FIELDS]


ATT2IN2_GRAD_FIELDS = ['embed', 'att_embed_w', 'att_embed_b', 'ctx2att_w', 'ctx2att_b', 'logit_w', 'logit_b', 'h2att_w', 'h2att_b', 'alpha_w', 'alpha_b',
                       'i2h_w', 'i2h_b', 'h2h_w', 'h2h_b', 'a2c_w', 'a2c_b']


class Att2in2Grads(Structure):
    _fields_ = [(f, c_void_p) for f in ATT2IN2_GRAD_FIELDS]


NEWFC_GRAD_FIELDS = ['embed', 'fc_embed_w', 'fc_embed_b', 'logit_w', 'logit_b', 'i2h_w', 'i2h_b', 'h2h_w', 'h2h_b']


class NewfcGrads(Structure):
    _fields_ = [(f, c_void_p) for f in NEWFC_GRAD_FIELDS]


TFM_MAX_LAYERS = 8


class TfmCfg(Structure):
    _fields_ = [(f, c_int) for f in ('vocab_size', 'd_model', 'd_ff', 'heads', 'n_enc', 'n_dec', 'att_feat_size', 'seq_length', 'numeric_mode')]


class MhaWeights(Structure):
    _fields_ = [(f, c_void_p) for f in ('q_w', 'q_b', 'k_w', 'k_b', 'v_w', 'v_b', 'o_w', 'o_b')]


class TfmEncLayer(Structure):
    _fields_ = [('self_attn', MhaWeights)] + [(f, c_void_p) for f in ('w1_w', 'w1_b', 'w2_w', 'w2_b', 'ln0_a', 'ln0_b', 'ln1_a', 'ln1_b')]


class TfmDecLayer(Structure):
    _fields_ = [('self_attn', MhaWeights), ('src_attn', MhaWeights)] + \
               [(f, c_void_p) for f in ('w1_w', 'w1_b', 'w2_w', 'w2_b', 'ln0_a', 'ln0_b', 'ln1_a', 'ln1_b', 'ln2_a', 'ln2_b')]


class TfmWeights(Structure):
    _fields_ = [('att_embed_w', c_void_p), ('att_embed_b', c_void_p), ('enc', TfmEncLayer * TFM_MAX_LAYERS), ('enc_norm_a', c_void_p),
                ('enc_norm_b', c_void_p), ('dec', TfmDecLayer * TFM_MAX_LAYERS), ('dec_norm_a', c_void_p), ('dec_norm_b', c_void_p),
                ('lut', c_void_p), ('pe', c_void_p), ('gen_w', c_void_p), ('gen_b', c_void_p)]


class TfmXeOpts(Structure):
    _fields_ = [('seq_per_img', c_int), ('seed', c_ulonglong), ('label_smoothing', c_float), ('upstream', c_float), ('drop_prob_lm', c_float),
                ('dropout', c_float), ('att_masks', c_void_p), ('keep_rows', c_int), ('row_loss', c_void_p)]


class TfmScstOpts(Structure):
    _fields_ = [('sample_n', c_int), ('temperature', c_float), ('seed', c_ulonglong), ('upstream', c_float), ('baseline', c_int),
                ('drop_prob_lm', c_float), ('dropout', c_float), ('forced_tokens', c_void_p), ('att_masks', c_void_p), ('keep_rows', c_int),
                ('row_loss', c_void_p), ('sampler', POINTER(SamplerOpts)), ('reward_weights', POINTER(RewardWeights))]


class VjpOpts(Structure):
    _fields_ = [('forward_only', c_int), ('dlogprobs', c_void_p), ('greedy', c_int)]


AOA_REFINER_LAYERS = 6


class AoaCfg(Structure):
    _fields_ = [(f, c_int) for f in ('vocab_size', 'input_encoding_size', 'rnn_size', 'heads', 'att_feat_size', 'seq_length', 'numeric_mode')]


class AoaRefinerLayer(Structure):
    _fields_ = [(f, c_void_p) for f in ('q_w', 'q_b', 'k_w', 'k_b', 'v_w', 'v_b', 'aoa_w', 'aoa_b', 'ln_a', 'ln_b')]


class AoaWeights(Structure):
    _fields_ = [('embed', c_void_p), ('att_embed_w', c_void_p), ('att_embed_b', c_void_p), ('refiner', AoaRefinerLayer * AOA_REFINER_LAYERS)] + \
               [(f, c_void_p) for f in ('refiner_norm_a', 'refiner_norm_b', 'ctx2att_w', 'ctx2att_b', 'att_lstm_w_ih', 'att_lstm_w_hh', 'att_lstm_b_ih',
                                        'att_lstm_b_hh', 'attn_norm_a', 'attn_norm_b', 'attn_q_w', 'attn_q_b', 'att2ctx_w', 'att2ctx_b', 'logit_w',
                                        'logit_b')]


class GemmEpilogue(Structure):
    _fields_ = [('bias', c_void_p), ('row_bias', c_void_p), ('ld_row_bias', c_long), ('rows_per_group', c_int), ('residual', c_void_p),
                ('ld_res', c_long), ('relu', c_int), ('C', c_void_p), ('ldc', c_long), ('C_hi', c_void_p), ('C_lo', c_void_p), ('ldcs', c_long),
                ('lstm', c_int), ('H', c_int), ('c_prev', c_void_p), ('ld_cprev', c_long), ('src_row', c_void_p), ('c_out', c_void_p),
                ('ld_cout', c_long), ('gather_bias', c_void_p), ('ld_gb', c_long), ('gather_idx', c_void_p), ('h_f', c_void_p), ('h_hi', c_void_p),
                ('h_lo', c_void_p), ('ld_h', c_long)]


# every exported symbol of include/capb200.h: (restype, argtypes)
SIGNATURES = {
    'capb200_last_error': (c_char_p, []),
    'capb200_abi_version': (c_int, []),
    'capb200_range_status': (c_int, [c_int]),
    'capb200_linear': (c_int, [c_void_p, c_long, c_void_p, c_long, c_void_p, c_void_p, c_long, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    'capb200_bench_linear': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    'capb200_gemm_tile_n': (c_int, [c_int, c_int]),
    'capb200_gemm_tile_m': (c_int, [c_int, c_int]),
    'capb200_lstm_cell': (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int,
                                  c_int, c_void_p]),
    'capb200_additive_attention': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                           c_void_p]),
    'capb200_log_softmax_topk': (c_int, [c_void_p, c_long, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    'capb200_vocab_stats_topk': (c_int, [c_void_p, c_long, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    'capb200_vocab_select': (c_int, [c_void_p, c_long, c_int, c_int, c_int, c_float, c_float, c_ulonglong, c_ulonglong, c_void_p, c_int, c_void_p,
                                     c_void_p, c_void_p]),
    'capb200_engine_create': (c_void_p, [POINTER(ModelCfg)]),
    'capb200_engine_destroy': (None, [c_void_p]),
    'capb200_engine_bind_weights': (c_int, [c_void_p, POINTER(Weights), c_void_p]),
    'capb200_engine_set_logit_layers': (c_int, [c_void_p, c_int]),
    'capb200_engine_bind_logit_head': (c_int, [c_void_p, POINTER(c_void_p), POINTER(c_void_p), c_void_p]),
    'capb200_engine_bind_logit_head_grads': (c_int, [c_void_p, POINTER(c_void_p), POINTER(c_void_p)]),
    'capb200_engine_set_logit_dropout': (c_int, [c_void_p, c_float]),
    'capb200_decode_beam': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(BeamOpts), c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_void_p]),
    'capb200_decode_beam_form': (c_int, [c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(BeamOpts), c_void_p, c_void_p, c_void_p,
                                         c_void_p, c_void_p, c_void_p, c_void_p]),
    'capb200_beam_record_logprobs': (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    'capb200_decode_beam_diverse': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(DiverseOpts), c_void_p, c_void_p, c_void_p,
                                            c_void_p, c_void_p, c_void_p, c_void_p]),
    'capb200_decode_sample': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(SampleOpts), c_void_p, c_long, c_void_p, c_void_p,
                                      c_void_p, c_void_p]),
    'capb200_engine_launch_count': (c_long, [c_void_p]),
    'capb200_engine_set_profiling': (c_int, [c_void_p, c_int]),
    'capb200_engine_read_profile': (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int]),
    'capb200_tfm_create': (c_void_p, [POINTER(TfmCfg)]),
    'capb200_tfm_destroy': (None, [c_void_p]),
    'capb200_tfm_bind_weights': (c_int, [c_void_p, POINTER(TfmWeights), c_void_p]),
    'capb200_tfm_decode_beam': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(BeamOpts), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                        c_void_p, c_void_p]),
    'capb200_tfm_beam_record_logprobs': (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    'capb200_tfm_decode_sample': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(SampleOpts), c_void_p, c_long, c_void_p, c_void_p, c_void_p,
                                          c_void_p]),
    'capb200_tfm_launch_count': (c_long, [c_void_p]),
    'capb200_aoa_create': (c_void_p, [POINTER(AoaCfg)]),
    'capb200_aoa_destroy': (None, [c_void_p]),
    'capb200_aoa_bind_weights': (c_int, [c_void_p, POINTER(AoaWeights), c_void_p]),
    'capb200_aoa_set_logit_layers': (c_int, [c_void_p, c_int]),
    'capb200_aoa_bind_logit_head': (c_int, [c_void_p, POINTER(c_void_p), POINTER(c_void_p), c_void_p]),
    'capb200_aoa_bind_logit_head_grads': (c_int, [c_void_p, POINTER(c_void_p), POINTER(c_void_p)]),
    'capb200_aoa_set_logit_dropout': (c_int, [c_void_p, c_float]),
    'capb200_aoa_decode_beam': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(BeamOpts), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                        c_void_p, c_void_p]),
    'capb200_aoa_beam_record_logprobs': (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    'capb200_aoa_decode_beam_diverse': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(DiverseOpts), c_void_p, c_void_p, c_void_p, c_void_p,
                                                c_void_p, c_void_p, c_void_p]),
    'capb200_aoa_decode_sample': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(SampleOpts), c_void_p, c_long, c_void_p, c_void_p, c_void_p,
                                          c_void_p]),
    'capb200_aoa_scst_step': (c_int, [c_void_p, c_void_p, c_int, c_int, POINTER(AoaScstOpts), c_void_p, c_void_p, c_void_p, c_int, POINTER(AoaWeights),
                                      c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'capb200_aoa_xe_step': (c_int, [c_void_p, c_void_p, c_int, c_int, POINTER(AoaXeOpts), c_void_p, c_void_p, c_int, POINTER(AoaWeights), c_void_p,
                                    c_void_p, c_void_p]),
    'capb200_aoa_launch_count': (c_long, [c_void_p]),
    'capb200_ensemble_create': (c_void_p, []),
    'capb200_ensemble_destroy': (None, [c_void_p]),
    'capb200_ensemble_decode_beam': (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(BeamOpts), c_void_p, c_void_p,
                                             c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'capb200_ensemble_beam_record_logprobs': (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    'capb200_ensemble_decode_sample': (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(SampleOpts), c_void_p, c_long,
                                               c_void_p, c_void_p, c_void_p, c_void_p]),
    'capb200_ensemble_launch_count': (c_long, [c_void_p]),
    'capb200_updown_scst_step': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(ScstOpts), c_void_p, c_void_p, c_void_p, c_int,
                                         POINTER(UpdownGrads), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'capb200_att2in2_scst_step': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(ScstOpts), c_void_p, c_void_p, c_void_p, c_int,
                                          POINTER(Att2in2Grads), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'capb200_att2in2_xe_step': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(XeOpts), c_void_p, c_void_p, c_int, POINTER(Att2in2Grads),
                                        c_void_p, c_void_p, c_void_p]),
    'capb200_newfc_scst_step': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(ScstOpts), c_void_p, c_void_p, c_void_p, c_int,
                                        POINTER(NewfcGrads), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'capb200_newfc_xe_step': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(XeOpts), c_void_p, c_void_p, c_int, POINTER(NewfcGrads),
                                      c_void_p, c_void_p, c_void_p]),
    'capb200_dropout_mask': (c_int, [c_void_p, c_long, c_ulonglong, c_int, c_int, c_float, c_void_p]),
    'capb200_mha_forward': (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_long, c_void_p, c_long, c_ulonglong, c_int,
                                    c_float, c_void_p, c_long, c_void_p]),
    'capb200_mha_self_backward': (c_int, [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_long, c_void_p, c_long, c_ulonglong, c_int,
                                          c_float, c_void_p, c_long, c_void_p, c_void_p, c_void_p, c_long, c_void_p]),
    'capb200_mha_cross_backward': (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_long, c_void_p, c_void_p, c_long, c_ulonglong,
                                           c_int, c_int, c_float, c_void_p, c_void_p, c_long, c_void_p, c_long, c_void_p, c_void_p, c_long, c_void_p]),
    'capb200_mha_causal_forward': (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_long, c_void_p, c_long,
                                           c_ulonglong, c_int, c_float, c_void_p, c_long, c_void_p]),
    'capb200_mha_causal_backward': (c_int, [c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_long, c_void_p, c_long, c_ulonglong,
                                            c_int, c_float, c_void_p, c_long, c_void_p, c_void_p, c_void_p, c_long, c_void_p]),
    'capb200_tfm_dec_self_attention': (c_int, [c_int, c_int, c_int, c_int, c_int, c_void_p, c_long, c_void_p, c_void_p, c_long, c_long, c_void_p,
                                               c_long, c_void_p, c_long, c_void_p, c_long, c_void_p]),
    'capb200_tfm_xe_step': (c_int, [c_void_p, c_void_p, c_int, c_int, POINTER(TfmXeOpts), c_void_p, c_void_p, c_int, POINTER(TfmWeights), c_void_p, c_void_p,
                                    c_void_p]),
    'capb200_tfm_scst_step': (c_int, [c_void_p, c_void_p, c_int, c_int, POINTER(TfmScstOpts), c_void_p, c_void_p, c_void_p, c_int, POINTER(TfmWeights),
                                      c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'capb200_tfm_set_grad_events': (c_int, [c_void_p, c_void_p, c_int]),
    'capb200_adam_chunk_elems': (c_int, []),
    'capb200_adam_step': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_double, c_double, c_double, c_double, c_double, c_long, c_double, c_int, c_void_p]),
    'capb200_engine_set_grad_events': (c_int, [c_void_p, c_void_p, c_int]),
    'capb200_aoa_set_grad_events': (c_int, [c_void_p, c_void_p, c_int]),
    'capb200_cider_table_create': (c_void_p, [c_void_p, c_void_p, c_long, c_double, c_void_p]),
    'capb200_cider_table_destroy': (None, [c_void_p]),
    'capb200_cider_corpus_table_create': (c_void_p, []),
    'capb200_cider_table_reserve': (c_int, [c_void_p, c_long, c_int]),
    'capb200_cider_table_is_corpus': (c_int, [c_void_p]),
    'capb200_cider_scores': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    'capb200_bleu4_scores': (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    'capb200_weighted_reward': (c_int, [c_void_p, POINTER(RewardWeights), c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p,
                                        c_void_p, c_void_p, c_void_p]),
    'capb200_updown_xe_step': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(XeOpts), c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                       c_void_p, c_void_p]),
    'capb200_self_critical_reward': (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p,
                                             c_void_p]),
    'capb200_reward_criterion_forward': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    'capb200_reward_criterion_backward': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_float, c_void_p, c_void_p]),
    'capb200_self_cider': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    'capb200_self_cider_div': (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    'capb200_div_stats': (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    'capb200_coco_scores': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p]),
    'capb200_decode_gemm': (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, POINTER(GemmEpilogue), c_void_p, c_int, c_void_p]),
    # autograd entry points: (engine, [fc,] att, B, R, opts, vjp, labels, label_cols, grads, logprobs, stream) /
    #                        (engine, [fc,] att, B, R, opts, vjp, grads, sample_seq, sample_logprobs, stream)
    'capb200_updown_xe_vjp': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(XeOpts), POINTER(VjpOpts), c_void_p, c_int,
                                      POINTER(UpdownGrads), c_void_p, c_void_p]),
    'capb200_updown_scst_vjp': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(ScstOpts), POINTER(VjpOpts), POINTER(UpdownGrads),
                                        c_void_p, c_void_p, c_void_p]),
    'capb200_att2in2_xe_vjp': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(XeOpts), POINTER(VjpOpts), c_void_p, c_int,
                                       POINTER(Att2in2Grads), c_void_p, c_void_p]),
    'capb200_att2in2_scst_vjp': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(ScstOpts), POINTER(VjpOpts), POINTER(Att2in2Grads),
                                         c_void_p, c_void_p, c_void_p]),
    'capb200_newfc_xe_vjp': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(XeOpts), POINTER(VjpOpts), c_void_p, c_int,
                                     POINTER(NewfcGrads), c_void_p, c_void_p]),
    'capb200_newfc_scst_vjp': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(ScstOpts), POINTER(VjpOpts), POINTER(NewfcGrads),
                                       c_void_p, c_void_p, c_void_p]),
    'capb200_aoa_xe_vjp': (c_int, [c_void_p, c_void_p, c_int, c_int, POINTER(AoaXeOpts), POINTER(VjpOpts), c_void_p, c_int, POINTER(AoaWeights),
                                   c_void_p, c_void_p]),
    'capb200_aoa_scst_vjp': (c_int, [c_void_p, c_void_p, c_int, c_int, POINTER(AoaScstOpts), POINTER(VjpOpts), POINTER(AoaWeights), c_void_p,
                                     c_void_p, c_void_p]),
    'capb200_tfm_xe_vjp': (c_int, [c_void_p, c_void_p, c_int, c_int, POINTER(TfmXeOpts), POINTER(VjpOpts), c_void_p, c_int, POINTER(TfmWeights),
                                   c_void_p, c_void_p]),
    'capb200_tfm_scst_vjp': (c_int, [c_void_p, c_void_p, c_int, c_int, POINTER(TfmScstOpts), POINTER(VjpOpts), POINTER(TfmWeights), c_void_p,
                                     c_void_p, c_void_p]),
    # PPO steps: (engine, old engine, [fc,] att, B, R, opts, ppo, table, refs, ref_offsets, L, grads, sample_seq, sample_logprobs, scores, loss,
    #             pg_loss, kl_loss, clipfrac, stream)
    'capb200_updown_ppo_step': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(ScstOpts), POINTER(PpoOpts), c_void_p, c_void_p,
                                        c_void_p, c_int, c_void_p] + [c_void_p] * 8),
    'capb200_att2in2_ppo_step': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(ScstOpts), POINTER(PpoOpts), c_void_p, c_void_p,
                                         c_void_p, c_int, c_void_p] + [c_void_p] * 8),
    'capb200_newfc_ppo_step': (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(ScstOpts), POINTER(PpoOpts), c_void_p, c_void_p,
                                       c_void_p, c_int, c_void_p] + [c_void_p] * 8),
    'capb200_aoa_ppo_step': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(AoaScstOpts), POINTER(PpoOpts), c_void_p, c_void_p, c_void_p,
                                     c_int, c_void_p] + [c_void_p] * 8),
    'capb200_tfm_ppo_step': (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, POINTER(TfmScstOpts), POINTER(PpoOpts), c_void_p, c_void_p, c_void_p,
                                     c_int, c_void_p] + [c_void_p] * 8),
}

_lib = None


def load() -> ctypes.CDLL:
    """Loads the shared library (building is the job of __graft_entry__.build / build.py) and types every symbol."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError('capb200: %s is missing -- run `python imagecaptioning.pytorch_b200/build.py`; there is no CPU fallback' % LIB_PATH)
    lib = ctypes.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)        # AttributeError here means the library and the header disagree
        fn.restype = res
        fn.argtypes = args
    if lib.capb200_abi_version() != 1:
        raise RuntimeError('capb200: ABI version mismatch')
    _lib = lib
    return lib


def check(rc: int, what: str = '') -> None:
    if rc != 0:
        msg = load().capb200_last_error()
        raise RuntimeError('capb200 %s failed: %s' % (what, msg.decode() if msg else 'unknown error'))


def ptr(t) -> int:
    """Device (or host) address of a torch tensor / numpy array, or None."""
    if t is None:
        return None
    if hasattr(t, 'data_ptr'):
        return t.data_ptr()
    return t.ctypes.data


def current_stream() -> int:
    import torch
    return torch.cuda.current_stream().cuda_stream
