"""ctypes binding of the C ABI declared in include/tfr_b200.h.

The CUDA library is the product: if `libtfr_b200.so` is missing this module
raises at import time (there is no CPU fallback).  Build it with
`python -c "import __graft_entry__ as g; g.build()"` from the repo root.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libtfr_b200.so')

if not os.path.exists(LIB_PATH):
  raise ImportError(
      'ranking_b200: %s not found. The CUDA extension is required (no CPU '
      'fallback exists); build it with __graft_entry__.build().' % LIB_PATH)

lib = C.CDLL(LIB_PATH)

# enums (mirror include/tfr_b200.h)
PHI_LOGISTIC, PHI_HINGE, PHI_SOFT_ZERO_ONE, PHI_MSE = 0, 1, 2, 3
(LAMBDA_NONE, LAMBDA_LABEL_DIFF, LAMBDA_DCG, LAMBDA_DCG_V2, LAMBDA_YETI,
 LAMBDA_PRECISION) = range(6)
GAIN_IDENTITY, GAIN_POW2_MINUS_1, GAIN_TABLE = 0, 1, 2
DISC_INVERSE, DISC_LOG2_INVERSE, DISC_LOG1P_INVERSE, DISC_TABLE = 0, 1, 2, 3
PREC_FP32, PREC_TF32X3, PREC_TF32, PREC_BF16, PREC_FP16 = 0, 1, 2, 3, 4
ACT_NONE, ACT_RELU = 0, 1
MLP_MAX_LAYERS = 8
GAM_MAX_FEATURES, GAM_MAX_HIDDEN, GAM_MAX_CONTEXT = 512, 4, 16


class LambdaCfg(C.Structure):
  _fields_ = [('kind', C.c_int32), ('topn', C.c_int32), ('gain_fn', C.c_int32),
              ('disc_fn', C.c_int32), ('normalized', C.c_int32),
              ('smooth_fraction', C.c_float), ('gain_table', C.c_void_p),
              ('disc_table', C.c_void_p)]


class FeatureSpec(C.Structure):
  _fields_ = [('name', C.c_char_p), ('dim', C.c_int32), ('default_value', C.c_float)]


class TokenSpec(C.Structure):
  _fields_ = [('name', C.c_char_p), ('max_tokens', C.c_int32), ('vocab', C.c_void_p)]


COMBINER_SUM, COMBINER_MEAN, COMBINER_SQRTN = 0, 1, 2


class MetricExt(C.Structure):
  _fields_ = [(k, C.c_void_p) for k in ('dcg', 'precision', 'recall', 'map', 'hits',
                                        'arp', 'opa', 'bpref', 'bpref_alt')]


class MlpCfg(C.Structure):
  _fields_ = [('n_dense', C.c_int32), ('dims', C.c_int32 * (MLP_MAX_LAYERS + 1)),
              ('activation', C.c_int32),
              ('use_batch_norm', C.c_int32), ('input_batch_norm', C.c_int32),
              ('bn_epsilon', C.c_float), ('bn_momentum', C.c_float),
              ('dropout', C.c_float), ('training', C.c_int32),
              ('dropout_seed', C.c_uint64), ('bn_state', C.c_void_p)]


class GamCfg(C.Structure):
  _fields_ = [('n_features', C.c_int32),
              ('feature_offsets', C.c_int32 * (GAM_MAX_FEATURES + 1)),
              ('n_hidden', C.c_int32), ('hidden', C.c_int32 * GAM_MAX_HIDDEN),
              ('n_context', C.c_int32), ('context_dims', C.c_int32 * GAM_MAX_CONTEXT),
              ('n_context_hidden', C.c_int32),
              ('context_hidden', C.c_int32 * (MLP_MAX_LAYERS - 1)),
              ('activation', C.c_int32), ('use_batch_norm', C.c_int32),
              ('bn_epsilon', C.c_float), ('bn_momentum', C.c_float),
              ('dropout', C.c_float), ('training', C.c_int32),
              ('dropout_seed', C.c_uint64), ('bn_state', C.c_void_p)]


DIN_MAX_LAYERS, DIN_MAX_HH, DIN_MAX_LIST = 8, 512, 1024


class DinCfg(C.Structure):
  _fields_ = [('input_dim', C.c_int32), ('head_size', C.c_int32), ('num_heads', C.c_int32),
              ('num_layers', C.c_int32), ('dropout', C.c_float),
              ('input_noise_stddev', C.c_float), ('training', C.c_int32),
              ('seed', C.c_uint64), ('precision', C.c_int32)]


class DasalcCfg(C.Structure):
  _fields_ = [('input_dim', C.c_int32), ('hidden_dim', C.c_int32), ('context_dim', C.c_int32),
              ('dropout', C.c_float), ('input_noise_stddev', C.c_float),
              ('bn_epsilon', C.c_float), ('bn_momentum', C.c_float), ('training', C.c_int32),
              ('seed', C.c_uint64), ('bn_state', C.c_void_p)]


class BertCfg(C.Structure):
  _fields_ = [('vocab_size', C.c_int32), ('hidden_size', C.c_int32), ('num_heads', C.c_int32),
              ('intermediate_size', C.c_int32), ('num_layers', C.c_int32),
              ('max_position', C.c_int32), ('type_vocab_size', C.c_int32),
              ('hidden_dropout', C.c_float), ('attention_dropout', C.c_float),
              ('output_dropout', C.c_float), ('training', C.c_int32), ('seed', C.c_uint64),
              ('precision', C.c_int32)]


_P = C.c_void_p
_I = C.c_int
_F = C.c_float

_SIGNATURES = {
    'tfr_last_error': (C.c_char_p, []),
    'tfr_version': (_I, []),
    'tfr_launch_count': (C.c_ulonglong, []),
    'tfr_pairwise_loss_fwd_bwd': (_I, [_P, _P, _P, _I, _P, _I, _I, _F, _I,
                                       C.POINTER(LambdaCfg), _F, _P, _P, _P, _P,
                                       _P, _P, _P]),
    'tfr_lambda_pair_weights': (_I, [_P, _P, _I, _I, C.POINTER(LambdaCfg), _P,
                                     _P]),
    'tfr_sorted_ranks': (_I, [_P, _P, _P, _I, _I, _P, _P]),
    'tfr_approx_loss_fwd_bwd': (_I, [_P, _P, _P, _I, _P, _I, _I, _F, _I, _F, _I,
                                     _P, _P, _P, _P]),
    'tfr_softmax_loss_fwd_bwd': (_I, [_P, _P, _P, _I, _P, _I, _I, _F,
                                      C.POINTER(LambdaCfg), _F, _I, _P, _P, _P,
                                      _P]),
    'tfr_misc_loss_fwd_bwd': (_I, [_P, _P, _P, _I, _P, _I, _I, _F, _I, _P, _P, _I, _F, _P, _P,
                                   _P, _P, _P, _P]),
    'tfr_extra_loss_fwd_bwd': (_I, [_P, _P, _P, _I, _P, _I, _I, _F, _I, _F, _F, _F, _P, _P, _P,
                                    _P]),
    'tfr_ordinal_loss_fwd_bwd': (_I, [_P, _P, _P, _I, _P, _I, _I, _I, _F, _I, _F, _P, _P, _P,
                                      _P, _P, _P]),
    'tfr_click_em_loss_fwd_bwd': (_I, [_P, _P, _I, _P, _P, _I, _P, _I, _I, _F, _F, _F, _F,
                                       _P, _P, _P, _P, _P, _P, _P]),
    'tfr_mixture_em_loss_fwd_bwd': (_I, [_P, _P, _P, _I, _P, _I, _I, _I, _F, _F, _F, _P, _P,
                                         _P, _P]),
    'tfr_gumbel_sample': (_I, [_P, _P, _I, _I, _I, _F, C.c_uint64, _I, _P, _P, _P, _P]),
    'tfr_rank_metrics': (_I, [_P, _P, _P, _I, _P, _I, _I, C.POINTER(C.c_int32),
                              _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P]),
    'tfr_rank_metrics_ext': (_I, [_P, _P, _P, _I, _P, _I, _I, C.POINTER(C.c_int32),
                                  _I, _I, _I, _P, _P, _P, _P, _P, _P, _P,
                                  C.POINTER(MetricExt), _P]),
    'tfr_div_metrics': (_I, [_P, _P, _P, _I, _P, _I, _I, _I, C.POINTER(C.c_int32), _I, _F, _I,
                             _P, _P, _P, _P, _P, _P]),
    'tfr_elwc_parse': (_I, [C.POINTER(C.c_char_p), C.POINTER(C.c_int64), _I, _I,
                            C.POINTER(FeatureSpec), _I, C.POINTER(FeatureSpec), _I, _P, _P, _P,
                            _P, _I]),
    'tfr_ranking_parse': (_I, [_I, C.POINTER(C.c_char_p), C.POINTER(C.c_int64), _I, _I,
                               C.POINTER(FeatureSpec), _I, C.POINTER(FeatureSpec), _I, _P, _P,
                               _P, _P, _I]),
    'tfr_masked_crc32c': (C.c_uint32, [C.c_char_p, C.c_size_t]),
    'tfr_vocab_create': (_I, [C.POINTER(C.c_char_p), C.POINTER(C.c_int64), _I, _I,
                              C.POINTER(C.c_void_p)]),
    'tfr_vocab_destroy': (_I, [_P]),
    'tfr_vocab_lookup': (_I, [_P, C.POINTER(C.c_char_p), C.POINTER(C.c_int64), _I, _P]),
    'tfr_ranking_parse_tokens': (_I, [_I, C.POINTER(C.c_char_p), C.POINTER(C.c_int64), _I, _I,
                                      C.POINTER(FeatureSpec), _I, C.POINTER(FeatureSpec), _I,
                                      C.POINTER(TokenSpec), _I, C.POINTER(TokenSpec), _I,
                                      _P, _P, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p),
                                      _P, _P, _P, _I]),
    'tfr_embedding_workspace_bytes': (C.c_size_t, [_I, _I, _I, _I]),
    'tfr_embedding_fwd': (_I, [_P, _I, _I, _P, _I, _I, _I, _I, _P, _I, _P, _P]),
    'tfr_embedding_bwd': (_I, [_P, _I, _I, _P, _I, _I, _I, _I, _I, _I, _P, _P, _P, _P]),
    'tfr_weighted_sum': (_I, [_P, _P, _I, _F, _P, _P]),
    'tfr_mlp_param_count': (C.c_size_t, [C.POINTER(MlpCfg)]),
    'tfr_mlp_bn_state_count': (C.c_size_t, [C.POINTER(MlpCfg)]),
    'tfr_mlp_workspace_bytes': (C.c_size_t, [C.POINTER(MlpCfg), _I]),
    'tfr_mlp_fwd': (_I, [_P, _I, C.POINTER(MlpCfg), _P, _P, _P, _P, _I, _P]),
    'tfr_mlp_bwd': (_I, [_P, _I, C.POINTER(MlpCfg), _P, _P, _P, _P, _P, _I, _P]),
    'tfr_mlp_fwd_tasks': (_I, [_P, _I, C.POINTER(MlpCfg), _P, _P, _P, _P, _I, _P]),
    'tfr_mlp_bwd_tasks': (_I, [_P, _I, C.POINTER(MlpCfg), _P, _P, _P, _P, _P, _P, _I, _P]),
    'tfr_mlp_input_grad': (_I, [C.POINTER(MlpCfg), _I, _P, _P, _I, _I, _P, _I, _I, _P]),
    'tfr_din_param_count': (C.c_size_t, [C.POINTER(DinCfg)]),
    'tfr_din_workspace_bytes': (C.c_size_t, [C.POINTER(DinCfg), _I, _I]),
    'tfr_din_fwd': (_I, [_P, _P, _I, _I, C.POINTER(DinCfg), _P, _P, _P, _I, _P]),
    'tfr_din_bwd': (_I, [_P, _P, _I, _I, C.POINTER(DinCfg), _P, _P, _I, _P, _P, _P]),
    'tfr_din_input_grad': (_I, [C.POINTER(DinCfg), _I, _I, _P, _P, _I, _I, _P, _I, _I, _P]),
    'tfr_dasalc_param_count': (C.c_size_t, [C.POINTER(DasalcCfg)]),
    'tfr_dasalc_bn_state_count': (C.c_size_t, [C.POINTER(DasalcCfg)]),
    'tfr_dasalc_workspace_bytes': (C.c_size_t, [C.POINTER(DasalcCfg), _I]),
    'tfr_dasalc_fwd': (_I, [_P, _P, _I, _I, C.POINTER(DasalcCfg), _P, _P, _P, _P, _I, _P]),
    'tfr_dasalc_bwd': (_I, [_P, _I, C.POINTER(DasalcCfg), _P, _P, _P, _P, _P, _P, _I, _I, _P]),
    'tfr_dasalc_param_count_tasks': (C.c_size_t, [C.POINTER(DasalcCfg), _I]),
    'tfr_dasalc_workspace_bytes_tasks': (C.c_size_t, [C.POINTER(DasalcCfg), _I, _I]),
    'tfr_dasalc_fwd_tasks': (_I, [_P, _P, _I, _I, C.POINTER(DasalcCfg), _P, _P, _P, _P, _I, _I,
                                  _P]),
    'tfr_dasalc_bwd_tasks': (_I, [_P, _I, C.POINTER(DasalcCfg), _P, _P, _P, _P, _P, _P, _P, _I,
                                  _I, _I, _P]),
    'tfr_symmetric_log1p_clip': (_I, [_P, C.c_size_t, _F, _P, _P]),
    'tfr_bilinear_param_count': (C.c_size_t, [_I, _I]),
    'tfr_bilinear_workspace_bytes': (C.c_size_t, [_I, _I, _I]),
    'tfr_bilinear_fwd': (_I, [_P, _P, _I, _I, _I, _P, _P, _P, _P]),
    'tfr_bilinear_bwd': (_I, [_P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _P, _P, _P]),
    'tfr_gam_param_count': (C.c_size_t, [C.POINTER(GamCfg)]),
    'tfr_gam_bn_state_count': (C.c_size_t, [C.POINTER(GamCfg)]),
    'tfr_gam_workspace_bytes': (C.c_size_t, [C.POINTER(GamCfg), _I]),
    'tfr_gam_fwd': (_I, [_P, _P, _I, C.POINTER(GamCfg), _P, _P, _P, _P, _P, _P, _P]),
    'tfr_gam_bwd': (_I, [_P, _P, _I, C.POINTER(GamCfg), _P, _P, _P, _P, _P, _P]),
    'tfr_circular_pad_gather': (_I, [_P, _P, _I, _I, _I, _P, _P, _P]),
    'tfr_group_indices': (_I, [_P, _P, _I, _I, _I, _I, _P, _P, _P]),
    'tfr_group_mlp_workspace_bytes': (C.c_size_t, [C.POINTER(MlpCfg), _I, _I, _I, _I]),
    'tfr_group_mlp_fwd': (_I, [_P, _I, _I, _I, _I, _P, _P, C.POINTER(MlpCfg), _P, _P, _P, _I,
                               _P]),
    'tfr_group_mlp_bwd': (_I, [_P, _I, _I, _I, _I, _P, _P, C.POINTER(MlpCfg), _P, _P, _P, _P,
                               _I, _P]),
    'tfr_group_mlp_check': (_I, [C.POINTER(MlpCfg), _I, _I, _I, _I, _P, _P]),
    'tfr_tc_gemm': (_I, [_P, _I, _P, _I, _P, _P, _I, _I, _I, _I, _I, _I, _I, _I, _I,
                         _P, _P, _I, _I, _I, C.c_size_t, _P, _P, _P]),
    'tfr_tc_gemm_bf16': (_I, [_P, _I, _P, _I, _P, _I, _I, _I, _I, _I, _I, _P, _I, _P, _P, _P,
                              _I, _P, _I, C.c_size_t, _P]),
    'tfr_tc_gemm_f16': (_I, [_P, _I, _P, _I, _P, _I, _I, _I, _I, _I, _I, _P, _I, _P, _P, _P,
                             _I, _P, _I, C.c_size_t, _P]),
    'tfr_attn_f16_fwd': (_I, [_P, _P, _I, _I, _I, _I, _F, C.c_uint64, _P, _P, _P]),
    'tfr_attn_f16_bwd': (_I, [_P, _P, _I, _I, _I, _I, _F, C.c_uint64, _P, _P, _P, _P, _P,
                              _P]),
    'tfr_attn_bf16_fwd': (_I, [_P, _P, _I, _I, _I, _I, _F, C.c_uint64, _P, _P, _P]),
    'tfr_attn_bf16_bwd': (_I, [_P, _P, _I, _I, _I, _I, _F, C.c_uint64, _P, _P, _P, _P, _P,
                               _P]),
    'tfr_dp_alloc': (_I, [C.c_size_t, C.POINTER(C.c_void_p), C.POINTER(C.c_ubyte * 64)]),
    'tfr_dp_open': (_I, [C.POINTER(C.c_ubyte * 64), C.POINTER(C.c_void_p)]),
    'tfr_dp_close': (_I, [_P]),
    'tfr_dp_free': (_I, [_P]),
    'tfr_allreduce_optimizer_step': (_I, [_P, _P, _I, _I, C.c_uint32, _P, _P, _P, C.c_size_t,
                                          _I, _F, _F, _F, _P]),
    'tfr_optimizer_step': (_I, [_P, _P, _P, C.c_size_t, _I, _F, _F, _F, _P]),
    'tfr_adamw_step': (_I, [_P, _P, _P, _P, _P, C.c_size_t, _F, _F, _F, _F, _F, C.c_int64, _F,
                            _P]),
    'tfr_global_norm_workspace_bytes': (C.c_size_t, [C.c_size_t]),
    'tfr_global_norm': (_I, [_P, C.c_size_t, _P, _P, C.c_size_t, _P]),
    'tfr_adamw_step_clipped': (_I, [_P, _P, _P, _P, _P, C.c_size_t, _F, _F, _F, _F, _F,
                                    C.c_int64, _F, _F, _P, _P]),
    'tfr_loss_scale_mul': (_I, [_P, C.c_size_t, _P, _P, _P]),
    'tfr_adamw_step_scaled': (_I, [_P, _P, _P, _P, _P, C.c_size_t, _F, _F, _F, _F, _F,
                                   C.c_int64, _F, _P, _P, _P]),
    'tfr_loss_scale_update': (_I, [_P, _P, _P, _P, C.c_int64, _P]),
    'tfr_bert_param_count': (C.c_size_t, [C.POINTER(BertCfg)]),
    'tfr_bert_workspace_bytes': (C.c_size_t, [C.POINTER(BertCfg), _I, _I]),
    'tfr_bert_fwd': (_I, [_P, _P, _P, _I, _I, C.POINTER(BertCfg), _P, _P, _P, _P, _P]),
    'tfr_bert_bwd': (_I, [_P, _P, _P, _I, _I, C.POINTER(BertCfg), _P, _P, _P, _P, _P]),
}

EXPORTED_SYMBOLS = sorted(_SIGNATURES)

for _name, (_res, _args) in _SIGNATURES.items():
  _fn = getattr(lib, _name)   # AttributeError here = symbol missing from the .so
  _fn.restype = _res
  _fn.argtypes = _args


def last_error():
  return lib.tfr_last_error().decode('utf-8', 'replace')


def check(status):
  """0 -> ok; argument errors -> ValueError (reference convention); else RuntimeError."""
  if status == 0:
    return
  msg = last_error()
  if status in (1, 2):
    raise ValueError(msg)
  raise RuntimeError('tfr_b200: ' + msg)


def ptr(t):
  """Device pointer of a tensor (None -> NULL)."""
  if t is None:
    return None
  return C.c_void_p(t.data_ptr())


def stream():
  return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def require_cuda(t, what):
  if not t.is_cuda:
    raise RuntimeError(
        'ranking_b200: %s must live on a CUDA device (got %s); the product '
        'path has no CPU implementation.' % (what, t.device))
