"""TFR-BERT (extension/premade/tfrbert_task.py): a BERT cross-encoder scores every (query,
document) token sequence of a list, trained end to end with a ranking loss and AdamW.

    BertEncoderConfig, BertEncoder     the encoder's sizes and its flat parameters (K15)
    TFRBertScorer                      Dropout(bert_output_dropout) + Dense(1) on the pooled
                                       [CLS] output
    TFRBertRankingTrainer              one fused step: tfr_bert_fwd, the fused loss kernel,
                                       tfr_bert_bwd, tfr_adamw_step (fp16: with dynamic loss
                                       scaling)
    TFRBertDataConfig, tfrbert_batches ELWC records with `input_ids` / `input_mask` /
                                       `segment_ids` (int64, dim seq_length) and a label

The encoder is tf-models-official's BertEncoder as TFRBertScorer uses it; its math and the
flat parameter layout are written out in include/tfr_b200.h (K15).  `set_weights` takes the
tensors in the documented order (`weight_names`); `BertEncoder.from_pretrained` and
`load_checkpoint` import a pretrained TF2 BertEncoder or Hugging Face BERT checkpoint
(bert_checkpoint.py), and `BertEncoderConfig.from_json` reads its `config.json`.
Precision: 'fp32', 'tf32', 'bf16' (the reference's 'mixed_bfloat16' policy: fp32 parameters
and optimizer, bf16 activations, GEMMs and attention core; sizes in multiples of 8) or 'fp16'
(the reference's 'mixed_float16', its choice for GPUs: the same with fp16, trained with dynamic
loss scaling).
"""
import ctypes
import dataclasses
import json
import os

import torch

from ranking_b200 import _C
from ranking_b200 import data as data_lib
from ranking_b200 import train as train_lib
from ranking_b200.extension import bert_checkpoint

_PRECISIONS = {'fp32': _C.PREC_FP32, 'tf32': _C.PREC_TF32, 'bf16': _C.PREC_BF16,
               'fp16': _C.PREC_FP16}


@dataclasses.dataclass
class BertEncoderConfig:
  """BERT-base by default (uncased_L-12_H-768_A-12)."""
  vocab_size: int = 30522
  hidden_size: int = 768
  num_layers: int = 12
  num_attention_heads: int = 12
  intermediate_size: int = 3072
  max_position_embeddings: int = 512
  type_vocab_size: int = 2
  hidden_dropout_prob: float = 0.1
  attention_dropout_prob: float = 0.1
  initializer_range: float = 0.02

  # the encoder's GELU is the tanh form; 'gelu' is the erf form in Hugging Face (and the
  # tanh form in Google's BERT code), so an HF 'gelu' model imported here differs from HF's
  # own outputs by the GELU approximation
  _HIDDEN_ACTS = ('gelu', 'gelu_new', 'gelu_pytorch_tanh')
  _JSON_KEYS = {'vocab_size': 'vocab_size', 'hidden_size': 'hidden_size',
                'num_hidden_layers': 'num_layers',
                'num_attention_heads': 'num_attention_heads',
                'intermediate_size': 'intermediate_size',
                'max_position_embeddings': 'max_position_embeddings',
                'type_vocab_size': 'type_vocab_size',
                'hidden_dropout_prob': 'hidden_dropout_prob',
                'attention_probs_dropout_prob': 'attention_dropout_prob',
                'initializer_range': 'initializer_range'}

  @classmethod
  def from_json(cls, path):
    """The config of a Google BERT `bert_config.json` or Hugging Face `config.json`
    (missing keys keep their defaults).  `hidden_act` must be 'gelu_new',
    'gelu_pytorch_tanh' or 'gelu' (see above), `layer_norm_eps` (if given) 1e-12 and
    `position_embedding_type` (if given) 'absolute'; ValueError otherwise, and for a head
    count that does not divide the hidden size."""
    with open(path) as f:
      d = json.load(f)
    act = d.get('hidden_act', 'gelu')
    if act not in cls._HIDDEN_ACTS:
      raise ValueError('%s: hidden_act %r unsupported (the encoder computes the tanh GELU: '
                       'one of %s)' % (path, act, list(cls._HIDDEN_ACTS)))
    # the encoder's LayerNorm epsilon is BERT's 1e-12 and its positions are absolute
    # (include/tfr_b200.h, K15); other values would import into a different model
    eps = float(d.get('layer_norm_eps', 1e-12))
    if eps != 1e-12:
      raise ValueError('%s: layer_norm_eps %g unsupported (the encoder uses 1e-12)' %
                       (path, eps))
    pos = d.get('position_embedding_type', 'absolute')
    if pos != 'absolute':
      raise ValueError('%s: position_embedding_type %r unsupported (absolute only)' %
                       (path, pos))
    kw = {}
    for key, field in cls._JSON_KEYS.items():
      if key in d:
        kw[field] = (float if field.endswith(('_prob', '_range')) else int)(d[key])
    c = cls(**kw)
    if c.num_attention_heads < 1 or c.hidden_size % c.num_attention_heads:
      raise ValueError('%s: hidden_size %d is not a multiple of num_attention_heads %d' %
                       (path, c.hidden_size, c.num_attention_heads))
    return c


def config_beside(checkpoint):
  """The `config.json` or `bert_config.json` in a checkpoint's directory (or in the
  directory itself), else None."""
  folder = checkpoint if os.path.isdir(checkpoint) else \
      os.path.dirname(os.path.abspath(checkpoint))
  for name in ('config.json', 'bert_config.json'):
    if os.path.isfile(os.path.join(folder, name)):
      return os.path.join(folder, name)
  return None


def weight_shapes(config):
  """[(name, shape), ...] in the flat parameter order of tfr_bert_fwd (the scorer's w_s / b_s
  included)."""
  c = config
  e, i = c.hidden_size, c.intermediate_size
  out = [('word_embeddings', (c.vocab_size, e)),
         ('position_embeddings', (c.max_position_embeddings, e)),
         ('type_embeddings', (c.type_vocab_size, e)),
         ('embeddings/layer_norm/gamma', (e,)), ('embeddings/layer_norm/beta', (e,))]
  for l in range(c.num_layers):
    p = 'transformer/layer_%d/' % l
    out += [(p + 'attention/qkv/kernel', (e, 3 * e)), (p + 'attention/qkv/bias', (3 * e,)),
            (p + 'attention/output/kernel', (e, e)), (p + 'attention/output/bias', (e,)),
            (p + 'attention_layer_norm/gamma', (e,)), (p + 'attention_layer_norm/beta', (e,)),
            (p + 'intermediate/kernel', (e, i)), (p + 'intermediate/bias', (i,)),
            (p + 'output/kernel', (i, e)), (p + 'output/bias', (e,)),
            (p + 'output_layer_norm/gamma', (e,)), (p + 'output_layer_norm/beta', (e,))]
  out += [('pooler/kernel', (e, e)), ('pooler/bias', (e,)),
          ('score/kernel', (e,)), ('score/bias', (1,))]
  return out


def _excluded_from_decay(name):
  # tf-models' BERT optimizer: exclude_from_weight_decay=['LayerNorm', 'layer_norm', 'bias']
  return 'layer_norm' in name or name.endswith('bias')


def _truncated_normal(gen, shape, stddev):
  """tf.keras TruncatedNormal: normal draws redrawn outside two standard deviations."""
  t = torch.randn(shape, generator=gen, dtype=torch.float64)
  while True:
    bad = t.abs() > 2.0
    if not bool(bad.any()):
      break
    t[bad] = torch.randn(int(bad.sum()), generator=gen, dtype=torch.float64)
  return (t * stddev).float()


class BertEncoder(object):
  """The encoder's flat parameters and configuration (pooler and score head included, so the
  scorer is one buffer: one gradient, one optimizer launch).  `precision` 'fp32' (default:
  3xTF32 GEMMs, FP32 attention core), 'tf32' (one TF32 pass, wgmma attention core), 'bf16'
  (mixed precision: bf16 activations, GEMMs and attention core on fp32 master weights, as
  Keras' 'mixed_bfloat16' policy; hidden, intermediate and head sizes must be multiples of 8)
  or 'fp16' (the same with fp16, as 'mixed_float16'; its trainer scales the loss).  The
  parameters are the same in all four, so `set_precision` can switch a trained encoder.
  Initialisation (host): truncated normal with stddev `initializer_range` for the tables and
  kernels, zero biases, LayerNorm gamma 1 / beta 0."""

  def __init__(self, config=None, seed=None, device='cuda', precision=None):
    self.config = config or BertEncoderConfig()
    self.set_precision(precision)
    cfg = self._make_cfg(0.0)
    n = _C.lib.tfr_bert_param_count(ctypes.byref(cfg))
    if n == 0:
      raise ValueError(_C.last_error())
    gen = torch.Generator()
    if seed is not None:
      gen.manual_seed(seed)
    self._base = int(seed if seed is not None else torch.seed()) & 0xFFFFFFFF
    self._calls = 0
    parts, mask = [], []
    for name, shape in weight_shapes(self.config):
      if 'layer_norm/gamma' in name:
        t = torch.ones(shape)
      elif _excluded_from_decay(name):
        t = torch.zeros(shape)
      else:
        t = _truncated_normal(gen, shape, self.config.initializer_range)
      parts.append(t.reshape(-1))
      mask.append(torch.full((t.numel(),), 0 if _excluded_from_decay(name) else 1,
                             dtype=torch.uint8))
    flat = torch.cat(parts)
    assert flat.numel() == n, (flat.numel(), n)
    self.flat = torch.nn.Parameter(flat.to(device))
    self.decay_mask = torch.cat(mask).to(device)
    self.output_dropout = 0.0
    self.dims = ['bert'] + list(dataclasses.astuple(self.config)[:7])
    self.bn_state = torch.zeros(0, device=device)

  def set_precision(self, precision):
    precision = precision or 'fp32'
    if precision not in _PRECISIONS:
      raise ValueError('precision must be one of %s' % sorted(_PRECISIONS))
    old = getattr(self, '_precision', None)
    self._precision = _PRECISIONS[precision]
    if _C.lib.tfr_bert_param_count(ctypes.byref(self._make_cfg(0.0))) == 0:
      self._precision = old
      raise ValueError(_C.last_error())
    self.precision = precision

  def _make_cfg(self, output_dropout, training=False, seed=0):
    c = self.config
    cfg = _C.BertCfg()
    cfg.vocab_size = c.vocab_size
    cfg.hidden_size = c.hidden_size
    cfg.num_heads = c.num_attention_heads
    cfg.intermediate_size = c.intermediate_size
    cfg.num_layers = c.num_layers
    cfg.max_position = c.max_position_embeddings
    cfg.type_vocab_size = c.type_vocab_size
    cfg.hidden_dropout = c.hidden_dropout_prob
    cfg.attention_dropout = c.attention_dropout_prob
    cfg.output_dropout = float(output_dropout)
    cfg.training = int(bool(training))
    cfg.seed = seed
    cfg.precision = self._precision
    return cfg

  def _run_cfg(self, training):
    """cfg of one call; training calls draw fresh dropout (seed = base << 32 | call)."""
    if training:
      self._calls += 1
    return self._make_cfg(self.output_dropout, training,
                          (self._base << 32) | (self._calls & 0xFFFFFFFF))

  def weight_names(self):
    return [n for n, _ in weight_shapes(self.config)]

  def get_weights(self):
    """CPU tensors in the documented order (`weight_names`)."""
    out, off = [], 0
    flat = self.flat.detach().cpu()
    for _, shape in weight_shapes(self.config):
      n = 1
      for s in shape:
        n *= s
      out.append(flat[off:off + n].reshape(shape).clone())
      off += n
    return out

  def set_weights(self, weights):
    shapes = weight_shapes(self.config)
    if len(weights) != len(shapes):
      raise ValueError('expected %d weights, got %d' % (len(shapes), len(weights)))
    parts = []
    for (name, shape), w in zip(shapes, weights):
      w = torch.as_tensor(w, dtype=torch.float32)
      if tuple(w.shape) != tuple(shape):
        raise ValueError('%s: expected shape %s, got %s' % (name, shape, tuple(w.shape)))
      parts.append(w.reshape(-1))
    with torch.no_grad():
      self.flat.copy_(torch.cat(parts).to(self.flat.device))

  def load_checkpoint(self, path):
    """Overwrites every encoder weight with a pretrained checkpoint's (a TF2 BertEncoder
    checkpoint prefix, a Hugging Face `model.safetensors` / `pytorch_model.bin`, or a
    directory holding one); the score head keeps its values, as the reference restores only
    the `encoder` object.  ValueError for a checkpoint that disagrees with the config."""
    loaded = bert_checkpoint.read_bert_weights(path, self.config)
    head = self.get_weights()[-2:]
    self.set_weights(list(loaded.values()) + head)

  @classmethod
  def from_pretrained(cls, path, config=None, seed=None, device='cuda', precision=None):
    """An encoder initialised from a pretrained checkpoint (see `load_checkpoint`).  The
    config is `config`, else the `config.json` or `bert_config.json` beside the checkpoint.
    The parameters are fp32 in every `precision`."""
    if config is None:
      config_file = config_beside(path)
      if config_file is None:
        raise ValueError('%s: no config.json or bert_config.json beside the checkpoint; '
                         'pass config=' % path)
      config = BertEncoderConfig.from_json(config_file)
    enc = cls(config, seed=seed, device=device, precision=precision)
    enc.load_checkpoint(path)
    return enc


class TFRBertScorer(object):
  """TFRBertScorer (tfrbert_task.py): Dropout(bert_output_dropout) on the encoder's pooled
  output, then Dense(1).  Shares the encoder's flat buffer, whose last E + 1 floats are the
  Dense(1) kernel and bias."""

  def __init__(self, encoder, bert_output_dropout=0.1):
    if not 0.0 <= bert_output_dropout < 1.0:
      raise ValueError('bert_output_dropout must be in [0, 1)')
    self.encoder = encoder
    encoder.output_dropout = float(bert_output_dropout)
    self.flat = encoder.flat
    self.decay_mask = encoder.decay_mask
    self.dims = encoder.dims
    self.bn_state = encoder.bn_state


class TFRBertRankingTrainer(train_lib.RankingTrainer):
  """Fused step of the reference's TFR-BERT recipe:

      scores [B, N] = scorer(ids, mask, type ids [B, N, L])   tfr_bert_fwd
      loss, d loss / d scores                                  fused loss kernel
      d loss / d params                                        tfr_bert_bwd
      params update                                            tfr_adamw_step (default) or the
                                                               base class's sgd / adagrad

  AdamW defaults are BERT's: weight_decay_rate 0.01 on every kernel and table (LayerNorm and
  biases excluded), beta_1 0.9, beta_2 0.999, epsilon 1e-6; `learning_rate` may be a float or
  a schedule such as `train.PolynomialWarmUp`; `gradient_clip_norm` (the base class's, off by
  default; the recipe's AdamWeightDecay uses 1.0) clips to a global norm first.  Padded items
  (label < 0) are encoded too, as in the reference; the loss ignores them.  fit / evaluate /
  checkpoints are the base class's; batches are ({'input_word_ids', 'input_mask',
  'input_type_ids'}, y) pairs.

  fp16 steps (an encoder in precision 'fp16') scale the loss, as Keras' LossScaleOptimizer
  does for 'mixed_float16' (the rule is include/tfr_b200.h's, next to AdamW's):
  `loss_scale` 'dynamic' (default) starts at `initial_loss_scale` (2^15), halves on a step
  whose scaled gradient holds an inf or NaN (that step is skipped: parameters and moments
  untouched, `adam_step` still advances) and doubles after `dynamic_growth_steps` (2000)
  finite steps in a row; a float is a fixed scale.  The step scales d loss / d scores by S on
  the device (trainer.dscores holds the scaled values), takes the global norm of the scaled
  gradient, and runs tfr_adamw_step_scaled and tfr_loss_scale_update: no host sync.
  `loss_scale` (0-d float32) and `good_steps` (0-d int64, the finite steps since the last
  change) are device tensors; `grad_norm` holds the last fp16 step's unscaled gradient norm,
  before clipping.  fp16 needs optimizer 'adamw' and one rank (ValueError otherwise).  fp32,
  tf32 and bf16 steps do not scale; `predict` never does."""

  def __init__(self, scorer, loss, optimizer='adamw', learning_rate=3e-5, epsilon=1e-6,
               weight_decay_rate=0.01, loss_scale='dynamic', initial_loss_scale=2 ** 15,
               dynamic_growth_steps=2000, **kw):
    self.scorer = scorer
    self.encoder = scorer.encoder
    if loss_scale == 'dynamic':
      init, growth = float(initial_loss_scale), int(dynamic_growth_steps)
      if not (1.0 <= init < float('inf')):
        raise ValueError('initial_loss_scale must be finite and >= 1, got %r' %
                         (initial_loss_scale,))
      if growth < 1:
        raise ValueError('dynamic_growth_steps must be >= 1, got %r' % (dynamic_growth_steps,))
    else:
      try:
        init, growth = float(loss_scale), 0
      except (TypeError, ValueError):
        raise ValueError("loss_scale must be 'dynamic' or a number, got %r" % (loss_scale,))
      if not (0.0 < init < float('inf')):
        raise ValueError('a fixed loss_scale must be finite and > 0, got %r' % (loss_scale,))
    super().__init__(scorer, loss, optimizer=optimizer, learning_rate=learning_rate,
                     epsilon=epsilon, weight_decay_rate=weight_decay_rate, **kw)
    self.bad_ids = torch.zeros(1, dtype=torch.int32, device=self.device)
    self.initial_loss_scale = init
    self.dynamic_growth_steps = growth   # 0: a fixed scale
    self.loss_scale = torch.full((), init, dtype=torch.float32, device=self.device)
    self.good_steps = torch.zeros((), dtype=torch.int64, device=self.device)
    if self.encoder.precision == 'fp16':
      self._check_fp16()

  def _check_fp16(self):
    """fp16's loss-scaled update is AdamW on one rank; its norm buffers on first use."""
    if self.opt_kind != train_lib._OPT['adamw']:
      raise ValueError("precision 'fp16' needs optimizer 'adamw' (loss scaling is built for "
                       "AdamW only)")
    if self.world > 1:
      raise ValueError('precision fp16 supports one rank only, got world size %d' % self.world)
    if getattr(self, '_scaled_norm', None) is None:
      dev, n = self.device, self.scorer.flat.numel()
      self._scaled_norm = torch.zeros((), dtype=torch.float32, device=dev)
      if getattr(self, 'grad_norm', None) is None:
        self.grad_norm = torch.zeros((), dtype=torch.float32, device=dev)
      if getattr(self, '_norm_ws', None) is None:
        self._norm_ws = torch.empty(_C.lib.tfr_global_norm_workspace_bytes(n),
                                    dtype=torch.uint8, device=dev)

  def reset_loss_scale(self):
    """The loss scale back to its initial value, the good-step count to 0."""
    self.loss_scale.fill_(self.initial_loss_scale)
    self.good_steps.zero_()

  def _apply(self, grads):
    if self.encoder.precision != 'fp16':
      super()._apply(grads)
      return
    # grads are the gradient of S * loss: norm, then the update and the scale's rule
    t = self.tower
    lr = self.lr(self.adam_step) if callable(self.lr) else self.lr
    self.adam_step += 1
    n = grads.numel()
    st = _C.stream()
    _C.check(_C.lib.tfr_global_norm(_C.ptr(grads), n, _C.ptr(self._scaled_norm),
                                     _C.ptr(self._norm_ws), self._norm_ws.numel(), st))
    _C.check(_C.lib.tfr_adamw_step_scaled(
        _C.ptr(t.flat.data), _C.ptr(grads), _C.ptr(self.accum[:n]), _C.ptr(self.accum[n:]),
        _C.ptr(self.decay_mask), n, lr, self.beta_1, self.beta_2, self.eps,
        self.weight_decay_rate, self.adam_step, self.gradient_clip_norm or 0.0,
        _C.ptr(self._scaled_norm), _C.ptr(self.loss_scale), st))
    _C.check(_C.lib.tfr_loss_scale_update(_C.ptr(self.loss_scale), _C.ptr(self.good_steps),
                                          _C.ptr(self._scaled_norm), _C.ptr(self.grad_norm),
                                          self.dynamic_growth_steps, st))

  def _ensure_bert(self, b, n, seq):
    if self._shape == (b, n, seq):
      return
    dev = self.device
    self.scores = torch.empty(b, n, dtype=torch.float32, device=dev)
    self.dscores = torch.empty(b, n, dtype=torch.float32, device=dev)
    self.per_list = torch.empty(2, b, dtype=torch.float32, device=dev)
    self.total2 = torch.zeros(2, dtype=torch.float32, device=dev)
    cfg = self.encoder._make_cfg(self.encoder.output_dropout)
    nbytes = _C.lib.tfr_bert_workspace_bytes(ctypes.byref(cfg), b * n, seq)
    if nbytes == 0:
      raise ValueError(_C.last_error())
    self.ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    self._shape = (b, n, seq)

  def _inputs(self, input_word_ids, input_mask, input_type_ids):
    if input_word_ids.dim() != 3:
      raise ValueError('input_word_ids must be [B, N, L], got %s' %
                       (tuple(input_word_ids.shape),))
    shape = tuple(input_word_ids.shape)
    for name, t in (('input_mask', input_mask), ('input_type_ids', input_type_ids)):
      if tuple(t.shape) != shape:
        raise ValueError('%s has shape %s, input_word_ids %s' % (name, tuple(t.shape), shape))
    dev = self.device
    wid = input_word_ids.to(dev, torch.int32, non_blocking=True).contiguous()
    msk = input_mask.to(dev, non_blocking=True)
    msk = (msk != 0).to(torch.uint8) if msk.dtype != torch.uint8 else msk.contiguous()
    tid = input_type_ids.to(dev, torch.int32, non_blocking=True).contiguous()
    b, n, seq = shape
    self._ensure_bert(b, n, seq)
    return wid, msk, tid, b * n, seq

  def check_ids(self):
    """Raises ValueError if a step has seen ids outside the tables (host sync)."""
    n = int(self.bad_ids.item())
    if n:
      raise ValueError('%d word / type ids lay outside their tables and were skipped' % n)

  def train_step(self, input_word_ids, input_mask, input_type_ids, y_true, sample_weight=None,
                 mask=None):
    """ids / mask / type ids [B, N, L] (device or host), y_true [B, N] (label < 0 = padded
    item).  Returns the scalar loss as a 0-d device tensor (no host sync)."""
    fp16 = self.encoder.precision == 'fp16'
    if fp16:
      self._check_fp16()
    wid, msk, tid, s, seq = self._inputs(input_word_ids, input_mask, input_type_ids)
    if mask is not None:
      y_true = torch.where(mask.to(y_true.device), y_true, torch.full_like(y_true, -1.0))
    cfg = ctypes.byref(self.encoder._run_cfg(True))
    flat = self.scorer.flat.data
    grads = self.grads
    st = _C.stream()
    _C.check(_C.lib.tfr_bert_fwd(_C.ptr(wid), _C.ptr(msk), _C.ptr(tid), s, seq, cfg,
                                 _C.ptr(flat), _C.ptr(self.ws), _C.ptr(self.scores),
                                 _C.ptr(self.bad_ids), st))
    self.loss.fused_fwd_bwd(y_true, self.scores, sample_weight, self.dscores, self.per_list,
                            self.total2)
    if fp16:   # d loss / d scores times S, in place
      _C.check(_C.lib.tfr_loss_scale_mul(_C.ptr(self.dscores), self.dscores.numel(),
                                         _C.ptr(self.loss_scale), _C.ptr(self.dscores), st))
    _C.check(_C.lib.tfr_bert_bwd(_C.ptr(wid), _C.ptr(msk), _C.ptr(tid), s, seq, cfg,
                                 _C.ptr(flat), _C.ptr(self.dscores), _C.ptr(self.ws),
                                 _C.ptr(grads), st))
    self._apply(grads)
    return self.total2[0]

  @torch.no_grad()
  def predict(self, input_word_ids, input_mask, input_type_ids, mask=None, y_true=None):
    """Scores [B, N] in inference mode (no dropout)."""
    wid, msk, tid, s, seq = self._inputs(input_word_ids, input_mask, input_type_ids)
    cfg = ctypes.byref(self.encoder._run_cfg(False))
    _C.check(_C.lib.tfr_bert_fwd(_C.ptr(wid), _C.ptr(msk), _C.ptr(tid), s, seq, cfg,
                                 _C.ptr(self.scorer.flat.data), _C.ptr(self.ws),
                                 _C.ptr(self.scores), _C.ptr(self.bad_ids), _C.stream()))
    return self.scores


@dataclasses.dataclass
class TFRBertDataConfig:
  """TFRBertDataConfig (tfrbert_task.py): the reference's recipe reads lists of 10 sequences
  of 64 tokens."""
  input_path: str = ''
  global_batch_size: int = 4
  list_size: int = 10
  seq_length: int = 128
  is_training: bool = True
  drop_remainder: bool = True
  label_feature: str = 'label'


_MAX_EXACT_ID = 1 << 24   # ids travel through the decoder's fp32 columns


def tfrbert_batches(paths, batch_size, list_size, seq_length, vocab_size=None,
                    type_vocab_size=None, label_feature='label', drop_remainder=True):
  """Yields ({'input_word_ids': int32, 'input_mask': uint8, 'input_type_ids': int32}
  [B, list_size, seq_length], y [B, list_size]) from TFRecord files of ELWC protos, as
  TFRBertDataLoader decodes them: example features `input_ids`, `input_mask`, `segment_ids`
  (int64, dim seq_length, default zeros) and the label (default -1).  Padded items and
  missing features take the defaults: a padded item is an all-masked sequence of id 0.  Ids
  must lie in [0, vocab_size) (and type ids in [0, type_vocab_size)) when those are given,
  and below 2^24 always (the decoder carries them exactly in fp32); ValueError otherwise."""
  seq = int(seq_length)
  spec = {'input_ids': (seq, 0.0), 'input_mask': (seq, 0.0), 'segment_ids': (seq, 0.0),
          label_feature: (1, -1.0)}
  limits = {'input_ids': vocab_size, 'segment_ids': type_vocab_size}
  buf = []

  def flush():
    out = data_lib.parse_from_example_list(buf, list_size, None, spec)
    ex = out['examples']
    feats = {}
    for i, (name, key) in enumerate((('input_ids', 'input_word_ids'),
                                     ('input_mask', 'input_mask'),
                                     ('segment_ids', 'input_type_ids'))):
      col = ex[:, :, i * seq:(i + 1) * seq]
      if name == 'input_mask':
        feats[key] = (col != 0).to(torch.uint8)
        continue
      lim = limits[name]
      top = min(lim, _MAX_EXACT_ID) if lim is not None else _MAX_EXACT_ID
      if bool(((col < 0) | (col >= top) | (col != col.round())).any()):
        raise ValueError('%s holds ids outside [0, %d)' % (name, top))
      feats[key] = col.to(torch.int32)
    y = ex[:, :, 3 * seq].clone()
    y = torch.where(out['mask'], y, torch.full_like(y, -1.0))
    return feats, y

  for path in ([paths] if isinstance(paths, str) else paths):
    for rec in data_lib.read_tfrecords(path):
      buf.append(rec)
      if len(buf) == batch_size:
        yield flush()
        buf = []
  if buf and not drop_remainder:
    yield flush()
