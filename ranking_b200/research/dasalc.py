"""DASALC ("Are Neural Rankers still Outperformed by Gradient Boosted Decision Trees?",
ICLR 2021; research/dasalc.py of the reference): the scorer and its feature transform.

`DASALCScorer` runs in the K13 kernels (csrc/dasalc.cu, tfr_dasalc_fwd / tfr_dasalc_bwd):

    a0 = BN_in(x) + GaussianNoise            x: log1p_cutoff-transformed features [.., D]
    a_l = Dropout(BN_l(relu(Dense_W(a_l-1))))  two hidden layers of width W
    t = Dense_W(a_2),  c = Dense_W(BN_c(e))   e: the DocumentInteractionAttention output [.., h]
    s = Dense_T(Dropout(relu(t * c + t)))     the latent cross, T = output_units tasks

All parameters live in ONE flat fp32 buffer (`flat`) in the layout of include/tfr_b200.h
(W_1, b_1, W_2, b_2, W_t, b_t, W_c, b_c, w_o, b_o, then gamma / beta of BN_in, BN_1, BN_2, BN_c);
the moving statistics live in `bn_state`.  `train()` / `eval()` select the mode.
"""
import ctypes
import math

import torch

from ranking_b200 import _C

_PRECISIONS = {'tf32x3': _C.PREC_TF32X3, 'tf32': _C.PREC_TF32}


def log1p_cutoff(x, cutoff=30.0):
  """clip(sign(x) log1p(|x|), -cutoff, cutoff) (research/dasalc.py:127-129), elementwise on
  the device (tfr_symmetric_log1p_clip)."""
  _C.require_cuda(x, 'log1p_cutoff input')
  x = x.float().contiguous()
  out = torch.empty_like(x)
  _C.check(_C.lib.tfr_symmetric_log1p_clip(_C.ptr(x), x.numel(), float(cutoff), _C.ptr(out),
                                           _C.stream()))
  return out


class _DASALCFn(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x, e, flat, m8, scorer):
    m, t = x.shape[0], scorer.output_units
    scores = torch.empty(t, m, dtype=torch.float32, device=x.device)
    ws = scorer._new_workspace(m)
    cfg = scorer._run_cfg()
    _C.check(_C.lib.tfr_dasalc_fwd_tasks(_C.ptr(x), _C.ptr(e), e.shape[1], m, ctypes.byref(cfg),
                                         _C.ptr(flat), _C.ptr(m8), _C.ptr(ws), _C.ptr(scores), t,
                                         scorer._precision, _C.stream()))
    ctx.cfg, ctx.ws, ctx.scorer = cfg, ws, scorer
    ctx.save_for_backward(x, flat, m8)
    return scores

  @staticmethod
  def backward(ctx, g):
    x, flat, m8 = ctx.saved_tensors
    m = x.shape[0]
    h = ctx.scorer.context_dim
    grads = torch.empty_like(flat)
    de = torch.empty(m, h, dtype=torch.float32, device=x.device)
    g = g.float().contiguous()
    _C.check(_C.lib.tfr_dasalc_bwd_tasks(_C.ptr(x), m, ctypes.byref(ctx.cfg), _C.ptr(flat),
                                         _C.ptr(g), None, _C.ptr(m8), _C.ptr(ctx.ws),
                                         _C.ptr(grads), _C.ptr(de), h, ctx.scorer.output_units,
                                         ctx.scorer._precision, _C.stream()))
    return None, de, grads, None, None


def _glorot(gen, fan_in, fan_out):
  limit = math.sqrt(6.0 / (fan_in + fan_out))
  return (torch.rand(fan_in, fan_out, generator=gen, dtype=torch.float64) * 2 * limit -
          limit).float()


class DASALCScorer(torch.nn.Module):
  """DASALC's scoring function (research/dasalc.py:167-201) over features already passed
  through `log1p_cutoff` and the DIN embedding of every item.

  Called as `scorer((x, e), mask)` with x [B, N, D] (or [M, D]) and e [B, N, h] (or [M, h]);
  returns scores of the same leading shape, ln(1e-10) where `mask` is False.  With
  `output_units` T > 1 (one unit per ranking task, MultiTaskDASALCRankingTrainer) the output
  layer is [W, T] and the result is [T, *leading shape], one score plane per task.  Gradients flow
  to `flat` and to `e` (not to x).  Keras initialisers: glorot-uniform kernels, zero biases,
  BN gamma ones / beta zeros, moving mean zeros / variance ones; BN epsilon 1e-3 as
  tf.compat.v1.layers.batch_normalization.  Limits: D, hidden_dim, context_dim multiples of 4,
  hidden_dim <= 4096, context_dim <= 128."""

  KERNELS = ('hidden1', 'hidden2', 'tower', 'context', 'output')
  NORMS = ('input', 'hidden1', 'hidden2', 'context')

  def __init__(self, input_dim, hidden_dim=512, context_dim=100, dropout=0.4,
               input_noise_stddev=1.5, batch_norm_moment=0.9, precision='tf32x3', seed=None,
               device='cuda', output_units=1):
    super().__init__()
    if precision not in _PRECISIONS:
      raise ValueError('precision must be one of %s' % sorted(_PRECISIONS))
    self.input_dim = int(input_dim)
    self.hidden_dim = int(hidden_dim)
    self.context_dim = int(context_dim)
    self.output_units = int(output_units)
    self.dropout = float(dropout or 0.0)
    self.input_noise_stddev = float(input_noise_stddev or 0.0)
    self.batch_norm_moment = float(batch_norm_moment)
    self.bn_epsilon = 1e-3
    self.precision = precision
    self._precision = _PRECISIONS[precision]
    cfg = _C.DasalcCfg()
    cfg.input_dim, cfg.hidden_dim, cfg.context_dim = self.input_dim, self.hidden_dim, \
        self.context_dim
    cfg.dropout = self.dropout
    cfg.input_noise_stddev = self.input_noise_stddev
    cfg.bn_epsilon = self.bn_epsilon
    cfg.bn_momentum = self.batch_norm_moment
    cfg.training = 1
    n = _C.lib.tfr_dasalc_param_count_tasks(ctypes.byref(cfg), self.output_units)
    if n == 0:
      raise ValueError(_C.last_error())
    ns = _C.lib.tfr_dasalc_bn_state_count(ctypes.byref(cfg))
    self._cfg = cfg
    d, w, h = self.input_dim, self.hidden_dim, self.context_dim
    # (name, rows, cols) of the kernels; every kernel is followed by its bias [cols]
    shapes = [('hidden1', d, w), ('hidden2', w, w), ('tower', w, w), ('context', h, w),
              ('output', w, self.output_units)]
    gen = torch.Generator()
    if seed is not None:
      gen.manual_seed(int(seed))
    parts, off = [], 0
    self._kernel_offsets = {}
    for name, r, c in shapes:
      parts += [_glorot(gen, r, c).reshape(-1), torch.zeros(c)]
      self._kernel_offsets[name] = (off, r, c)
      off += r * c + c
    self._bn_offsets = {}
    state, soff = [], 0
    for name, width in zip(self.NORMS, (d, w, w, h)):
      parts += [torch.ones(width), torch.zeros(width)]
      state += [torch.zeros(width), torch.ones(width)]
      self._bn_offsets[name] = (off, soff, width)
      off += 2 * width
      soff += 2 * width
    flat = torch.cat(parts)
    assert flat.numel() == n and soff == ns, (flat.numel(), n, soff, ns)
    self.dims = ['dasalc', d, w, h]
    if self.output_units > 1:
      self.dims.append(self.output_units)
    self.flat = torch.nn.Parameter(flat.to(device))
    self.register_buffer('bn_state', torch.cat(state).to(device))
    self._base = int(seed if seed is not None else torch.seed()) & 0xFFFFFFFF
    self._calls = 0

  # -- accessors (views of `flat` / `bn_state`) ---------------------------------
  def kernel(self, name):
    off, r, c = self._kernel_offsets[name]
    return self.flat[off:off + r * c].view(r, c)

  def bias(self, name):
    off, r, c = self._kernel_offsets[name]
    return self.flat[off + r * c:off + r * c + c]

  def batch_norm(self, name):
    """(gamma, beta) of BN layer `name` in NORMS."""
    off, _, w = self._bn_offsets[name]
    return self.flat[off:off + w], self.flat[off + w:off + 2 * w]

  def moving_stats(self, name):
    """(moving_mean, moving_variance) of BN layer `name` in NORMS."""
    _, soff, w = self._bn_offsets[name]
    return self.bn_state[soff:soff + w], self.bn_state[soff + w:soff + 2 * w]

  # -- kernel plumbing ------------------------------------------------------------
  def _run_cfg(self, training=None):
    cfg = _C.DasalcCfg()
    ctypes.memmove(ctypes.byref(cfg), ctypes.byref(self._cfg), ctypes.sizeof(cfg))
    training = self.training if training is None else training
    cfg.training = int(bool(training))
    if training and (self.dropout > 0 or self.input_noise_stddev > 0):
      self._calls += 1
    cfg.seed = (self._base << 32) | (self._calls & 0xFFFFFFFF)
    cfg.bn_state = self.bn_state.data_ptr()
    return cfg

  def _new_workspace(self, m):
    nbytes = _C.lib.tfr_dasalc_workspace_bytes_tasks(ctypes.byref(self._cfg), int(m),
                                                     self.output_units)
    if nbytes == 0:
      raise ValueError(_C.last_error())
    return torch.empty(nbytes, dtype=torch.uint8, device=self.flat.device)

  def forward(self, inputs, mask=None):
    x, e = inputs
    _C.require_cuda(x, 'DASALCScorer features')
    _C.require_cuda(e, 'DASALCScorer context embedding')
    if x.requires_grad:
      raise NotImplementedError('gradients w.r.t. the DASALC features are not computed')
    lead = x.shape[:-1]
    if x.shape[-1] != self.input_dim or e.shape[-1] != self.context_dim or \
        e.shape[:-1] != lead:
      raise ValueError('expected features [..., %d] and embedding [..., %d] with the same '
                       'leading shape, got %s and %s' % (self.input_dim, self.context_dim,
                                                         tuple(x.shape), tuple(e.shape)))
    x = x.float().reshape(-1, self.input_dim).contiguous()
    e = e.float().reshape(-1, self.context_dim).contiguous()
    m8 = None
    if mask is not None:
      m8 = torch.as_tensor(mask, device=x.device).reshape(-1).to(torch.uint8).contiguous()
    scores = _DASALCFn.apply(x, e, self.flat, m8, self)
    if self.output_units == 1:
      return scores.reshape(lead)
    return scores.reshape((self.output_units,) + tuple(lead))

  def get_config(self):
    return {'input_dim': self.input_dim, 'hidden_dim': self.hidden_dim,
            'context_dim': self.context_dim, 'dropout': self.dropout,
            'input_noise_stddev': self.input_noise_stddev,
            'batch_norm_moment': self.batch_norm_moment, 'precision': self.precision,
            'output_units': self.output_units}
