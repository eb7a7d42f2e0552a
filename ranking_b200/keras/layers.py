"""`tfr.keras.layers` pieces on the hot path: create_tower, FlattenList, RestoreList
(keras/layers.py:26-77, 80-182, 185-272).

`create_tower` returns a `Tower`: a torch.nn.Module whose forward/backward run in
the CUDA scorer kernels (tfr_mlp_fwd / tfr_mlp_bwd).  All Dense kernels and
biases live in ONE flat fp32 parameter (`Tower.flat`), Keras layout
(kernel [in, out]), so data-parallel training needs a single all-reduce.
"""
import ctypes
import math

import torch

from ranking_b200 import _C
from ranking_b200 import utils as tfr_utils

_LOG_EPSILON = math.log(1e-10)

_PRECISIONS = {'fp32': _C.PREC_FP32, 'tf32x3': _C.PREC_TF32X3,
               'tf32': _C.PREC_TF32, 'bf16': _C.PREC_BF16}
# DocumentInteractionAttention builds no 3xTF32 or bf16 attention core
_DIN_PRECISIONS = {'fp32': _C.PREC_FP32, 'tf32': _C.PREC_TF32}


def _activation_enum(activation):
  if activation is None or activation == 'linear':
    return _C.ACT_NONE
  if activation == 'relu' or activation is torch.relu or \
      activation is torch.nn.functional.relu:
    return _C.ACT_RELU
  raise NotImplementedError(
      'activation %r: the CUDA tower supports None and relu' % (activation,))


class _TowerFn(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x, flat, mask, tower):
    m = x.shape[0]
    out = torch.empty(m, tower.output_units, dtype=torch.float32,
                      device=x.device)
    # The workspace carries the activations to backward; one per forward call
    # so that several forwards may be outstanding (caching allocator: cheap).
    ws = tower._new_workspace(m)
    cfg = tower._run_cfg()
    _C.check(_C.lib.tfr_mlp_fwd(_C.ptr(x), m, ctypes.byref(cfg),
                                _C.ptr(flat), _C.ptr(mask), _C.ptr(ws),
                                _C.ptr(out), tower._precision, _C.stream()))
    ctx.tower = tower
    ctx.cfg = cfg      # backward sees the mode (training / inference) of ITS forward
    ctx.ws = ws
    ctx.save_for_backward(x, flat, mask)
    return out

  @staticmethod
  def backward(ctx, g_out):
    x, flat, mask = ctx.saved_tensors
    tower = ctx.tower
    m = x.shape[0]
    grads = torch.empty_like(flat)
    ws = ctx.ws
    _C.check(_C.lib.tfr_mlp_bwd(_C.ptr(x), m, ctypes.byref(ctx.cfg),
                                _C.ptr(flat), _C.ptr(g_out.contiguous()),
                                _C.ptr(mask), _C.ptr(ws), _C.ptr(grads),
                                tower._precision, _C.stream()))
    dx = None
    if ctx.needs_input_grad[0]:
      dx = torch.empty(m, tower.input_dim, dtype=torch.float32, device=x.device)
      _C.check(_C.lib.tfr_mlp_input_grad(ctypes.byref(ctx.cfg), m, _C.ptr(flat), _C.ptr(ws), 0,
                                         tower.input_dim, _C.ptr(dx), tower.input_dim,
                                         tower._precision, _C.stream()))
    return dx, grads, None, None


class Tower(torch.nn.Module):
  """Feed-forward tower (keras/layers.py:65-77):
  [BN] -> (Dense -> [BN] -> activation -> [Dropout]) x L -> Dense(output_units).

  `module.train()` / `module.eval()` select batch statistics + dropout vs moving
  statistics, as Keras' `training` argument does."""

  def __init__(self, input_dim, hidden_layer_dims, output_units, activation=None,
               precision=None, seed=None, device='cuda', input_batch_norm=False,
               use_batch_norm=False, batch_norm_moment=0.999, dropout=0.0,
               batch_norm_epsilon=1e-3):
    super().__init__()
    self.input_dim = int(input_dim)
    self.hidden_layer_dims = [int(h) for h in hidden_layer_dims]
    self.output_units = int(output_units)
    self.activation = activation
    dims = [self.input_dim] + self.hidden_layer_dims + [self.output_units]
    if len(dims) - 1 > _C.MLP_MAX_LAYERS:
      raise ValueError('at most %d Dense layers are supported' % _C.MLP_MAX_LAYERS)
    cfg = _C.MlpCfg()
    cfg.n_dense = len(dims) - 1
    for i, d in enumerate(dims):
      cfg.dims[i] = d
    cfg.activation = _activation_enum(activation)
    if not 0.0 <= float(dropout) < 1.0:
      raise ValueError('dropout must be in [0, 1)')
    cfg.use_batch_norm = int(bool(use_batch_norm) and len(self.hidden_layer_dims) > 0)
    cfg.input_batch_norm = int(bool(input_batch_norm))
    cfg.bn_epsilon = float(batch_norm_epsilon)
    cfg.bn_momentum = float(batch_norm_moment)
    cfg.dropout = float(dropout) if self.hidden_layer_dims else 0.0
    cfg.training = 1
    cfg.dropout_seed = 0
    cfg.bn_state = None
    self.use_batch_norm = bool(cfg.use_batch_norm)
    self.input_batch_norm = bool(cfg.input_batch_norm)
    self.dropout = float(cfg.dropout)
    self._dropout_base = int(seed if seed is not None else
                             torch.seed()) & 0xFFFFFFFF
    self._dropout_calls = 0
    self._cfg = cfg
    self.dims = dims
    self.set_precision(precision)
    n = _C.lib.tfr_mlp_param_count(ctypes.byref(cfg))
    if n == 0:
      raise ValueError(_C.last_error())
    # Keras defaults: glorot_uniform kernels, zero biases.
    gen = torch.Generator()
    if seed is not None:
      gen.manual_seed(seed)
    flat = torch.zeros(n, dtype=torch.float32)
    self.offsets = []
    off = 0
    for i in range(cfg.n_dense):
      fi, fo = dims[i], dims[i + 1]
      limit = math.sqrt(6.0 / (fi + fo))
      w = (torch.rand(fi, fo, generator=gen, dtype=torch.float64) * 2 * limit -
           limit).float()
      flat[off:off + fi * fo] = w.reshape(-1)
      self.offsets.append((off, off + fi * fo, off + fi * fo + fo))
      off += fi * fo + fo
    # BatchNormalization parameters follow the Dense ones: gamma (ones), beta (zeros);
    # moving_mean (zeros) / moving_variance (ones) live in `bn_state`.
    self.bn_offsets = {}        # 'input' | hidden index -> (gamma_off, beta_off, width)
    self.bn_state_offsets = {}  # same keys -> (mean_off, var_off, width)
    soff = 0
    bn_layers = (['input'] if self.input_batch_norm else []) + (
        list(range(len(self.hidden_layer_dims))) if self.use_batch_norm else [])
    state = []
    for key in bn_layers:
      w_ = dims[0] if key == 'input' else dims[key + 1]
      flat[off:off + w_] = 1.0
      self.bn_offsets[key] = (off, off + w_, w_)
      off += 2 * w_
      self.bn_state_offsets[key] = (soff, soff + w_, w_)
      state += [torch.zeros(w_), torch.ones(w_)]
      soff += 2 * w_
    assert off == n and soff == _C.lib.tfr_mlp_bn_state_count(ctypes.byref(cfg))
    self.flat = torch.nn.Parameter(flat.to(device))
    self.register_buffer(
        'bn_state', torch.cat(state).to(device) if state else
        torch.zeros(0, device=device))

  def _run_cfg(self, training=None):
    """A per-call copy of the config: mode, dropout seed, BN state pointer."""
    cfg = _C.MlpCfg()
    ctypes.memmove(ctypes.byref(cfg), ctypes.byref(self._cfg), ctypes.sizeof(cfg))
    training = self.training if training is None else training
    cfg.training = int(bool(training))
    if training and self.dropout > 0:
      self._dropout_calls += 1
    cfg.dropout_seed = (self._dropout_base << 32) | (self._dropout_calls & 0xFFFFFFFF)
    cfg.bn_state = self.bn_state.data_ptr() if self.bn_state.numel() else None
    return cfg

  def bn_gamma(self, key):
    a, b, w_ = self.bn_offsets[key]
    return self.flat[a:a + w_]

  def bn_beta(self, key):
    a, b, w_ = self.bn_offsets[key]
    return self.flat[b:b + w_]

  def bn_moving(self, key):
    a, b, w_ = self.bn_state_offsets[key]
    return self.bn_state[a:a + w_], self.bn_state[b:b + w_]

  def set_precision(self, precision):
    if precision is None or precision == 'auto':
      # tensor cores whenever the layer widths allow it: the fp32-faithful 3xTF32 engine
      # needs every Dense input width to be a multiple of 4
      ok = all(d % 4 == 0 for d in self.dims[:-1])
      precision = 'tf32x3' if ok else 'fp32'
    if precision not in _PRECISIONS:
      raise ValueError('precision must be one of %s' % sorted(_PRECISIONS))
    self.precision = precision
    self._precision = _PRECISIONS[precision]
    # the bf16 mode reads its inputs (and keeps its activations) as bf16 in HBM
    self.input_dtype = torch.bfloat16 if precision == 'bf16' else torch.float32

  def kernel(self, i):
    a, b, _ = self.offsets[i]
    return self.flat[a:b].view(self.dims[i], self.dims[i + 1])

  def bias(self, i):
    _, b, c = self.offsets[i]
    return self.flat[b:c]

  def load_keras_weights(self, kernels, biases):
    """Loads per-layer Dense kernels [in, out] / biases (Keras `get_weights()`)."""
    with torch.no_grad():
      for i, (k, b) in enumerate(zip(kernels, biases)):
        self.kernel(i).copy_(torch.as_tensor(k, dtype=torch.float32))
        self.bias(i).copy_(torch.as_tensor(b, dtype=torch.float32))

  def _new_workspace(self, m):
    nbytes = _C.lib.tfr_mlp_workspace_bytes(ctypes.byref(self._cfg), m)
    return torch.empty(nbytes, dtype=torch.uint8, device=self.flat.device)

  def forward(self, inputs, mask=None):
    """inputs [..., input_dim] -> [..., output_units] (flattened internally).
    `mask` (flat bool [M]) applies RestoreList's ln(1e-10) fill in-kernel."""
    x = inputs
    _C.require_cuda(x, 'tower inputs')
    lead = x.shape[:-1]
    if x.shape[-1] != self.input_dim:
      raise ValueError('expected last dim %d, got %d' % (self.input_dim,
                                                        x.shape[-1]))
    # Input gradients (tfr_mlp_input_grad) need precision tf32x3 / tf32 and no input BN;
    # backward raises ValueError otherwise.
    x = x.reshape(-1, self.input_dim).to(self.input_dtype).contiguous()
    m8 = None if mask is None else mask.reshape(-1).to(torch.uint8).contiguous()
    out = _TowerFn.apply(x, self.flat, m8, self)
    return out.reshape(*lead, self.output_units)


def create_tower(hidden_layer_dims, output_units, activation=None,
                 input_batch_norm=False, use_batch_norm=True,
                 batch_norm_moment=0.999, dropout=0.5, name=None,
                 input_dim=None, precision=None, seed=None, **kwargs):
  """keras/layers.py:26-77.  Same arguments and defaults as the reference.

  `precision`: None (default) = 'tf32x3' (wgmma, fp32-faithful) when every Dense input
  width is a multiple of 4, else 'fp32' (FFMA); 'tf32', 'bf16' on request.

  BatchNormalization (batch statistics in `train()` mode, moving statistics in
  `eval()` mode) and Dropout run as HBM-bound passes next to the Dense GEMMs
  (csrc/mlp_norm.cu); the headline benchmark configuration uses neither.
  `input_dim` is required here because torch modules are built eagerly (Keras
  infers it at first call); `DNNScorer` supplies it automatically.
  """
  if input_dim is None:
    raise ValueError('create_tower needs input_dim')
  return Tower(input_dim, hidden_layer_dims, output_units, activation,
               precision=precision, seed=seed, input_batch_norm=input_batch_norm,
               use_batch_norm=use_batch_norm, batch_norm_moment=batch_norm_moment,
               dropout=dropout)


class FlattenList(torch.nn.Module):
  """keras/layers.py:80-182."""

  def __init__(self, circular_padding=True, name=None, **kwargs):
    super().__init__()
    self._circular_padding = circular_padding

  def forward(self, inputs):
    context_features, example_features, list_mask = inputs
    if not example_features:
      raise ValueError('Need a valid example feature.')
    list_mask = torch.as_tensor(list_mask)
    b, n = list_mask.shape
    flat_ctx = {}
    for name, t in context_features.items():
      flat_ctx[name] = t.unsqueeze(1).expand(b, n, *t.shape[1:]).reshape(
          b * n, *t.shape[1:])
    idx = None
    if self._circular_padding and not bool(list_mask.all()):
      idx, _ = tfr_utils.padded_nd_indices(list_mask)
    flat_ex = {}
    for name, t in example_features.items():
      if idx is not None:
        gi = idx.reshape(b, n, *([1] * (t.dim() - 2))).expand(-1, -1,
                                                              *t.shape[2:])
        t = torch.gather(t, 1, gi)
      flat_ex[name] = t.reshape(b * n, *t.shape[2:])
    return flat_ctx, flat_ex

  def get_config(self):
    return {'circular_padding': self._circular_padding}


class RestoreList(torch.nn.Module):
  """keras/layers.py:185-272."""

  def __init__(self, name=None, by_scatter=False, **kwargs):
    super().__init__()
    self._by_scatter = by_scatter

  def forward(self, inputs):
    flattened_logits, list_mask = inputs
    list_mask = torch.as_tensor(list_mask)
    try:
      logits = flattened_logits.reshape(list_mask.shape)
    except RuntimeError:
      raise ValueError('`flattened_logits` needs to be either 1D of [batch_size '
                       '* list_size] or 2D of [batch_size * list_size, 1].')
    fill = torch.full_like(logits, _LOG_EPSILON)
    if self._by_scatter:
      idx, _ = tfr_utils.padded_nd_indices(list_mask)
      counts = torch.zeros_like(logits).scatter_add_(1, idx,
                                                     torch.ones_like(logits))
      summed = torch.zeros_like(logits).scatter_add_(1, idx, logits)
      return torch.where(counts > 0., summed / counts.clamp(min=1.), fill)
    return torch.where(list_mask, logits, fill)

  def get_config(self):
    return {'by_scatter': self._by_scatter}


def _tower_sizes(dims, use_batch_norm):
  """(parameter count, bn_state count) of one tower in the tfr_mlp layout."""
  n = sum(dims[i] * dims[i + 1] + dims[i + 1] for i in range(len(dims) - 1))
  hidden = dims[1:-1]
  bn = 2 * sum(hidden) if use_batch_norm and hidden else 0
  return n + bn, bn


class _GAMFn(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x, flat, mask, gam, context):
    m = x.shape[0]
    f = gam.example_feature_num
    dev = x.device
    logits = torch.empty(m, dtype=torch.float32, device=dev)
    sub = torch.empty(m, f, dtype=torch.float32, device=dev)
    n_ctx = len(context) if context else 0
    subw = torch.empty(n_ctx, m, f, dtype=torch.float32, device=dev)
    ptrs = None
    if context:
      ptrs = (ctypes.c_void_p * n_ctx)(*[t.data_ptr() for t in context])
    ws = gam._new_workspace(m)
    cfg = gam._run_cfg()
    _C.check(_C.lib.tfr_gam_fwd(_C.ptr(x), ptrs, m, ctypes.byref(cfg), _C.ptr(flat),
                                _C.ptr(mask), _C.ptr(ws), _C.ptr(logits), _C.ptr(sub),
                                _C.ptr(subw) if n_ctx else None, _C.stream()))
    ctx.gam, ctx.cfg, ctx.ws, ctx.context, ctx.ptrs = gam, cfg, ws, context, ptrs
    ctx.save_for_backward(x, flat, mask)
    ctx.mark_non_differentiable(sub, subw)
    return logits, sub, subw

  @staticmethod
  def backward(ctx, g_logits, g_sub, g_subw):
    x, flat, mask = ctx.saved_tensors
    grads = torch.empty_like(flat)
    _C.check(_C.lib.tfr_gam_bwd(_C.ptr(x), ctx.ptrs, x.shape[0], ctypes.byref(ctx.cfg),
                                _C.ptr(flat), _C.ptr(g_logits.contiguous()), _C.ptr(mask),
                                _C.ptr(ctx.ws), _C.ptr(grads), _C.stream()))
    return None, grads, None, None, None


class GAMLayer(torch.nn.Module):
  """keras/layers.py:591-803: neural generalized additive model (Zhuang et al. 2021).

  Example feature f gets its own tower create_tower(example_hidden_layer_dims, 1); the
  logits are the sum of the towers' outputs, weighted per feature by the summed softmaxed
  outputs of the context towers create_tower(context_hidden_layer_dims, F) when context
  inputs are passed.  The towers run in the fused GAM kernels (csrc/gam.cu, tfr_gam_fwd /
  tfr_gam_bwd); all parameters live in ONE flat fp32 buffer (`flat`): example towers, then
  context towers, each in the create_tower layout (see `tower_slice`).

  Input dimensions come from the tensors, so the layer is built at its first call (or by
  `build`).  Returns `(logits [M, 1], sub_logits_list, sub_weights_list)`; gradients flow
  through `logits` only: the sub-outputs are returned for interpretation and are marked
  non-differentiable.  Inputs must not require grad.  `train()` / `eval()` select batch
  statistics + dropout or moving statistics.  Context towers need F <= 8."""

  def __init__(self, example_feature_num, example_hidden_layer_dims,
               context_feature_num=None, context_hidden_layer_dims=None, activation=None,
               use_batch_norm=True, batch_norm_moment=0.999, dropout=0.5, name=None,
               seed=None, device='cuda', batch_norm_epsilon=1e-3, **kwargs):
    super().__init__()
    self.example_feature_num = int(example_feature_num)
    self.example_hidden_layer_dims = [int(h) for h in example_hidden_layer_dims]
    self.context_feature_num = int(context_feature_num or 0)
    if self.context_feature_num > 0 and not context_hidden_layer_dims:
      raise ValueError(
          'When `context_feature_num` > 0, `context_hidden_layer_dims` is '
          'required! Currently `context_feature_num` is {}, but '
          '`context_hidden_layer_dims` is {}'.format(context_feature_num,
                                                    context_hidden_layer_dims))
    self.context_hidden_layer_dims = [int(h) for h in (context_hidden_layer_dims or [])]
    self.activation = activation
    self._act = _activation_enum(activation)
    if not 0.0 <= float(dropout or 0.0) < 1.0:
      raise ValueError('dropout must be in [0, 1)')
    self.dropout = float(dropout or 0.0)
    self._use_bn = bool(use_batch_norm)
    self.batch_norm_moment = float(batch_norm_moment)
    self.batch_norm_epsilon = float(batch_norm_epsilon)
    self._seed = seed
    self._device = device
    self._dropout_base = int(seed if seed is not None else torch.seed()) & 0xFFFFFFFF
    self._dropout_calls = 0
    self.input_batch_norm = False
    self.input_dtype = torch.float32
    self.use_batch_norm = self._use_bn and bool(self.example_hidden_layer_dims)
    self.register_parameter('flat', None)
    self.register_buffer('bn_state', None)
    self._cfg = None

  @property
  def built(self):
    return self._cfg is not None

  def build(self, example_dims, context_dims=None):
    """Creates the parameters for example feature widths `example_dims` and context
    feature widths `context_dims` (Keras initialisers: glorot_uniform kernels, zero
    biases, BN gamma ones / beta zeros, moving mean zeros / variance ones)."""
    example_dims = [int(d) for d in example_dims]
    context_dims = [int(d) for d in (context_dims or [])]
    if len(example_dims) != self.example_feature_num:
      raise ValueError('expected %d example features, got %d' %
                       (self.example_feature_num, len(example_dims)))
    if context_dims and len(context_dims) != self.context_feature_num:
      raise ValueError('expected %d context features, got %d' %
                       (self.context_feature_num, len(context_dims)))
    if not context_dims:
      # built by a call without context inputs: the context towers take width-1 inputs
      # unless `build` is called with their widths first
      context_dims = [1] * self.context_feature_num
    f = self.example_feature_num
    cfg = _C.GamCfg()
    if not 1 <= f <= _C.GAM_MAX_FEATURES:
      raise ValueError('example_feature_num must be in [1, %d]' % _C.GAM_MAX_FEATURES)
    if len(self.example_hidden_layer_dims) > _C.GAM_MAX_HIDDEN:
      raise ValueError('at most %d example hidden layers' % _C.GAM_MAX_HIDDEN)
    if self.context_feature_num > _C.GAM_MAX_CONTEXT:
      raise ValueError('at most %d context features' % _C.GAM_MAX_CONTEXT)
    if len(self.context_hidden_layer_dims) > _C.MLP_MAX_LAYERS - 1:
      raise ValueError('at most %d context hidden layers' % (_C.MLP_MAX_LAYERS - 1))
    cfg.n_features = f
    off = 0
    cfg.feature_offsets[0] = 0
    for i, d in enumerate(example_dims):
      off += d
      cfg.feature_offsets[i + 1] = off
    cfg.n_hidden = len(self.example_hidden_layer_dims)
    for i, h in enumerate(self.example_hidden_layer_dims):
      cfg.hidden[i] = h
    cfg.n_context = self.context_feature_num
    for j, d in enumerate(context_dims):
      cfg.context_dims[j] = d
    cfg.n_context_hidden = len(self.context_hidden_layer_dims)
    for i, h in enumerate(self.context_hidden_layer_dims):
      cfg.context_hidden[i] = h
    cfg.activation = self._act
    cfg.use_batch_norm = int(self._use_bn)
    cfg.bn_epsilon = self.batch_norm_epsilon
    cfg.bn_momentum = self.batch_norm_moment
    cfg.dropout = self.dropout
    cfg.training = 1
    n = _C.lib.tfr_gam_param_count(ctypes.byref(cfg))
    if n == 0:
      raise ValueError(_C.last_error())
    # per-tower slices: (kind, index) -> (param_off, n_params, state_off, n_state, dims)
    self.towers = []
    poff = soff = 0
    hid, chid = self.example_hidden_layer_dims, self.context_hidden_layer_dims
    for d in example_dims:
      dims = [d] + hid + [1]
      np_, ns = _tower_sizes(dims, self._use_bn)
      self.towers.append(('example', poff, np_, soff, ns, dims))
      poff += np_
      soff += ns
    for d in context_dims:
      dims = [d] + chid + [f]
      np_, ns = _tower_sizes(dims, self._use_bn)
      self.towers.append(('context', poff, np_, soff, ns, dims))
      poff += np_
      soff += ns
    assert poff == n and soff == _C.lib.tfr_gam_bn_state_count(ctypes.byref(cfg))
    gen = torch.Generator()
    if self._seed is not None:
      gen.manual_seed(self._seed)
    flat = torch.zeros(n, dtype=torch.float32)
    state = torch.zeros(soff, dtype=torch.float32)
    for _, po, np_, so, ns, dims in self.towers:
      o = po
      for i in range(len(dims) - 1):
        fi, fo = dims[i], dims[i + 1]
        limit = math.sqrt(6.0 / (fi + fo))
        w = torch.rand(fi, fo, generator=gen, dtype=torch.float64) * 2 * limit - limit
        flat[o:o + fi * fo] = w.float().reshape(-1)
        o += fi * fo + fo
      for h in dims[1:-1] if ns else []:
        flat[o:o + h] = 1.0
        o += 2 * h
      s = so
      for h in dims[1:-1] if ns else []:
        state[s + h:s + 2 * h] = 1.0
        s += 2 * h
    self._cfg = cfg
    self.example_dims = example_dims
    self.context_dims = context_dims
    self.dims = ['gam', example_dims, hid, context_dims, chid, self._act, int(self._use_bn)]
    self.flat = torch.nn.Parameter(flat.to(self._device))
    self.bn_state = state.to(self._device)
    return self

  def tower_slice(self, i):
    """(flat slice, bn_state slice, dims) of tower i: example towers 0..F-1, then context
    towers.  Each slice is in the create_tower / tfr_mlp layout: W_0, b_0, ..., W_L, b_L,
    then gamma / beta per BN layer; bn_state: moving mean / variance per BN layer."""
    _, po, np_, so, ns, dims = self.towers[i]
    return self.flat[po:po + np_], self.bn_state[so:so + ns], dims

  def load_keras_weights(self, i, kernels, biases):
    """Loads per-layer Dense kernels [in, out] / biases of tower i."""
    flat, _, dims = self.tower_slice(i)
    o = 0
    with torch.no_grad():
      for k, b in zip(kernels, biases):
        k = torch.as_tensor(k, dtype=torch.float32)
        flat[o:o + k.numel()].copy_(k.reshape(-1))
        o += k.numel()
        flat[o:o + k.shape[1]].copy_(torch.as_tensor(b, dtype=torch.float32))
        o += k.shape[1]

  def _run_cfg(self, training=None):
    cfg = _C.GamCfg()
    ctypes.memmove(ctypes.byref(cfg), ctypes.byref(self._cfg), ctypes.sizeof(cfg))
    training = self.training if training is None else training
    cfg.training = int(bool(training))
    if training and self.dropout > 0:
      self._dropout_calls += 1
    cfg.dropout_seed = (self._dropout_base << 32) | (self._dropout_calls & 0xFFFFFFFF)
    cfg.bn_state = self.bn_state.data_ptr() if self.bn_state.numel() else None
    return cfg

  def _new_workspace(self, m):
    nbytes = _C.lib.tfr_gam_workspace_bytes(ctypes.byref(self._cfg), m)
    if nbytes == 0:
      raise ValueError(_C.last_error())
    return torch.empty(nbytes, dtype=torch.uint8, device=self.flat.device)

  def forward(self, inputs, mask=None):
    """inputs = (example_inputs, context_inputs): lists of [M, ...] tensors (context may
    be None).  `mask` (flat bool [M], optional) applies RestoreList's ln(1e-10) fill to the
    logits in-kernel."""
    example_inputs, context_inputs = inputs
    if len(example_inputs) != self.example_feature_num:
      raise ValueError('Mismatched number of features in `example_inputs` ({}) '
                       'with `example_feature_num` ({})'.format(
                           len(example_inputs), self.example_feature_num))
    if context_inputs:
      if not self.context_feature_num or len(context_inputs) != self.context_feature_num:
        raise ValueError('Mismatched number of features in `context_inputs` '
                         '({}) with `_context_feature_num` ({})'.format(
                             len(context_inputs), self.context_feature_num))
    m = example_inputs[0].shape[0]
    ex = [t.reshape(m, -1) for t in example_inputs]
    cx = [t.reshape(m, -1) for t in context_inputs] if context_inputs else []
    for t in ex + cx:
      _C.require_cuda(t, 'GAM inputs')
      if t.requires_grad:
        raise NotImplementedError('gradients w.r.t. GAM inputs are not computed')
    if not self.built:
      self.build([t.shape[1] for t in ex], [t.shape[1] for t in cx] or None)
    elif cx and self.context_dims != [t.shape[1] for t in cx]:
      raise ValueError('context widths %s, the layer was built for %s' %
                       ([t.shape[1] for t in cx], self.context_dims))
    if [t.shape[1] for t in ex] != self.example_dims:
      raise ValueError('example widths %s, the layer was built for %s' %
                       ([t.shape[1] for t in ex], self.example_dims))
    x = torch.cat(ex, 1).float().contiguous() if len(ex) > 1 else ex[0].float().contiguous()
    cx = [t.float().contiguous() for t in cx]
    m8 = None if mask is None else mask.reshape(-1).to(torch.uint8).contiguous()
    logits, sub, subw = _GAMFn.apply(x, self.flat, m8, self, cx or None)
    sub_logits = [sub[:, f:f + 1] for f in range(self.example_feature_num)]
    sub_weights = [subw[j] for j in range(len(cx))]
    return logits.reshape(m, 1), sub_logits, sub_weights


class ConcatFeatures(torch.nn.Module):
  """keras/layers.py:276-375: context features repeated list_size times, then the example
  features (FlattenList, circular padding by default), concatenated in sorted name order:
  [batch_size, list_size, sum of feature dims]."""

  def __init__(self, circular_padding=True, name=None, **kwargs):
    super().__init__()
    self._circular_padding = circular_padding
    self._flatten_list = FlattenList(circular_padding=self._circular_padding)

  def forward(self, inputs):
    context_features, example_features, list_mask = inputs
    flat_ctx, flat_ex = self._flatten_list((context_features, example_features, list_mask))
    parts = [flat_ctx[k].reshape(flat_ctx[k].shape[0], -1) for k in sorted(flat_ctx)] + \
            [flat_ex[k].reshape(flat_ex[k].shape[0], -1) for k in sorted(flat_ex)]
    b, n = torch.as_tensor(list_mask).shape
    return torch.cat(parts, 1).reshape(b, n, -1)

  def get_config(self):
    return {'circular_padding': self._circular_padding}


class SelfAttentionMask(torch.nn.Module):
  """keras/layers.py:380-416: [batch_size, from_seq_length, to_seq_length] mask with
  mask[b, i, j] = to_mask[b, j], in the dtype of `inputs`."""

  def forward(self, inputs, to_mask=None):
    if isinstance(inputs, (list, tuple)) and to_mask is None:
      to_mask = inputs[1]
      inputs = inputs[0]
    inputs = torch.as_tensor(inputs)
    to_mask = torch.as_tensor(to_mask)
    b, f = inputs.shape[0], inputs.shape[1]
    t = to_mask.shape[1]
    ones = torch.ones(b, f, 1, dtype=inputs.dtype, device=inputs.device)
    return ones * to_mask.reshape(b, 1, t).to(inputs.dtype)

  def get_config(self):
    return {}


class _DINFn(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x, flat, m8, din):
    b, n, _ = x.shape
    out = torch.empty(b, n, din.head_size, dtype=torch.float32, device=x.device)
    ws = din._new_workspace(b, n)
    cfg = din._run_cfg()
    _C.check(_C.lib.tfr_din_fwd(_C.ptr(x), _C.ptr(m8), b, n, ctypes.byref(cfg), _C.ptr(flat),
                                _C.ptr(ws), _C.ptr(out), din.head_size, _C.stream()))
    ctx.cfg, ctx.ws = cfg, ws
    ctx.save_for_backward(x, flat, m8)
    return out

  @staticmethod
  def backward(ctx, g_out):
    x, flat, m8 = ctx.saved_tensors
    b, n, _ = x.shape
    grads = torch.empty_like(flat)
    g = g_out.contiguous()
    _C.check(_C.lib.tfr_din_bwd(_C.ptr(x), _C.ptr(m8), b, n, ctypes.byref(ctx.cfg),
                                _C.ptr(flat), _C.ptr(g), g.shape[-1], _C.ptr(ctx.ws),
                                _C.ptr(grads), _C.stream()))
    return None, grads, None, None


def _glorot(gen, shape, fan_in, fan_out):
  limit = math.sqrt(6.0 / (fan_in + fan_out))
  return (torch.rand(*shape, generator=gen, dtype=torch.float64) * 2 * limit - limit).float()


class DocumentInteractionAttention(torch.nn.Module):
  """keras/layers.py:420-588: `num_layers` layers of multi-head self-attention over the
  items of every list (Pasumarthi et al. 2020), after a Dense(head_size, relu) input
  projection and optional GaussianNoise.  Output [batch_size, list_size, head_size].

  Runs in the K11 kernels (csrc/din.cu, tfr_din_fwd / tfr_din_bwd).  All parameters live in
  ONE flat fp32 buffer (`flat`) in Keras get_weights() order (see include/tfr_b200.h).  The
  input dimension comes from the first call (or `build`).  Called as `din((x, list_mask))`;
  `train()` / `eval()` select Keras' `training`.  Gradients flow to the parameters only:
  inputs must not require grad.  Limits: input dim and head_size multiples of 4, head_size
  <= 128, num_heads * head_size <= 512, num_layers <= 8, list_size <= 1024.

  `precision`: None / 'fp32' (default) runs the projections in 3xTF32 and the attention core
  in FP32; 'tf32' runs the projections in one TF32 pass and the attention core on the TF32
  tensor cores (csrc/din_tc.cu), as TensorFlow's default TF32 matmuls and einsums do.  The
  parameters are the same in both, so `set_precision` can switch a trained layer."""

  def __init__(self, num_heads, head_size, num_layers=1, dropout=0.5, name=None,
               input_noise_stddev=None, seed=None, device='cuda', precision=None, **kwargs):
    super().__init__()
    self.set_precision(precision)
    self.num_heads = int(num_heads)
    self.head_size = int(head_size)
    self.num_layers = int(num_layers)
    self.dropout = float(dropout or 0.0)
    self.input_noise_stddev = input_noise_stddev
    self.name = name
    if not 0.0 <= self.dropout < 1.0:
      raise ValueError('dropout must be in [0, 1)')
    if input_noise_stddev is not None and float(input_noise_stddev) < 0:
      raise ValueError('input_noise_stddev must be >= 0')
    self._seed = seed
    self._device = device
    self._base = int(seed if seed is not None else torch.seed()) & 0xFFFFFFFF
    self._calls = 0
    self.register_parameter('flat', None)
    self._cfg = None

  @property
  def built(self):
    return self._cfg is not None

  def set_precision(self, precision):
    """None / 'fp32': 3xTF32 projections, FP32 attention core; 'tf32': all on TF32 tensor
    cores.  Takes effect from the next call."""
    if precision is None:
      precision = 'fp32'
    if precision not in _DIN_PRECISIONS:
      raise ValueError('precision must be one of %s' % sorted(_DIN_PRECISIONS))
    self.precision = precision
    self._precision = _DIN_PRECISIONS[precision]

  def _make_cfg(self, input_dim):
    cfg = _C.DinCfg()
    cfg.input_dim = int(input_dim)
    cfg.head_size = self.head_size
    cfg.num_heads = self.num_heads
    cfg.num_layers = self.num_layers
    cfg.dropout = self.dropout
    cfg.input_noise_stddev = float(self.input_noise_stddev or 0.0)
    cfg.training = 1
    cfg.seed = 0
    cfg.precision = self._precision
    return cfg

  def build(self, input_dim):
    """Creates the parameters (Keras initialisers: glorot_uniform kernels with the
    EinsumDense fan-in / fan-out of their 3-D shapes, zero biases, LayerNorm gamma ones /
    beta zeros)."""
    cfg = self._make_cfg(input_dim)
    n = _C.lib.tfr_din_param_count(ctypes.byref(cfg))
    if n == 0:
      raise ValueError(_C.last_error())
    d, h, heads = int(input_dim), self.head_size, self.num_heads
    gen = torch.Generator()
    if self._seed is not None:
      gen.manual_seed(self._seed)
    parts = [_glorot(gen, (d, h), d, h).reshape(-1), torch.zeros(h)]
    for _ in range(self.num_layers):
      for _ in range(3):   # query / key / value kernels [h, H, h]: fan_in H h, fan_out h h
        parts += [_glorot(gen, (h, heads, h), heads * h, h * h).reshape(-1),
                  torch.zeros(heads * h)]
      parts += [_glorot(gen, (heads, h, h), heads * h, heads * h).reshape(-1), torch.zeros(h),
                torch.ones(h), torch.zeros(h)]
    flat = torch.cat(parts)
    assert flat.numel() == n
    self.input_dim = d
    self._cfg = cfg
    self.dims = ['din', d, h, heads, self.num_layers]
    self.flat = torch.nn.Parameter(flat.to(self._device))
    return self

  def load_keras_weights(self, weights):
    """Loads Keras `get_weights()`: W_in, b_in, then per layer query kernel / bias, key
    kernel / bias, value kernel / bias, output kernel / bias, LayerNorm gamma / beta."""
    weights = [torch.as_tensor(w, dtype=torch.float32).reshape(-1) for w in weights]
    if not self.built:
      self.build(int(weights[0].numel() // self.head_size))
    flat = torch.cat(weights)
    if flat.numel() != self.flat.numel():
      raise ValueError('expected %d weights in total, got %d' %
                       (self.flat.numel(), flat.numel()))
    with torch.no_grad():
      self.flat.copy_(flat)

  def _run_cfg(self, training=None):
    cfg = _C.DinCfg()
    ctypes.memmove(ctypes.byref(cfg), ctypes.byref(self._cfg), ctypes.sizeof(cfg))
    training = self.training if training is None else training
    cfg.training = int(bool(training))
    cfg.precision = self._precision
    if training and (self.dropout > 0 or self.input_noise_stddev):
      self._calls += 1
    cfg.seed = (self._base << 32) | (self._calls & 0xFFFFFFFF)
    return cfg

  def _new_workspace(self, b, n):
    nbytes = _C.lib.tfr_din_workspace_bytes(ctypes.byref(self._cfg), b, n)
    if nbytes == 0:
      raise ValueError(_C.last_error())
    return torch.empty(nbytes, dtype=torch.uint8, device=self.flat.device)

  def forward(self, inputs):
    example_inputs, list_mask = inputs
    x = example_inputs
    _C.require_cuda(x, 'DocumentInteractionAttention inputs')
    if x.requires_grad:
      raise NotImplementedError(
          'gradients w.r.t. DocumentInteractionAttention inputs are not computed')
    if x.dim() != 3:
      raise ValueError('expected inputs [batch_size, list_size, feature_dims]')
    if not self.built:
      self.build(x.shape[-1])
    elif x.shape[-1] != self.input_dim:
      raise ValueError('expected last dim %d, got %d' % (self.input_dim, x.shape[-1]))
    x = x.float().contiguous()
    m8 = None
    if list_mask is not None:
      m8 = torch.as_tensor(list_mask, device=x.device).reshape(x.shape[:2]).to(
          torch.uint8).contiguous()
    return _DINFn.apply(x, self.flat, m8, self)

  def get_config(self):
    cfg = {'num_heads': self.num_heads, 'head_size': self.head_size,
           'num_layers': self.num_layers, 'dropout': self.dropout,
           'input_noise_stddev': self.input_noise_stddev}
    if self.precision != 'fp32':   # the default is left out, as before the option existed
      cfg['precision'] = self.precision
    return cfg


_COMBINERS = {'sum': _C.COMBINER_SUM, 'mean': _C.COMBINER_MEAN, 'sqrtn': _C.COMBINER_SQRTN}


class _TokenEmbeddingFn(torch.autograd.Function):

  @staticmethod
  def forward(ctx, ids, flat, layer):
    r, t = ids.shape
    out = torch.empty(r, layer.embedding_dim, dtype=torch.float32, device=ids.device)
    bad = torch.zeros(1, dtype=torch.int32, device=ids.device)
    _C.check(_C.lib.tfr_embedding_fwd(_C.ptr(ids), r, t, _C.ptr(flat), layer.vocab_size,
                                      layer.embedding_dim, layer._combiner, 1, _C.ptr(out),
                                      layer.embedding_dim, _C.ptr(bad), _C.stream()))
    n_bad = int(bad.item())
    if n_bad:
      raise ValueError('%d token ids lie outside [-1, %d)' % (n_bad, layer.vocab_size))
    ctx.layer = layer
    ctx.save_for_backward(ids)
    return out

  @staticmethod
  def backward(ctx, g_out):
    ids, = ctx.saved_tensors
    layer = ctx.layer
    r, t = ids.shape
    g = g_out.contiguous()
    grads = torch.empty(layer.vocab_size * layer.embedding_dim, dtype=torch.float32,
                        device=ids.device)
    ws = layer._new_workspace(r, t)
    _C.check(_C.lib.tfr_embedding_bwd(_C.ptr(ids), r, t, _C.ptr(g), layer.embedding_dim, 1,
                                      layer.vocab_size, layer.embedding_dim, layer._combiner,
                                      0, _C.ptr(ws), _C.ptr(grads), None, _C.stream()))
    return None, grads, None


class TokenEmbedding(torch.nn.Module):
  """A pooled embedding table: `tf.feature_column.embedding_column` over a categorical
  vocabulary column, or Keras `Embedding` followed by a reduction over the token axis
  (examples/keras/antique_kpl_din.py:256-278).

  forward(ids [..., T] int) -> [..., embedding_dim]: the combiner ('mean', 'sum' or
  'sqrtn') of the rows of the bag's ids in [0, vocab_size); -1 marks an empty slot.  A bag
  with no id pools to zeros (a Keras ragged reduce_mean would give NaN there).  An id that
  occurs twice counts twice.  Any other id raises ValueError (the kernel never reads it).
  The table is ONE flat fp32 parameter (`flat`, [vocab_size * embedding_dim] row-major),
  initialised as Keras Embedding does, uniform(-0.05, 0.05), from a generator seeded with
  `seed`.  Gradients flow to the table (csrc/embedding.cu, K12), not to the ids."""

  def __init__(self, vocab_size, embedding_dim, combiner='mean', seed=None, device='cuda',
               name=None):
    super().__init__()
    if combiner not in _COMBINERS:
      raise ValueError('combiner must be one of %s' % sorted(_COMBINERS))
    self.vocab_size = int(vocab_size)
    self.embedding_dim = int(embedding_dim)
    if self.vocab_size < 1 or self.embedding_dim < 1 or self.embedding_dim > 1024:
      raise ValueError('need vocab_size >= 1 and 1 <= embedding_dim <= 1024')
    self.combiner = combiner
    self._combiner = _COMBINERS[combiner]
    self.name = name
    gen = torch.Generator()
    gen.manual_seed(int(seed) if seed is not None else torch.seed())
    table = (torch.rand(self.vocab_size * self.embedding_dim, generator=gen,
                        dtype=torch.float64) * 0.1 - 0.05).float()
    self.flat = torch.nn.Parameter(table.to(device))
    self.dims = ['embedding', self.vocab_size, self.embedding_dim]

  @property
  def table(self):
    return self.flat.view(self.vocab_size, self.embedding_dim)

  def _new_workspace(self, r, t):
    nbytes = _C.lib.tfr_embedding_workspace_bytes(r, t, self.vocab_size, self.embedding_dim)
    if nbytes == 0:
      raise ValueError(_C.last_error())
    return torch.empty(nbytes, dtype=torch.uint8, device=self.flat.device)

  def forward(self, ids):
    _C.require_cuda(ids, 'TokenEmbedding ids')
    if ids.dim() < 1:
      raise ValueError('ids must have a token axis')
    lead = ids.shape[:-1]
    t = ids.shape[-1]
    flat_ids = ids.reshape(-1, t).to(torch.int32).contiguous()
    out = _TokenEmbeddingFn.apply(flat_ids, self.flat, self)
    return out.reshape(*lead, self.embedding_dim)

  def get_config(self):
    return {'vocab_size': self.vocab_size, 'embedding_dim': self.embedding_dim,
            'combiner': self.combiner}


class _BilinearFn(torch.autograd.Function):

  @staticmethod
  def forward(ctx, v1, v2, flat, layer):
    m = v1.shape[0]
    e, k = layer.embedding_dim, layer.output_dim
    out = torch.empty(m, k, dtype=torch.float32, device=v1.device)
    if m:
      _C.check(_C.lib.tfr_bilinear_fwd(_C.ptr(v1), _C.ptr(v2), m, e, k, _C.ptr(flat), None,
                                        _C.ptr(out), _C.stream()))
    ctx.layer = layer
    ctx.save_for_backward(v1, v2, flat)
    return out

  @staticmethod
  def backward(ctx, g_out):
    v1, v2, flat = ctx.saved_tensors
    layer = ctx.layer
    m = v1.shape[0]
    e, k = layer.embedding_dim, layer.output_dim
    dv1, dv2 = torch.empty_like(v1), torch.empty_like(v2)
    grads = torch.zeros_like(flat)
    if m:
      g = g_out.contiguous()
      ws = torch.empty(_C.lib.tfr_bilinear_workspace_bytes(m, e, k), dtype=torch.uint8,
                       device=v1.device)
      _C.check(_C.lib.tfr_bilinear_bwd(_C.ptr(v1), _C.ptr(v2), m, e, k, _C.ptr(flat), None,
                                        _C.ptr(g), _C.ptr(dv1), _C.ptr(dv2), _C.ptr(grads),
                                        _C.ptr(ws), _C.stream()))
    return dv1, dv2, grads, None


class Bilinear(torch.nn.Module):
  """keras/layers.py:807-890: the bilinear interaction of two vectors of the same width E,
  used by two-tower models for unbiased learning to rank (Yan et al., "Revisiting two tower
  models for unbiased learning to rank"):

      y[..., k] = v1 W[:, :, k] v2 + v1 W1[:, k] + v2 W2[:, k] + b[k]

  forward((v1, v2)) takes two tensors of the same shape [..., E] and returns [..., K].  Runs
  in the K14 kernels (csrc/bilinear.cu); gradients reach both inputs and the parameters.  The
  parameters are ONE flat fp32 parameter (`flat`) in Keras get_weights() order: W
  `bilinear_term` [E, E, K], W1 `linear_term_1` [E, K], W2 `linear_term_2` [E, K], b
  `const_term` [K], initialised as the reference does (RandomNormal(stddev=1/E) for W,
  RandomNormal(stddev=1/sqrt(E)) for W1 and W2, zeros for b) from a generator seeded with
  `seed`.  Limits: 1 <= E <= 128, 1 <= K <= 32, E * E * K <= 16384."""

  def __init__(self, embedding_dim, output_dim, seed=None, device='cuda', name=None):
    super().__init__()
    self.embedding_dim = int(embedding_dim)
    self.output_dim = int(output_dim)
    self.name = name
    e, k = self.embedding_dim, self.output_dim
    n = _C.lib.tfr_bilinear_param_count(e, k)
    if n == 0:
      raise ValueError(_C.last_error())
    gen = torch.Generator()
    gen.manual_seed(int(seed) if seed is not None else torch.seed())
    normal = lambda size, std: (torch.randn(size, generator=gen, dtype=torch.float64) *  # noqa
                                std).float()
    flat = torch.cat([normal(e * e * k, 1.0 / e), normal(e * k, 1.0 / math.sqrt(e)),
                      normal(e * k, 1.0 / math.sqrt(e)), torch.zeros(k)])
    assert flat.numel() == n
    self.flat = torch.nn.Parameter(flat.to(device))
    self.dims = ['bilinear', e, k]

  def _offsets(self):
    e, k = self.embedding_dim, self.output_dim
    return e * e * k, e * e * k + e * k, e * e * k + 2 * e * k

  def bilinear_term(self):
    e, k = self.embedding_dim, self.output_dim
    return self.flat[:e * e * k].view(e, e, k)

  def linear_term_1(self):
    a, b, _ = self._offsets()
    return self.flat[a:b].view(self.embedding_dim, self.output_dim)

  def linear_term_2(self):
    _, b, c = self._offsets()
    return self.flat[b:c].view(self.embedding_dim, self.output_dim)

  def const_term(self):
    _, _, c = self._offsets()
    return self.flat[c:c + self.output_dim]

  def load_keras_weights(self, weights):
    """Loads Keras `get_weights()`: [bilinear_term, linear_term_1, linear_term_2,
    const_term]."""
    parts = [torch.as_tensor(w, dtype=torch.float32).reshape(-1) for w in weights]
    flat = torch.cat(parts) if parts else torch.zeros(0)
    if len(parts) != 4 or flat.numel() != self.flat.numel():
      raise ValueError('expected the 4 weights of a Bilinear(%d, %d) (%d values), got %d arrays '
                       'with %d values' % (self.embedding_dim, self.output_dim,
                                           self.flat.numel(), len(parts), flat.numel()))
    with torch.no_grad():
      self.flat.copy_(flat)

  def forward(self, inputs):
    v1, v2 = inputs
    _C.require_cuda(v1, 'Bilinear inputs')
    _C.require_cuda(v2, 'Bilinear inputs')
    if v1.shape != v2.shape:
      raise ValueError('the two inputs must have the same shape, got %s and %s' %
                       (tuple(v1.shape), tuple(v2.shape)))
    if v1.dim() < 1 or v1.shape[-1] != self.embedding_dim:
      raise ValueError('expected last dim %d, got %s' % (self.embedding_dim, tuple(v1.shape)))
    lead = v1.shape[:-1]
    e = self.embedding_dim
    a = v1.reshape(-1, e).float().contiguous()
    c = v2.reshape(-1, e).float().contiguous()
    out = _BilinearFn.apply(a, c, self.flat, self)
    return out.reshape(*lead, self.output_dim)

  def get_config(self):
    return {'embedding_dim': self.embedding_dim, 'output_dim': self.output_dim}
