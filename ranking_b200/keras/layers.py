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
    return None, grads, None, None


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
    if x.requires_grad:
      raise NotImplementedError('gradients w.r.t. tower inputs are not computed')
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
