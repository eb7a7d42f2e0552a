"""Fused training step of the hot path (the reference's `model.fit` inner step,
keras/pipeline.py:605-632 and SURVEY.md §3.1):

    scores = scorer(x)                       tfr_mlp_fwd   (+ RestoreList fill)
    loss, d loss/d scores                    one fused loss kernel + 1-CTA reduce
    d loss/d params                          tfr_mlp_bwd   (flat gradient buffer)
    all-reduce(SUM) of the flat gradient     NCCL over NVLink (world_size > 1)
    params -= optimizer(grads / world_size)  tfr_optimizer_step

Data-parallel semantics follow the reference (extension/task.py:256-262):
each rank reduces its loss over its LOCAL batch, the loss is scaled by
1/num_replicas and gradients are summed — done here by one all-reduce of the
flat fp32 gradient and a 1/world_size factor inside the optimizer kernel.
"""
import ctypes

import torch

from ranking_b200 import _C
from ranking_b200 import dp

_OPT = {'sgd': 0, 'adagrad': 1}


class RankingTrainer(object):
  """Owns the static buffers of one training configuration [B, N, D].

  collective: how the data-parallel gradient sum is done when world_size > 1
    'fused' (default on CUDA ranks of one node): the all-reduce is part of the optimizer
            kernel — peer loads over NVLink, one flag round (csrc/dp_fused.cu, K7);
    'nccl'  one ncclAllReduce of the flat gradient, then the optimizer kernel.
  """

  def __init__(self, tower, loss, optimizer='adagrad', learning_rate=0.001,
               epsilon=1e-7, initial_accumulator_value=0.1, process_group=None,
               collective='fused', keep_summed_grads=False):
    if optimizer not in _OPT:
      raise ValueError('optimizer must be one of %s' % sorted(_OPT))
    if not hasattr(loss, 'fused_fwd_bwd'):
      raise ValueError('loss must be a ranking_b200.keras.losses object')
    if collective not in ('fused', 'nccl'):
      raise ValueError("collective must be 'fused' or 'nccl'")
    self.tower = tower
    self.loss = loss
    self.opt_kind = _OPT[optimizer]
    self.lr = float(learning_rate)
    self.eps = float(epsilon)
    dev = tower.flat.device
    self.device = dev
    self.accum = torch.full_like(tower.flat.data, initial_accumulator_value)
    self.group = process_group
    self.world = dp.world_size(process_group)
    self.reducer = None
    if self.world > 1 and collective == 'fused':
      self.reducer = dp.FusedGradReducer(tower.flat.numel(), dev, process_group)
      self.grads = self.reducer.grads()
      self.summed = torch.zeros_like(tower.flat.data) if keep_summed_grads else None
    else:
      self.grads = torch.zeros_like(tower.flat.data)
      self.summed = None
    self._shape = None
    self.launches_per_step = None

  # -- buffers ---------------------------------------------------------------
  def _ensure(self, b, n):
    if self._shape == (b, n):
      return
    dev = self.device
    m = b * n
    self.scores = torch.empty(b, n, dtype=torch.float32, device=dev)
    self.dscores = torch.empty(b, n, dtype=torch.float32, device=dev)
    self.per_list = torch.empty(2, b, dtype=torch.float32, device=dev)
    self.total2 = torch.zeros(2, dtype=torch.float32, device=dev)
    self.ws = self._new_workspace(b, n)
    self._shape = (b, n)

  def _new_workspace(self, b, n):
    return self.tower._new_workspace(b * n)

  def _prep_x(self, x):
    t = self.tower
    if x.dtype != t.input_dtype or not x.is_contiguous():
      x = x.to(t.input_dtype).contiguous()   # bf16 mode wants bf16 features in HBM
    return x

  def _circular_pad(self, x, valid):
    """FlattenList(circular_padding=True) (keras/layers.py:163-173): with BatchNormalization
    in the tower the batch statistics must only see copies of VALID rows, so padded slots
    are filled circularly with the list's valid items before the tower (K9).  Only done
    when the tower normalises; without BN padded rows cannot influence valid ones."""
    t = self.tower
    if not (t.use_batch_norm or t.input_batch_norm) or valid is None:
      return x
    b, n, d = x.shape
    if getattr(self, '_xg', None) is None or self._xg.shape != x.shape or \
        self._xg.dtype != x.dtype:
      self._xg = torch.empty_like(x)
      self._pad_idx = torch.empty(b, n, dtype=torch.int32, device=x.device)
    row_bytes = d * x.element_size()
    if row_bytes % 16:
      raise ValueError('circular padding needs feature rows that are multiples of 16 bytes')
    v8 = valid.reshape(b, n).to(torch.uint8).contiguous()
    _C.check(_C.lib.tfr_circular_pad_gather(_C.ptr(x), _C.ptr(v8), b, n, row_bytes,
                                            _C.ptr(self._pad_idx), _C.ptr(self._xg),
                                            _C.stream()))
    return self._xg

  # -- scorer forward / backward (overridden by the groupwise trainer) ----------
  def _forward(self, x, y_true, m8, cfg, training):
    b, n, _ = x.shape
    t = self.tower
    _C.check(_C.lib.tfr_mlp_fwd(_C.ptr(x), b * n, cfg, _C.ptr(t.flat.data),
                                _C.ptr(m8), _C.ptr(self.ws), _C.ptr(self.scores),
                                t._precision, _C.stream()))

  def _backward(self, x, m8, cfg, grads):
    b, n, _ = x.shape
    t = self.tower
    _C.check(_C.lib.tfr_mlp_bwd(_C.ptr(x), b * n, cfg, _C.ptr(t.flat.data),
                                _C.ptr(self.dscores), _C.ptr(m8), _C.ptr(self.ws),
                                _C.ptr(grads), t._precision, _C.stream()))

  def _apply(self, grads):
    """Gradient sum over the replicas + optimizer update."""
    t = self.tower
    if self.reducer is not None:
      self.reducer.step(t.flat.data, self.accum, self.opt_kind, self.lr, self.eps,
                        summed_out=self.summed)
      return
    dp.all_reduce_sum_(grads, self.group)   # 'nccl': the one collective of the step
    _C.check(_C.lib.tfr_optimizer_step(
        _C.ptr(t.flat.data), _C.ptr(grads), _C.ptr(self.accum), grads.numel(),
        self.opt_kind, self.lr, self.eps, dp.replica_grad_scale(self.group), _C.stream()))

  # -- one step on device-resident inputs -------------------------------------
  def train_step(self, x, y_true, sample_weight=None, mask=None):
    """x [B, N, D] (device; fp32, or bf16 in the bf16 mode), y_true [B, N] (label < 0 =
    padding).  Returns the scalar loss as a 0-d device tensor (no host sync)."""
    b, n, d = x.shape
    self._ensure(b, n)
    x = self._prep_x(x)
    run_cfg = self.tower._run_cfg(training=True)
    cfg = ctypes.byref(run_cfg)
    m8 = None
    if mask is not None:
      m8 = mask.reshape(-1).to(torch.uint8).contiguous()
    grads = self.reducer.grads() if self.reducer is not None else self.grads
    self.grads = grads
    x = self._circular_pad(x, mask if mask is not None else (y_true >= 0))
    self._forward(x, y_true, m8, cfg, True)
    self.loss.fused_fwd_bwd(y_true, self.scores, sample_weight, self.dscores,
                            self.per_list, self.total2)
    self._backward(x, m8, cfg, grads)
    self._apply(grads)
    return self.total2[0]

  # -- evaluation --------------------------------------------------------------
  @torch.no_grad()
  def predict(self, x, mask=None, y_true=None):
    b, n, d = x.shape
    self._ensure(b, n)
    x = self._prep_x(x)
    m8 = None if mask is None else mask.reshape(-1).to(torch.uint8).contiguous()
    cfg = ctypes.byref(self.tower._run_cfg(training=False))
    valid = mask if mask is not None else (None if y_true is None else y_true >= 0)
    x = self._circular_pad(x, valid)
    self._forward(x, y_true, m8, cfg, False)
    return self.scores


class GroupwiseRankingTrainer(RankingTrainer):
  """Fused step for groupwise scoring (tfr.model._GroupwiseRankingModel, model.py:273-421):
  `tower` is the group score function over the concatenated member features
  (input_dim = group_size * D, output_units = group_size).  Group formation, the folded
  first layer, the scatter-average and their backward run in csrc/mlp_group.cu; the
  [B, G, group_size, D] gather of the reference is never formed.  Validity = label >= 0
  (model.py `_infer_sizes`); `permutations` ([num_shuffles, B, N] int, optional) are the
  shuffles of the valid-first order (identity = the reference's PREDICT mode)."""

  def __init__(self, tower, loss, group_size, num_shuffles=1, **kw):
    super().__init__(tower, loss, **kw)
    if group_size <= 0:
      raise ValueError('Invalid group_size %d' % group_size)
    if tower.output_units != group_size or tower.input_dim % group_size:
      raise ValueError('the group score tower needs input_dim = group_size * D and '
                       'output_units = group_size')
    self.group_size = int(group_size)
    self.num_shuffles = int(num_shuffles)
    self.permutations = None

  def _new_workspace(self, b, n):
    g = self.num_shuffles * n
    nbytes = _C.lib.tfr_group_mlp_workspace_bytes(ctypes.byref(self.tower._cfg), b, n, g,
                                                  self.group_size)
    if nbytes == 0:
      raise ValueError(_C.last_error())
    dev = self.device
    self.idx = torch.empty(b, g, self.group_size, dtype=torch.int32, device=dev)
    self.gmask = torch.empty(b, g, dtype=torch.uint8, device=dev)
    return torch.empty(nbytes, dtype=torch.uint8, device=dev)

  def _forward(self, x, y_true, m8, cfg, training):
    b, n, _ = x.shape
    t = self.tower
    if y_true is None:
      valid = torch.ones(b, n, dtype=torch.uint8, device=self.device)
    else:
      valid = (y_true >= 0).to(torch.uint8).contiguous()
    perm = self.permutations
    if perm is not None:
      perm = perm.to(torch.int32).contiguous()
    g = self.num_shuffles * n
    st = _C.stream()
    _C.check(_C.lib.tfr_group_indices(_C.ptr(valid), _C.ptr(perm), b, n, self.num_shuffles,
                                      self.group_size, _C.ptr(self.idx), _C.ptr(self.gmask),
                                      st))
    _C.check(_C.lib.tfr_group_mlp_fwd(_C.ptr(x), b, n, g, self.group_size, _C.ptr(self.idx),
                                      _C.ptr(self.gmask), cfg, _C.ptr(t.flat.data),
                                      _C.ptr(self.ws), _C.ptr(self.scores), t._precision, st))

  def _backward(self, x, m8, cfg, grads):
    b, n, _ = x.shape
    t = self.tower
    g = self.num_shuffles * n
    _C.check(_C.lib.tfr_group_mlp_bwd(_C.ptr(x), b, n, g, self.group_size, _C.ptr(self.idx),
                                      _C.ptr(self.gmask), cfg, _C.ptr(t.flat.data),
                                      _C.ptr(self.dscores), _C.ptr(self.ws), _C.ptr(grads),
                                      t._precision, _C.stream()))


class GAMRankingTrainer(RankingTrainer):
  """Fused step for the neural additive model (GAMLayer, keras/layers.py:591-803), as in
  the reference's canned-GAM recipe (examples/tf_ranking_canned_gam.py): example features
  only.  `x` is dense [B, N, D] and `feature_dims` partitions D into the F features, in
  order; `gam` is a `keras.layers.GAMLayer` (built here for those widths if it has not
  been).  The towers run in csrc/gam.cu (tfr_gam_fwd / tfr_gam_bwd); circular padding,
  the fused loss, the optimizer / all-reduce, fit, evaluate and checkpoints are the base
  class's."""

  def __init__(self, gam, loss, feature_dims, **kw):
    feature_dims = [int(d) for d in feature_dims]
    if not gam.built:
      gam.build(feature_dims)
    elif gam.example_dims != feature_dims:
      raise ValueError('feature_dims %s, the GAM was built for %s' %
                       (feature_dims, gam.example_dims))
    super().__init__(gam, loss, **kw)
    self.feature_dims = feature_dims

  def _forward(self, x, y_true, m8, cfg, training):
    b, n, d = x.shape
    if d != sum(self.feature_dims):
      raise ValueError('x has %d features, feature_dims sum to %d' %
                       (d, sum(self.feature_dims)))
    _C.check(_C.lib.tfr_gam_fwd(_C.ptr(x), None, b * n, cfg, _C.ptr(self.tower.flat.data),
                                _C.ptr(m8), _C.ptr(self.ws), _C.ptr(self.scores), None, None,
                                _C.stream()))

  def _backward(self, x, m8, cfg, grads):
    b, n, _ = x.shape
    _C.check(_C.lib.tfr_gam_bwd(_C.ptr(x), None, b * n, cfg, _C.ptr(self.tower.flat.data),
                                _C.ptr(self.dscores), _C.ptr(m8), _C.ptr(self.ws),
                                _C.ptr(grads), _C.stream()))


class HostBatchPipeline(object):
  """End-to-end step from HOST buffers: pinned-memory batches are copied to the
  device on a copy stream, double-buffered so the copy of batch k+1 overlaps the
  compute of batch k; the scalar loss of every step is read back to the host."""

  def __init__(self, trainer, b, n, d):
    self.trainer = trainer
    dev = trainer.device
    self.copy_stream = torch.cuda.Stream(device=dev)
    xdt = trainer.tower.input_dtype    # bf16 mode: features travel and live as bf16
    self.x = [torch.empty(b, n, d, dtype=xdt, device=dev) for _ in range(2)]
    self.y = [torch.empty(b, n, dtype=torch.float32, device=dev) for _ in range(2)]
    self.ready = [torch.cuda.Event() for _ in range(2)]
    self.free = [torch.cuda.Event() for _ in range(2)]
    self.done = [torch.cuda.Event() for _ in range(2)]
    self.loss_host = torch.zeros(2, dtype=torch.float32).pin_memory()
    self.h2d_bytes = b * n * d * self.x[0].element_size() + b * n * 4
    self.d2h_bytes = 4
    self._slot = 0
    self._primed = False

  def _upload(self, slot, x_host, y_host):
    with torch.cuda.stream(self.copy_stream):
      self.copy_stream.wait_event(self.free[slot])
      self.x[slot].copy_(x_host, non_blocking=True)
      self.y[slot].copy_(y_host, non_blocking=True)
      self.ready[slot].record(self.copy_stream)

  def run(self, host_batches, sample_weight=None):
    """host_batches: sequence of (x_pinned [B,N,D], y_pinned [B,N]).  Returns the
    list of per-step losses (python floats).  The loss of step k is copied to its
    pinned slot right after the step and READ one step late (after step k + 1 has been
    queued), so the host never drains the GPU between steps."""
    tr = self.trainer
    cur = torch.cuda.current_stream()
    losses = []
    it = iter(host_batches)
    nxt = next(it, None)
    if nxt is None:
      return losses
    for s in range(2):
      self.free[s].record(cur)
    slot = 0
    self._upload(slot, *nxt)
    pending = None                   # (slot, event) of the step whose loss is in flight
    while nxt is not None:
      upcoming = next(it, None)
      if upcoming is not None:
        self._upload(slot ^ 1, *upcoming)
      cur.wait_event(self.ready[slot])
      loss = tr.train_step(self.x[slot], self.y[slot], sample_weight)
      self.free[slot].record(cur)
      self.loss_host[slot].copy_(loss, non_blocking=True)
      self.done[slot].record(cur)
      if pending is not None:
        pending[1].synchronize()
        losses.append(float(self.loss_host[pending[0]]))
      pending = (slot, self.done[slot])
      nxt = upcoming
      slot ^= 1
    pending[1].synchronize()
    losses.append(float(self.loss_host[pending[0]]))
    return losses
