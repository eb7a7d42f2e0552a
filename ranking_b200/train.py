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

_OPT = {'sgd': 0, 'adagrad': 1, 'adamw': 2}


class PolynomialWarmUp(object):
  """Learning rate of BERT's recipe, evaluated on the host per optimizer step (0-based):
  linear warmup to `initial_learning_rate` over `warmup_steps`, then polynomial decay with
  power 1 to `end_learning_rate` at `decay_steps` (tf-models' PolynomialWarmUp over
  PolynomialDecay, power 1):
      lr(t) = initial * t / warmup_steps                                    t < warmup_steps
      lr(t) = end + (initial - end) * (1 - min(t, decay_steps) / decay_steps)   otherwise"""

  def __init__(self, initial_learning_rate, decay_steps, warmup_steps=0,
               end_learning_rate=0.0):
    if decay_steps < 1 or warmup_steps < 0:
      raise ValueError('decay_steps must be >= 1 and warmup_steps >= 0')
    self.initial_learning_rate = float(initial_learning_rate)
    self.decay_steps = int(decay_steps)
    self.warmup_steps = int(warmup_steps)
    self.end_learning_rate = float(end_learning_rate)

  def __call__(self, step):
    step = int(step)
    if step < self.warmup_steps:
      return self.initial_learning_rate * step / self.warmup_steps
    frac = 1.0 - min(step, self.decay_steps) / self.decay_steps
    return self.end_learning_rate + (self.initial_learning_rate - self.end_learning_rate) * frac


class RankingTrainer(object):
  """Owns the static buffers of one training configuration [B, N, D].

  collective: how the data-parallel gradient sum is done when world_size > 1
    'fused' (default on CUDA ranks of one node): the all-reduce is part of the optimizer
            kernel — peer loads over NVLink, one flag round (csrc/dp_fused.cu, K7);
    'nccl'  one ncclAllReduce of the flat gradient, then the optimizer kernel.

  optimizer 'adamw' (tfr_adamw_step): accum holds [m | v]; `adam_step` counts the updates
  and checkpoints keep it; `learning_rate` may be a float or a schedule called with the
  0-based update index (PolynomialWarmUp); tower.decay_mask (uint8 per parameter, if the
  tower has one) picks the weights that decay.  Needs world size 1 or collective 'nccl'.

  gradient_clip_norm (adamw only, world size 1; default None = off): tf-models'
  AdamWeightDecay clipping, g *= clip / max(||g||, clip) over the whole flat gradient
  (tfr_global_norm, then tfr_adamw_step_clipped, which scales g inside the update).
  `grad_norm` is then a 0-d device tensor holding the last step's pre-clip norm.
  """

  def __init__(self, tower, loss, optimizer='adagrad', learning_rate=0.001,
               epsilon=1e-7, initial_accumulator_value=0.1, process_group=None,
               collective='fused', keep_summed_grads=False, beta_1=0.9, beta_2=0.999,
               weight_decay_rate=0.0, gradient_clip_norm=None):
    if optimizer not in _OPT:
      raise ValueError('optimizer must be one of %s' % sorted(_OPT))
    if not hasattr(loss, 'fused_fwd_bwd'):
      raise ValueError('loss must be a ranking_b200.keras.losses object')
    if collective not in ('fused', 'nccl'):
      raise ValueError("collective must be 'fused' or 'nccl'")
    self.tower = tower
    self.loss = loss
    self.opt_kind = _OPT[optimizer]
    self.lr = learning_rate if callable(learning_rate) else float(learning_rate)
    self.eps = float(epsilon)
    dev = tower.flat.device
    self.device = dev
    self.group = process_group
    self.world = dp.world_size(process_group)
    self.gradient_clip_norm = None
    if gradient_clip_norm is not None:
      clip = float(gradient_clip_norm)
      if optimizer != 'adamw':
        raise ValueError("gradient_clip_norm needs optimizer 'adamw', got %r" % optimizer)
      if self.world > 1:
        # tf-models clips each replica's gradient before the all-reduce; this trainer only
        # sees the sum
        raise ValueError('gradient_clip_norm supports one rank only, got world size %d' %
                         self.world)
      if not (clip > 0.0 and clip != float('inf')):
        raise ValueError('gradient_clip_norm must be finite and > 0, got %r' %
                         (gradient_clip_norm,))
      self.gradient_clip_norm = clip
      n = tower.flat.numel()
      self.grad_norm = torch.zeros((), dtype=torch.float32, device=dev)
      self._norm_ws = torch.empty(_C.lib.tfr_global_norm_workspace_bytes(n),
                                  dtype=torch.uint8, device=dev)
    if optimizer == 'adamw':
      if self.world > 1 and collective == 'fused':
        raise ValueError("optimizer 'adamw' with more than one rank needs collective='nccl'")
      self.accum = torch.zeros(2 * tower.flat.numel(), dtype=torch.float32, device=dev)
      self.adam_step = 0
      self.beta_1, self.beta_2 = float(beta_1), float(beta_2)
      self.weight_decay_rate = float(weight_decay_rate)
      self.decay_mask = getattr(tower, 'decay_mask', None)
    else:
      self.accum = torch.full_like(tower.flat.data, initial_accumulator_value)
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
    if self.opt_kind == _OPT['adamw']:
      lr = self.lr(self.adam_step) if callable(self.lr) else self.lr
      self.adam_step += 1
      n = grads.numel()
      if self.gradient_clip_norm is not None:
        _C.check(_C.lib.tfr_global_norm(_C.ptr(grads), n, _C.ptr(self.grad_norm),
                                         _C.ptr(self._norm_ws), self._norm_ws.numel(),
                                         _C.stream()))
        _C.check(_C.lib.tfr_adamw_step_clipped(
            _C.ptr(t.flat.data), _C.ptr(grads), _C.ptr(self.accum[:n]),
            _C.ptr(self.accum[n:]), _C.ptr(self.decay_mask), n, lr, self.beta_1, self.beta_2,
            self.eps, self.weight_decay_rate, self.adam_step, dp.replica_grad_scale(self.group),
            self.gradient_clip_norm, _C.ptr(self.grad_norm), _C.stream()))
        return
      _C.check(_C.lib.tfr_adamw_step(
          _C.ptr(t.flat.data), _C.ptr(grads), _C.ptr(self.accum[:n]), _C.ptr(self.accum[n:]),
          _C.ptr(self.decay_mask), n, lr, self.beta_1, self.beta_2, self.eps,
          self.weight_decay_rate, self.adam_step, dp.replica_grad_scale(self.group),
          _C.stream()))
      return
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


_MAX_TASKS = 8


class _TaskPlanes(object):
  """The task handling every multi-task trainer shares; mixed in before a single-task
  trainer, whose scorer then writes task-major score planes [T, B, N] and reads T dscore
  planes.  `losses` is an ordered dict task -> `ranking_b200.keras.losses` object; dict order
  is the order of the scorer's output units.  `loss_weights` maps tasks to weights (missing:
  1.0).  One step is

      scorer forward             task-major score planes, RestoreList on each
      loss_t.fused_fwd_bwd       one per task, on plane t, into dscore plane t
      scorer backward            applies w_t as it reads dscore plane t
      optimizer / all-reduce     as RankingTrainer

  and returns sum_t w_t L_t (each L_t reduced by its own loss's reduction), the Keras
  compile-time `loss_weights` semantics, as a 0-d device tensor; `task_losses` holds the
  [T] per-task values of the last step."""

  def _set_tasks(self, losses, loss_weights, output_units):
    """Checks the tasks against the scorer's output units; returns the first task's loss."""
    losses = dict(losses)
    if not losses:
      raise ValueError('losses must name at least one task')
    if len(losses) > _MAX_TASKS:
      raise ValueError('at most %d tasks, got %d' % (_MAX_TASKS, len(losses)))
    for name, loss in losses.items():
      if not getattr(loss, 'fused_single_score', False):
        raise ValueError('task %r: %s has no single-score fused step' %
                         (name, type(loss).__name__))
    weights = dict(loss_weights or {})
    unknown = sorted(set(weights) - set(losses))
    if unknown:
      raise ValueError('loss_weights name unknown tasks %s (tasks: %s)' %
                       (unknown, list(losses)))
    if output_units != len(losses):
      raise ValueError('the tower has %d output units for %d tasks' %
                       (output_units, len(losses)))
    self.tasks = list(losses)
    self.losses = losses
    self.loss_weights = [float(weights.get(t, 1.0)) for t in self.tasks]
    if not all(w == w and abs(w) != float('inf') for w in self.loss_weights):
      raise ValueError('loss weights must be finite: %s' % self.loss_weights)
    return losses[self.tasks[0]]

  def _set_task_weights(self):
    """After RankingTrainer.__init__: the weights as the backward and the loss sum take them."""
    t = len(self.tasks)
    self._w_host = (ctypes.c_float * t)(*self.loss_weights)
    # tfr_weighted_sum over the [T, 2] task totals {L_t, sum of weights}: (w_t, 0) pairs
    self._w_pairs = torch.tensor([[w, 0.0] for w in self.loss_weights], dtype=torch.float32,
                                 device=self.device).reshape(-1)
    self.total2 = torch.zeros(2, dtype=torch.float32, device=self.device)

  def _ensure(self, b, n):
    if self._shape == (b, n):
      return
    t, dev = len(self.tasks), self.device
    self.scores = torch.empty(t, b, n, dtype=torch.float32, device=dev)
    self.dscores = torch.empty(t, b, n, dtype=torch.float32, device=dev)
    self.per_list = torch.empty(t, 2, b, dtype=torch.float32, device=dev)
    self.task_totals = torch.zeros(t, 2, dtype=torch.float32, device=dev)
    self.task_losses = self.task_totals[:, 0]
    self.ws = self._new_workspace(b, n)
    self._shape = (b, n)

  def _labels(self, labels):
    missing = [t for t in self.tasks if t not in labels]
    if missing or len(labels) != len(self.tasks):
      raise ValueError('labels must map exactly the tasks %s (got %s)' %
                       (self.tasks, sorted(labels)))
    return [labels[t] for t in self.tasks]

  @staticmethod
  def _any_label(ys):
    mask = ys[0] >= 0
    for y in ys[1:]:
      mask = mask | (y >= 0)
    return mask

  def train_step(self, x, labels, sample_weight=None, mask=None):
    """x [B, N, D] (device), labels {task: [B, N]} (label < 0: no label for that task),
    sample_weight [B, N] or [B] shared by the tasks, mask [B, N] the list mask (default: any
    task has a label >= 0).  Returns sum_t w_t L_t as a 0-d device tensor (no host sync)."""
    b, n, d = x.shape
    ys = self._labels(labels)
    self._ensure(b, n)
    x = self._prep_x(x)
    if mask is None:
      mask = self._any_label(ys)
    m8 = mask.reshape(-1).to(torch.uint8).contiguous()
    cfg = ctypes.byref(self.tower._run_cfg(training=True))
    grads = self.reducer.grads() if self.reducer is not None else self.grads
    self.grads = grads
    x = self._circular_pad(x, mask)
    self._forward(x, None, m8, cfg, True)
    for i, task in enumerate(self.tasks):
      self.losses[task].fused_fwd_bwd(ys[i], self.scores[i], sample_weight, self.dscores[i],
                                      self.per_list[i], self.task_totals[i])
    _C.check(_C.lib.tfr_weighted_sum(_C.ptr(self.task_totals), _C.ptr(self._w_pairs),
                                     2 * len(self.tasks), 1.0, _C.ptr(self.total2),
                                     _C.stream()))
    self._backward(x, m8, cfg, grads)
    self._apply(grads)
    return self.total2[0]

  @torch.no_grad()
  def predict(self, x, mask=None, labels=None):
    """{task: [B, N] score view}; masked items (`mask`, else items without any label >= 0
    when `labels` is given) hold ln(1e-10) in every task's plane."""
    if mask is None and labels is not None:
      mask = self._any_label(self._labels(labels))
    scores = super().predict(x, mask=mask)
    return {t: scores[i] for i, t in enumerate(self.tasks)}


class MultiTaskRankingTrainer(_TaskPlanes, RankingTrainer):
  """Fused step for several ranking tasks on one tower (the reference's multi-task
  `UnivariateScorer` with `MultiTaskPipeline`'s per-task losses and `loss_weights`,
  keras/model.py:755-777 and keras/pipeline.py:733-824): `tower.output_units ==
  len(losses)`, the scorer forward / backward are tfr_mlp_fwd_tasks / tfr_mlp_bwd_tasks, and
  the rest of the step is _TaskPlanes'."""

  def __init__(self, tower, losses, loss_weights=None, **kw):
    first = self._set_tasks(losses, loss_weights, tower.output_units)
    if tower._precision not in (_C.PREC_FP32, _C.PREC_TF32X3, _C.PREC_TF32):
      raise ValueError('multi-task towers need precision fp32, tf32x3 or tf32')
    super().__init__(tower, first, **kw)
    self._set_task_weights()

  def _forward(self, x, y_true, m8, cfg, training):
    b, n, _ = x.shape
    t = self.tower
    _C.check(_C.lib.tfr_mlp_fwd_tasks(_C.ptr(x), b * n, cfg, _C.ptr(t.flat.data), _C.ptr(m8),
                                      _C.ptr(self.ws), _C.ptr(self.scores), t._precision,
                                      _C.stream()))

  def _backward(self, x, m8, cfg, grads):
    b, n, _ = x.shape
    t = self.tower
    _C.check(_C.lib.tfr_mlp_bwd_tasks(_C.ptr(x), b * n, cfg, _C.ptr(t.flat.data),
                                      _C.ptr(self.dscores), self._w_host, _C.ptr(m8),
                                      _C.ptr(self.ws), _C.ptr(grads), t._precision,
                                      _C.stream()))


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


class _DINScorer(object):
  """DocumentInteractionAttention + tower as one scorer with ONE flat parameter buffer: the
  DIN's parameters first, then the tower's (the modules' `flat` become views of it), so the
  step keeps one gradient all-reduce and one optimizer launch."""

  def __init__(self, din, tower):
    self.n_din = din.flat.numel()
    self.flat = torch.nn.Parameter(torch.cat([din.flat.data, tower.flat.data]))
    din.flat = torch.nn.Parameter(self.flat.data[:self.n_din])
    tower.flat = torch.nn.Parameter(self.flat.data[self.n_din:])
    self.bn_state = tower.bn_state
    self.dims = [list(din.dims), list(tower.dims)]
    self.use_batch_norm = tower.use_batch_norm
    self.input_batch_norm = tower.input_batch_norm
    self.input_dtype = torch.float32
    self._run_cfg = tower._run_cfg


class DINRankingTrainer(RankingTrainer):
  """Fused step for the listwise-context scorer of the reference's DIN examples
  (examples/keras/antique_kpl_din.py): the DocumentInteractionAttention embedding E of
  every item becomes an extra input column block of a create_tower tower:

      [X | E] with E = din((X, list_mask))    tfr_din_fwd writes E into columns [D, D + h)
      scores = tower([X | E])                 tfr_mlp_fwd
      loss, d loss / d scores                 fused loss kernel
      tower gradients, d loss / d E           tfr_mlp_bwd, tfr_mlp_input_grad
      DIN gradients                           tfr_din_bwd
      optimizer                               one launch over the shared flat buffer

  `tower` needs input_dim = D + head_size, precision tf32x3 or tf32, at least one hidden
  layer and no input BN.  With BN in the tower the items are circularly padded before the
  DIN (K9), as FlattenList / ConcatFeatures do in the reference; list validity is `mask`,
  or label >= 0.  fit / evaluate / checkpoints are the base class's."""

  def __init__(self, din, tower, loss, **kw):
    if not din.built:
      din.build(tower.input_dim - din.head_size)
    if tower.input_dim != din.input_dim + din.head_size:
      raise ValueError('the tower needs input_dim = %d (features) + %d (head_size), got %d' %
                       (din.input_dim, din.head_size, tower.input_dim))
    if tower.precision not in ('tf32x3', 'tf32') or tower.input_batch_norm or \
        not tower.hidden_layer_dims:
      raise ValueError('the tower must use precision tf32x3 or tf32, have a hidden layer and '
                       'no input BatchNormalization (its input gradient feeds the DIN)')
    self.din = din
    self.mlp = tower
    super().__init__(_DINScorer(din, tower), loss, **kw)

  def _new_workspace(self, b, n):
    dev = self.device
    h = self.din.head_size
    self.xe = torch.empty(b * n, self.mlp.input_dim, dtype=torch.float32, device=dev)
    self.d_emb = torch.empty(b * n, h, dtype=torch.float32, device=dev)
    self.din_ws = self.din._new_workspace(b, n)
    return self.mlp._new_workspace(b * n)

  def _forward(self, x, y_true, m8, cfg, training):
    b, n, d = x.shape
    din, width = self.din, self.mlp.input_dim
    if d != din.input_dim:
      raise ValueError('x has %d features, the DIN was built for %d' % (d, din.input_dim))
    lm = m8
    if lm is None and y_true is not None:
      lm = (y_true >= 0).reshape(-1).to(torch.uint8).contiguous()
    self._lm = lm
    self._din_cfg = din._run_cfg(training=training)
    self.xe.view(b, n, width)[..., :d].copy_(x)
    st = _C.stream()
    _C.check(_C.lib.tfr_din_fwd(_C.ptr(x), _C.ptr(lm), b, n, ctypes.byref(self._din_cfg),
                                _C.ptr(din.flat.data), _C.ptr(self.din_ws),
                                ctypes.c_void_p(self.xe.data_ptr() + 4 * d), width, st))
    self._tower_fwd(b * n, m8, cfg, st)

  def _tower_fwd(self, m, m8, cfg, st):
    _C.check(_C.lib.tfr_mlp_fwd(_C.ptr(self.xe), m, cfg, _C.ptr(self.mlp.flat.data),
                                _C.ptr(m8), _C.ptr(self.ws), _C.ptr(self.scores),
                                self.mlp._precision, st))

  def _tower_bwd(self, m, m8, cfg, tower_grads, st):
    _C.check(_C.lib.tfr_mlp_bwd(_C.ptr(self.xe), m, cfg, _C.ptr(self.mlp.flat.data),
                                _C.ptr(self.dscores), _C.ptr(m8), _C.ptr(self.ws), tower_grads,
                                self.mlp._precision, st))

  def _backward(self, x, m8, cfg, grads):
    b, n, d = x.shape
    din, mlp = self.din, self.mlp
    n_din = self.tower.n_din
    st = _C.stream()
    self._tower_bwd(b * n, m8, cfg, ctypes.c_void_p(grads.data_ptr() + 4 * n_din), st)
    _C.check(_C.lib.tfr_mlp_input_grad(cfg, b * n, _C.ptr(mlp.flat.data), _C.ptr(self.ws), d,
                                       din.head_size, _C.ptr(self.d_emb), din.head_size,
                                       mlp._precision, st))
    _C.check(_C.lib.tfr_din_bwd(_C.ptr(x), _C.ptr(self._lm), b, n,
                                ctypes.byref(self._din_cfg), _C.ptr(din.flat.data),
                                _C.ptr(self.d_emb), din.head_size, _C.ptr(self.din_ws),
                                _C.ptr(grads), st))


class _DASALCJoint(object):
  """DocumentInteractionAttention + DASALCScorer with ONE flat parameter buffer, the DIN's
  parameters first (the modules' `flat` become views of it), as _DINScorer."""

  def __init__(self, din, scorer):
    self.n_din = din.flat.numel()
    self.flat = torch.nn.Parameter(torch.cat([din.flat.data, scorer.flat.data]))
    din.flat = torch.nn.Parameter(self.flat.data[:self.n_din])
    scorer.flat = torch.nn.Parameter(self.flat.data[self.n_din:])
    self.bn_state = scorer.bn_state
    self.dims = [list(din.dims), list(scorer.dims)]
    self.use_batch_norm = True
    self.input_batch_norm = True
    self.input_dtype = torch.float32
    self._run_cfg = scorer._run_cfg


class DASALCRankingTrainer(RankingTrainer):
  """Fused step for DASALC (research/dasalc.py): raw features x [B, N, D] go through

      log1p_cutoff                            tfr_symmetric_log1p_clip
      circular padding of the padded items    tfr_circular_pad_gather (K9)
      E = din((x, list_mask))                 tfr_din_fwd
      scores = scorer((x, E))                 tfr_dasalc_fwd (K13)
      loss, d loss / d scores                 fused loss kernel
      scorer gradients, d loss / d E          tfr_dasalc_bwd
      DIN gradients                           tfr_din_bwd
      optimizer                               one launch over the shared flat buffer

  `din` is a DocumentInteractionAttention (built here for scorer.input_dim if it has not
  been) with head_size == scorer.context_dim.  List validity is `mask`, or label >= 0.
  predict runs the same chain in inference mode; fit / evaluate / checkpoints are the base
  class's."""

  def __init__(self, din, scorer, loss, cutoff=30.0, **kw):
    if not din.built:
      din.build(scorer.input_dim)
    if din.input_dim != scorer.input_dim:
      raise ValueError('the DIN was built for %d features, the scorer takes %d' %
                       (din.input_dim, scorer.input_dim))
    if din.head_size != scorer.context_dim:
      raise ValueError('din.head_size %d must equal scorer.context_dim %d' %
                       (din.head_size, scorer.context_dim))
    if not float(cutoff) > 0:
      raise ValueError('cutoff must be > 0')
    if scorer.output_units != self._scorer_units():
      raise ValueError('the scorer has %d output units, the trainer scores %d task(s)' %
                       (scorer.output_units, self._scorer_units()))
    self.din = din
    self.scorer = scorer
    self.cutoff = float(cutoff)
    super().__init__(_DASALCJoint(din, scorer), loss, **kw)

  def _new_workspace(self, b, n):
    dev = self.device
    h = self.din.head_size
    self.emb = torch.empty(b * n, h, dtype=torch.float32, device=dev)
    self.d_emb = torch.empty(b * n, h, dtype=torch.float32, device=dev)
    self.din_ws = self.din._new_workspace(b, n)
    return self.scorer._new_workspace(b * n)

  def _prep_x(self, x):
    if x.shape[-1] != self.scorer.input_dim:
      raise ValueError('x has %d features, the scorer takes %d' %
                       (x.shape[-1], self.scorer.input_dim))
    x = x.float().contiguous()
    if getattr(self, '_xt', None) is None or self._xt.shape != x.shape:
      self._xt = torch.empty_like(x)
    _C.check(_C.lib.tfr_symmetric_log1p_clip(_C.ptr(x), x.numel(), self.cutoff,
                                             _C.ptr(self._xt), _C.stream()))
    return self._xt

  def _forward(self, x, y_true, m8, cfg, training):
    b, n, _ = x.shape
    din = self.din
    lm = m8
    if lm is None and y_true is not None:
      lm = (y_true >= 0).reshape(-1).to(torch.uint8).contiguous()
    self._lm = lm
    self._din_cfg = din._run_cfg(training=training)
    st = _C.stream()
    _C.check(_C.lib.tfr_din_fwd(_C.ptr(x), _C.ptr(lm), b, n, ctypes.byref(self._din_cfg),
                                _C.ptr(din.flat.data), _C.ptr(self.din_ws), _C.ptr(self.emb),
                                din.head_size, st))
    self._scorer_fwd(x, b * n, m8, cfg, st)

  def _scorer_units(self):
    return 1

  def _scorer_fwd(self, x, m, m8, cfg, st):
    sc = self.scorer
    _C.check(_C.lib.tfr_dasalc_fwd(_C.ptr(x), _C.ptr(self.emb), sc.context_dim, m, cfg,
                                   _C.ptr(sc.flat.data), _C.ptr(m8), _C.ptr(self.ws),
                                   _C.ptr(self.scores), sc._precision, st))

  def _scorer_bwd(self, x, m, m8, cfg, scorer_grads, st):
    sc = self.scorer
    _C.check(_C.lib.tfr_dasalc_bwd(_C.ptr(x), m, cfg, _C.ptr(sc.flat.data),
                                   _C.ptr(self.dscores), _C.ptr(m8), _C.ptr(self.ws),
                                   scorer_grads, _C.ptr(self.d_emb), sc.context_dim,
                                   sc._precision, st))

  def _backward(self, x, m8, cfg, grads):
    b, n, _ = x.shape
    din = self.din
    h = din.head_size
    st = _C.stream()
    scorer_grads = ctypes.c_void_p(grads.data_ptr() + 4 * self.tower.n_din)
    self._scorer_bwd(x, b * n, m8, cfg, scorer_grads, st)
    _C.check(_C.lib.tfr_din_bwd(_C.ptr(x), _C.ptr(self._lm), b, n, ctypes.byref(self._din_cfg),
                                _C.ptr(din.flat.data), _C.ptr(self.d_emb), h,
                                _C.ptr(self.din_ws), _C.ptr(grads), st))


class MultiTaskDINRankingTrainer(_TaskPlanes, DINRankingTrainer):
  """DINRankingTrainer with a score plane per task: the DocumentInteractionAttention
  embedding feeds one create_tower tower with `tower.output_units == len(losses)` output
  units, one per task.  One step is

      [X | E] with E = din((X, list_mask))    tfr_din_fwd
      score planes = tower([X | E])           tfr_mlp_fwd_tasks
      per-task losses                         one fused loss kernel per task
      tower gradients, d loss / d E           tfr_mlp_bwd_tasks (loss weights), tfr_mlp_input_grad
      DIN gradients                           tfr_din_bwd
      optimizer                               one launch over the shared flat buffer

  The tower constraints are DINRankingTrainer's; labels, masks, the returned loss and
  predict are MultiTaskRankingTrainer's."""

  def __init__(self, din, tower, losses, loss_weights=None, **kw):
    first = self._set_tasks(losses, loss_weights, tower.output_units)
    super().__init__(din, tower, first, **kw)
    self._set_task_weights()

  def _tower_fwd(self, m, m8, cfg, st):
    _C.check(_C.lib.tfr_mlp_fwd_tasks(_C.ptr(self.xe), m, cfg, _C.ptr(self.mlp.flat.data),
                                      _C.ptr(m8), _C.ptr(self.ws), _C.ptr(self.scores),
                                      self.mlp._precision, st))

  def _tower_bwd(self, m, m8, cfg, tower_grads, st):
    _C.check(_C.lib.tfr_mlp_bwd_tasks(_C.ptr(self.xe), m, cfg, _C.ptr(self.mlp.flat.data),
                                      _C.ptr(self.dscores), self._w_host, _C.ptr(m8),
                                      _C.ptr(self.ws), tower_grads, self.mlp._precision, st))


class MultiTaskDASALCRankingTrainer(_TaskPlanes, DASALCRankingTrainer):
  """DASALCRankingTrainer with a score plane per task: `scorer` is a DASALCScorer with
  `output_units == len(losses)`, run by tfr_dasalc_fwd_tasks / tfr_dasalc_bwd_tasks (K13
  with a [W, T] output layer; the loss weights are applied as the backward reads the dscore
  planes).  The log1p transform, circular padding, DIN and optimizer are
  DASALCRankingTrainer's; labels, masks, the returned loss and predict are
  MultiTaskRankingTrainer's."""

  def __init__(self, din, scorer, losses, loss_weights=None, cutoff=30.0, **kw):
    first = self._set_tasks(losses, loss_weights, scorer.output_units)
    super().__init__(din, scorer, first, cutoff=cutoff, **kw)
    self._set_task_weights()

  def _scorer_units(self):
    return len(self.tasks)

  def _scorer_fwd(self, x, m, m8, cfg, st):
    sc = self.scorer
    _C.check(_C.lib.tfr_dasalc_fwd_tasks(_C.ptr(x), _C.ptr(self.emb), sc.context_dim, m, cfg,
                                         _C.ptr(sc.flat.data), _C.ptr(m8), _C.ptr(self.ws),
                                         _C.ptr(self.scores), len(self.tasks), sc._precision,
                                         st))

  def _scorer_bwd(self, x, m, m8, cfg, scorer_grads, st):
    sc = self.scorer
    _C.check(_C.lib.tfr_dasalc_bwd_tasks(_C.ptr(x), m, cfg, _C.ptr(sc.flat.data),
                                         _C.ptr(self.dscores), self._w_host, _C.ptr(m8),
                                         _C.ptr(self.ws), scorer_grads, _C.ptr(self.d_emb),
                                         sc.context_dim, len(self.tasks), sc._precision, st))


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


class _EmbeddingScorer(object):
  """Embedding tables (+ one module between them and the tower: a
  DocumentInteractionAttention or a Bilinear) + tower as one scorer with ONE flat parameter
  buffer: the tables first (in the given order), then the middle module if there is one, then
  the tower (the modules' `flat` become views of it), so the step keeps one gradient
  all-reduce and one optimizer launch.  The middle block takes its size rounded up to a
  multiple of `middle_align` floats; the padding stays zero and is never read."""

  def __init__(self, tables, tower, middle=None, middle_align=1):
    parts = [t.flat.data for t in tables]
    n_mid = 0
    if middle is not None:
      n_mid = middle.flat.numel()
      pad = -n_mid % middle_align
      parts += [middle.flat.data, middle.flat.data.new_zeros(pad)]
    self.flat = torch.nn.Parameter(torch.cat(parts + [tower.flat.data]))
    self.table_offsets = []
    off = 0
    for t in tables:
      n = t.flat.numel()
      t.flat = torch.nn.Parameter(self.flat.data[off:off + n])
      self.table_offsets.append(off)
      off += n
    self.n_tables = off
    self.n_middle = n_mid
    if middle is not None:
      middle.flat = torch.nn.Parameter(self.flat.data[off:off + n_mid])
      off += n_mid + pad
    mods = list(tables) + ([middle] if middle is not None else [])
    self.tower_offset = off
    tower.flat = torch.nn.Parameter(self.flat.data[off:])
    self.bn_state = tower.bn_state
    self.dims = [list(t.dims) for t in mods] + [list(tower.dims)]
    self.use_batch_norm = tower.use_batch_norm
    self.input_batch_norm = tower.input_batch_norm
    self.input_dtype = torch.float32
    self._run_cfg = tower._run_cfg


class EmbeddingRankingTrainer(RankingTrainer):
  """Fused step for scorers over token (text) features, the model of the reference's ANTIQUE
  examples (examples/keras/antique_kpl_din.py:256-288, without the DIN; with it:
  DINEmbeddingRankingTrainer): every token feature
  is a bag of ids pooled through an embedding table (keras.layers.TokenEmbedding), and the
  pooled vectors become input columns of a create_tower tower:

      xe = [x | context features by sorted name | example features by sorted name]
           x: the dense columns ([B, N, D], D >= 0); every token feature takes E columns of
           its table; a context bag is repeated over its list, as FlattenList does
      scores = tower(xe)                              tfr_embedding_fwd, tfr_mlp_fwd
      loss, d loss / d scores                         fused loss kernel
      tower gradients, d loss / d pooled columns      tfr_mlp_bwd, tfr_mlp_input_grad
      table gradients                                 tfr_embedding_bwd (several features on
                                                      one table accumulate)
      optimizer                                       one launch over the shared flat buffer

  `embeddings`: {table name: TokenEmbedding}; `token_features`: {'context': {feature: table
  name}, 'example': {feature: table name}}.  Batches carry `tokens = {'context': {feature:
  int [B, T]}, 'example': {feature: int [B, N, T]}}` (data.elwc_batches with
  token_feature_spec).  The tower needs input_dim = D + E * (number of token features),
  precision tf32x3 or tf32, a hidden layer and no input BN.  With BN in the tower, example id
  rows are circularly padded like the dense rows (K9; needs T % 4 == 0), so a padded slot
  holds a copy of a valid item's bag.  Table rows no id hit get a zero gradient: with SGD and
  the Keras-form Adagrad that leaves them unchanged, as TF's sparse update does.  Ids outside
  [-1, V) are skipped and counted; `check_ids()` raises if any were seen.  fit / evaluate /
  checkpoints / data parallelism are the base class's."""

  def __init__(self, embeddings, token_features, tower, loss, **kw):
    tf = dict(token_features)
    extra = set(tf) - {'context', 'example'}
    if extra:
      raise ValueError("token_features takes the keys 'context' and 'example', got %s" %
                       sorted(extra))
    self.table_names = sorted(embeddings)
    tables = [embeddings[k] for k in self.table_names]
    feats = []                     # (kind, feature, table index), in tower column order
    for kind in ('context', 'example'):
      for name in sorted(tf.get(kind) or {}):
        key = tf[kind][name]
        if key not in embeddings:
          raise ValueError('token feature %r uses table %r, which is not in embeddings' %
                           (name, key))
        feats.append((kind, name, self.table_names.index(key)))
    if not feats:
      raise ValueError('token_features names no feature')
    width = sum(tables[i].embedding_dim for _, _, i in feats)
    if tower.input_dim < width:
      raise ValueError('the tower has input_dim %d, the token features alone take %d columns' %
                       (tower.input_dim, width))
    if tower.precision not in ('tf32x3', 'tf32') or tower.input_batch_norm or \
        not tower.hidden_layer_dims:
      raise ValueError('the tower must use precision tf32x3 or tf32, have a hidden layer and '
                       'no input BatchNormalization (its input gradient feeds the tables)')
    self.embeddings = tables
    self.features = feats
    self.dense_dim = tower.input_dim - width
    self.emb_width = width
    self.mlp = tower
    super().__init__(self._scorer(tables, tower), loss, **kw)
    self.bad_ids = torch.zeros(1, dtype=torch.int32, device=self.device)
    self._emb_ws = None
    self._padded = {}

  def _scorer(self, tables, tower):
    return _EmbeddingScorer(tables, tower)

  def check_ids(self):
    """Raises ValueError if a step has seen ids outside [-1, V) (host sync)."""
    n = int(self.bad_ids.item())
    if n:
      raise ValueError('%d token ids lay outside [-1, vocab_size) and were skipped' % n)

  def _new_workspace(self, b, n):
    self.xe = torch.empty(b * n, self.mlp.input_dim, dtype=torch.float32, device=self.device)
    self.d_emb = torch.empty(b * n, self.emb_width, dtype=torch.float32, device=self.device)
    return self.mlp._new_workspace(b * n)

  def _set_tokens(self, tokens, b, n):
    if tokens is None:
      raise ValueError('EmbeddingRankingTrainer needs the token features of the batch')
    ids = []
    for kind, name, _ in self.features:
      t = (tokens.get(kind) or {}).get(name)
      if t is None:
        raise ValueError('the batch has no %s token feature %r' % (kind, name))
      want = (b,) if kind == 'context' else (b, n)
      if tuple(t.shape[:-1]) != want or t.dim() != len(want) + 1:
        raise ValueError('%s token feature %r has shape %s, expected %s + (T,)' %
                         (kind, name, tuple(t.shape), want))
      ids.append(t.to(self.device, torch.int32, non_blocking=True).contiguous())
    self._ids = ids

  def train_step(self, x, y_true, tokens=None, sample_weight=None, mask=None):
    b, n, _ = x.shape
    self._set_tokens(tokens, b, n)
    return super().train_step(x, y_true, sample_weight=sample_weight, mask=mask)

  @torch.no_grad()
  def predict(self, x, mask=None, y_true=None, tokens=None):
    b, n, _ = x.shape
    self._set_tokens(tokens, b, n)
    return super().predict(x, mask=mask, y_true=y_true)

  def _circular_pad(self, x, valid):
    """K9 over the dense rows and over every example feature's id rows (same indices)."""
    t = self.tower
    self._step_ids = list(self._ids)
    if not (t.use_batch_norm or t.input_batch_norm) or valid is None:
      return x
    b, n, d = x.shape
    if d:
      x = super()._circular_pad(x, valid)
    v8 = valid.reshape(b, n).to(torch.uint8).contiguous()
    if getattr(self, '_pad_idx', None) is None or self._pad_idx.shape != (b, n):
      self._pad_idx = torch.empty(b, n, dtype=torch.int32, device=x.device)
    for k, (kind, name, _) in enumerate(self.features):
      if kind != 'example':
        continue
      ids = self._ids[k]
      if ids.shape[-1] % 4:
        raise ValueError('circular padding of token feature %r needs max_tokens to be a '
                         'multiple of 4, got %d' % (name, ids.shape[-1]))
      out = self._padded.get(name)
      if out is None or out.shape != ids.shape:
        out = self._padded[name] = torch.empty_like(ids)
      _C.check(_C.lib.tfr_circular_pad_gather(_C.ptr(ids), _C.ptr(v8), b, n,
                                              ids.shape[-1] * 4, _C.ptr(self._pad_idx),
                                              _C.ptr(out), _C.stream()))
      self._step_ids[k] = out
    return x

  def _bags(self, k, b, n):
    """(ids, R, T, rows_per_bag) of feature k."""
    ids = self._step_ids[k]
    t = ids.shape[-1]
    if self.features[k][0] == 'context':
      return ids, b, t, n
    return ids, b * n, t, 1

  def _pool(self, x, buf, ld):
    """buf [B * N, ld] = [x | every token feature's pooled bag, in feature order]."""
    b, n, d = x.shape
    if d != self.dense_dim:
      raise ValueError('x has %d dense features, the tower expects %d' % (d, self.dense_dim))
    st = _C.stream()
    if d:
      buf.view(b, n, ld)[..., :d].copy_(x)
    col = d
    for k, (_, _, ti) in enumerate(self.features):
      emb = self.embeddings[ti]
      ids, r, t, rpb = self._bags(k, b, n)
      _C.check(_C.lib.tfr_embedding_fwd(_C.ptr(ids), r, t, _C.ptr(emb.flat.data),
                                        emb.vocab_size, emb.embedding_dim, emb._combiner, rpb,
                                        ctypes.c_void_p(buf.data_ptr() + 4 * col), ld,
                                        _C.ptr(self.bad_ids), st))
      col += emb.embedding_dim

  def _forward(self, x, y_true, m8, cfg, training):
    b, n, _ = x.shape
    self._pool(x, self.xe, self.mlp.input_dim)
    _C.check(_C.lib.tfr_mlp_fwd(_C.ptr(self.xe), b * n, cfg, _C.ptr(self.mlp.flat.data),
                                _C.ptr(m8), _C.ptr(self.ws), _C.ptr(self.scores),
                                self.mlp._precision, _C.stream()))

  def _backward(self, x, m8, cfg, grads):
    b, n, d = x.shape
    mlp, sc = self.mlp, self.tower
    st = _C.stream()
    _C.check(_C.lib.tfr_mlp_bwd(_C.ptr(self.xe), b * n, cfg, _C.ptr(mlp.flat.data),
                                _C.ptr(self.dscores), _C.ptr(m8), _C.ptr(self.ws),
                                ctypes.c_void_p(grads.data_ptr() + 4 * sc.tower_offset),
                                mlp._precision, st))
    _C.check(_C.lib.tfr_mlp_input_grad(cfg, b * n, _C.ptr(mlp.flat.data), _C.ptr(self.ws), d,
                                       self.emb_width, _C.ptr(self.d_emb), self.emb_width,
                                       mlp._precision, st))
    cols, col = [], 0
    for _, _, ti in self.features:
      cols.append(col)
      col += self.embeddings[ti].embedding_dim
    self._tables_bwd(b, n, grads, self.d_emb, self.emb_width, cols)

  def _tables_bwd(self, b, n, grads, d_pooled, ld, cols):
    """Table gradients: feature k's pooled gradient is columns cols[k] .. of d_pooled (row
    pitch ld)."""
    sc = self.tower
    st = _C.stream()
    need = 0
    for k, (_, _, ti) in enumerate(self.features):
      emb = self.embeddings[ti]
      _, r, t, _ = self._bags(k, b, n)
      need = max(need, _C.lib.tfr_embedding_workspace_bytes(r, t, emb.vocab_size,
                                                            emb.embedding_dim))
    if self._emb_ws is None or self._emb_ws.numel() < need:
      self._emb_ws = torch.empty(need, dtype=torch.uint8, device=self.device)
    written = set()
    for k, (_, _, ti) in enumerate(self.features):
      emb = self.embeddings[ti]
      ids, r, t, rpb = self._bags(k, b, n)
      _C.check(_C.lib.tfr_embedding_bwd(
          _C.ptr(ids), r, t, ctypes.c_void_p(d_pooled.data_ptr() + 4 * cols[k]), ld,
          rpb, emb.vocab_size, emb.embedding_dim, emb._combiner, int(ti in written),
          _C.ptr(self._emb_ws), ctypes.c_void_p(grads.data_ptr() + 4 * sc.table_offsets[ti]),
          None, st))
      written.add(ti)
    for ti, emb in enumerate(self.embeddings):
      if ti not in written:     # a table no feature reads: zero gradient
        off = sc.table_offsets[ti]
        grads[off:off + emb.flat.numel()].zero_()


class DINEmbeddingRankingTrainer(EmbeddingRankingTrainer):
  """EmbeddingRankingTrainer with a DocumentInteractionAttention between the pooled token
  features and the tower: the reference's ANTIQUE example as it runs by default
  (examples/keras/antique_kpl_din.py, use_document_interaction=True).

      xd = [x | context features by sorted name | example features by sorted name]
           the DIN's input, ConcatFeatures' order (D_din = D + E * F columns)
      xe = the same blocks with the DIN's h columns inserted where `din_feature` sorts among
           the example features (the reference's sorted-name rule), e.g. for ANTIQUE
           [query_tokens | document_interaction_embedding | document_tokens]
      xd, xe                                         tfr_embedding_fwd, strided copies
      E = din((xd, list_mask)) into xe's DIN block   tfr_din_fwd
      scores = tower(xe)                             tfr_mlp_fwd
      loss, d loss / d scores                        fused loss kernel
      tower gradients, d loss / d xe[:, D:]          tfr_mlp_bwd, tfr_mlp_input_grad
      DIN gradients                                  tfr_din_bwd on the DIN block of d xe
      d loss / d xd[:, D:] added to d xe's token     tfr_din_input_grad (accumulate), one
      columns                                        window each side of the DIN block
      table gradients                                tfr_embedding_bwd
      optimizer                                      one launch over the shared flat buffer

  No gradient is formed for the dense x.  The flat buffer holds the tables, then the DIN, then
  the tower.  `tower` needs input_dim = D_din + head_size with D_din a multiple of 4, and the
  limits of EmbeddingRankingTrainer.  The DIN is built for D_din on first use if it has not
  been.  The list mask, the DIN's training flag and its seed follow DINRankingTrainer.  With
  BN in the tower, the dense rows and the example id rows are circularly padded before the
  DIN, as DINRankingTrainer does (the reference pads after it); with DIN dropout the padded
  rows then draw their own dropout masks instead of repeating their source item's."""

  def __init__(self, embeddings, token_features, din, tower, loss,
               din_feature='document_interaction_embedding', **kw):
    h = din.head_size
    names = {f for kind in dict(token_features).values() for f in (kind or {})}
    if din_feature in names:
      raise ValueError('din_feature %r is also the name of a token feature' % din_feature)
    d_din = tower.input_dim - h
    if d_din <= 0 or d_din % 4:
      raise ValueError('the DIN input (tower input_dim %d - head_size %d = %d columns) must be '
                       'a positive multiple of 4' % (tower.input_dim, h, d_din))
    if not din.built:
      din.build(d_din)
    if din.input_dim != d_din:
      raise ValueError('the tower needs input_dim = %d (DIN input) + %d (head_size), got %d' %
                       (din.input_dim, h, tower.input_dim))
    self.din = din
    self.din_feature = din_feature
    super().__init__(embeddings, token_features, tower, loss, **kw)
    self.dense_dim = d_din - self.emb_width
    if self.dense_dim < 0:
      raise ValueError('the token features take %d columns, the DIN input has %d' %
                       (self.emb_width, d_din))
    # DIN input column where the DIN block goes in the tower input
    self.split = self.dense_dim
    for kind, name, ti in self.features:
      if kind == 'context' or name < din_feature:
        self.split += self.embeddings[ti].embedding_dim

  def _scorer(self, tables, tower):
    return _EmbeddingScorer(tables, tower, middle=self.din)

  def _new_workspace(self, b, n):
    m, dev = b * n, self.device
    self.xd = torch.empty(m, self.din.input_dim, dtype=torch.float32, device=dev)
    self.xe = torch.empty(m, self.mlp.input_dim, dtype=torch.float32, device=dev)
    self.d_xe = torch.empty(m, self.mlp.input_dim - self.dense_dim, dtype=torch.float32,
                            device=dev)
    self.din_ws = self.din._new_workspace(b, n)
    return self.mlp._new_workspace(m)

  def _forward(self, x, y_true, m8, cfg, training):
    b, n, _ = x.shape
    din, s, h = self.din, self.split, self.din.head_size
    width = self.mlp.input_dim
    self._pool(x, self.xd, din.input_dim)
    self.xe[:, :s].copy_(self.xd[:, :s])
    self.xe[:, s + h:].copy_(self.xd[:, s:])
    lm = m8
    if lm is None and y_true is not None:
      lm = (y_true >= 0).reshape(-1).to(torch.uint8).contiguous()
    self._lm = lm
    self._din_cfg = din._run_cfg(training=training)
    st = _C.stream()
    _C.check(_C.lib.tfr_din_fwd(_C.ptr(self.xd), _C.ptr(lm), b, n, ctypes.byref(self._din_cfg),
                                _C.ptr(din.flat.data), _C.ptr(self.din_ws),
                                ctypes.c_void_p(self.xe.data_ptr() + 4 * s), width, st))
    _C.check(_C.lib.tfr_mlp_fwd(_C.ptr(self.xe), b * n, cfg, _C.ptr(self.mlp.flat.data),
                                _C.ptr(m8), _C.ptr(self.ws), _C.ptr(self.scores),
                                self.mlp._precision, st))

  def _backward(self, x, m8, cfg, grads):
    b, n, d = x.shape
    din, mlp, sc = self.din, self.mlp, self.tower
    s, h, d_din = self.split, din.head_size, din.input_dim
    ld = mlp.input_dim - d          # d_xe: the tower input's columns [D, width)
    st = _C.stream()
    _C.check(_C.lib.tfr_mlp_bwd(_C.ptr(self.xe), b * n, cfg, _C.ptr(mlp.flat.data),
                                _C.ptr(self.dscores), _C.ptr(m8), _C.ptr(self.ws),
                                ctypes.c_void_p(grads.data_ptr() + 4 * sc.tower_offset),
                                mlp._precision, st))
    _C.check(_C.lib.tfr_mlp_input_grad(cfg, b * n, _C.ptr(mlp.flat.data), _C.ptr(self.ws), d,
                                       ld, _C.ptr(self.d_xe), ld, mlp._precision, st))
    cfg_din = ctypes.byref(self._din_cfg)
    _C.check(_C.lib.tfr_din_bwd(_C.ptr(self.xd), _C.ptr(self._lm), b, n, cfg_din,
                                _C.ptr(din.flat.data),
                                ctypes.c_void_p(self.d_xe.data_ptr() + 4 * (s - d)), ld,
                                _C.ptr(self.din_ws),
                                ctypes.c_void_p(grads.data_ptr() + 4 * sc.n_tables), st))
    # the DIN input's token columns before and after the DIN block, added onto d_xe's
    for c0, c1, dst in ((d, s, 0), (s, d_din, s + h - d)):
      if c1 > c0:
        _C.check(_C.lib.tfr_din_input_grad(cfg_din, b, n, _C.ptr(din.flat.data),
                                           _C.ptr(self.din_ws), c0, c1 - c0,
                                           ctypes.c_void_p(self.d_xe.data_ptr() + 4 * dst), ld,
                                           1, st))
    cols, col = [], d
    for _, _, ti in self.features:
      cols.append(col - d if col < s else col - d + h)
      col += self.embeddings[ti].embedding_dim
    self._tables_bwd(b, n, grads, self.d_xe, ld, cols)


class ClickEMRankingTrainer(RankingTrainer):
  """Learns a relevance scorer from position-biased clicks, jointly with a per-position
  examination propensity: the examination x relevance click model of Wang et al. 2018
  (losses_impl.py:1324-1422) trained online, as the reference's ClickEMLoss does with a
  two-tower model.

      exam = table[position]                 tfr_embedding_fwd (one id per item, SUM)
      rel  = tower(x)                        tfr_mlp_fwd
      loss, d exam, d rel                    K3d ClickEM on the two [B, N] planes
      tower gradients                        tfr_mlp_bwd
      table gradient                         tfr_embedding_bwd (deterministic)
      optimizer                              one launch over the shared flat buffer

  `tower`: a create_tower tower with output_units 1 (precision fp32, tf32x3 or tf32; BN is
  allowed, with circular padding as in the base class).  `loss`: a keras.losses.ClickEMLoss.
  The position table is a keras.layers.TokenEmbedding(num_positions, 1, combiner='sum'); it
  and the tower share one flat parameter buffer (_EmbeddingScorer), so checkpoints, the
  optimizer and the data-parallel reducer cover it.  Its row count is rounded up to a
  multiple of 64 so that the tower's parameters, which follow it, keep the 256-byte
  alignment of a tower's own allocation; the extra rows are never read and keep their
  initial values.  Labels are clicks (>= 1 clicked, < 0 padding).  `predict` returns the
  relevance scores only, so pipeline.fit / evaluate work unchanged."""

  _ROW_ALIGN = 64

  def __init__(self, tower, loss, num_positions, seed=None, **kw):
    from ranking_b200.keras import layers as keras_layers
    from ranking_b200.keras import losses as keras_losses
    if not isinstance(loss, keras_losses.ClickEMLoss):
      raise ValueError('ClickEMRankingTrainer needs a keras.losses.ClickEMLoss')
    if tower.precision not in ('fp32', 'tf32x3', 'tf32'):
      raise ValueError('the click EM tower must use precision fp32, tf32x3 or tf32')
    if tower.output_units != 1:
      raise ValueError('the relevance tower needs output_units = 1')
    num_positions = int(num_positions)
    if num_positions < 1:
      raise ValueError('num_positions must be >= 1')
    rows = -(-num_positions // self._ROW_ALIGN) * self._ROW_ALIGN
    self.num_positions = num_positions
    self.positions_table = keras_layers.TokenEmbedding(rows, 1, combiner='sum', seed=seed,
                                                       device=tower.flat.device)
    self.mlp = tower
    super().__init__(_EmbeddingScorer([self.positions_table], tower), loss, **kw)
    self._pos = None
    self._emb_ws = None

  def _new_workspace(self, b, n):
    dev = self.device
    self.exam = torch.empty(b, n, dtype=torch.float32, device=dev)
    self.dexam = torch.empty(b, n, dtype=torch.float32, device=dev)
    self._default_pos = torch.arange(n, device=dev).clamp(max=self.num_positions - 1).to(
        torch.int32).expand(b, n).contiguous()
    self._emb_ws = torch.empty(
        _C.lib.tfr_embedding_workspace_bytes(b * n, 1, self.positions_table.vocab_size, 1),
        dtype=torch.uint8, device=dev)
    return self.mlp._new_workspace(b * n)

  def _set_positions(self, positions, b, n):
    if positions is None:
      self._pos = self._default_pos
      return
    if tuple(positions.shape) != (b, n):
      raise ValueError('positions must have shape [batch_size, list_size] = %s, got %s' %
                       ((b, n), tuple(positions.shape)))
    pos = positions.to(self.device, torch.int32).contiguous()
    if bool(((pos < 0) | (pos >= self.num_positions)).any()):
      raise ValueError('positions must lie in [0, %d)' % self.num_positions)
    self._pos = pos

  def examination_propensity(self):
    """sigmoid(table) [num_positions]: the learned P(examination | position)."""
    return torch.sigmoid(self.positions_table.flat.detach()[:self.num_positions])

  def _forward(self, x, y_true, m8, cfg, training):
    b, n, _ = x.shape
    mlp = self.mlp
    _C.check(_C.lib.tfr_mlp_fwd(_C.ptr(x), b * n, cfg, _C.ptr(mlp.flat.data), _C.ptr(m8),
                                _C.ptr(self.ws), _C.ptr(self.scores), mlp._precision,
                                _C.stream()))

  def _backward(self, x, m8, cfg, grads):
    b, n, _ = x.shape
    mlp, sc, emb = self.mlp, self.tower, self.positions_table
    st = _C.stream()
    _C.check(_C.lib.tfr_mlp_bwd(_C.ptr(x), b * n, cfg, _C.ptr(mlp.flat.data),
                                _C.ptr(self.dscores), _C.ptr(m8), _C.ptr(self.ws),
                                ctypes.c_void_p(grads.data_ptr() + 4 * sc.n_tables),
                                mlp._precision, st))
    _C.check(_C.lib.tfr_embedding_bwd(_C.ptr(self._pos), b * n, 1, _C.ptr(self.dexam), 1, 1,
                                      emb.vocab_size, 1, emb._combiner, 0, _C.ptr(self._emb_ws),
                                      _C.ptr(grads), None, st))

  def train_step(self, x, clicks, positions=None, sample_weight=None, mask=None):
    """x [B, N, D] (device, fp32), clicks [B, N] (>= 1 clicked, < 0 padding), positions
    ([B, N] int in [0, num_positions), optional: by default an item's position is its row
    in the list, clipped to num_positions - 1, i.e. the logged display order).  Returns the
    scalar loss as a 0-d device tensor."""
    b, n, _ = x.shape
    self._ensure(b, n)
    self._set_positions(positions, b, n)
    x = self._prep_x(x)
    cfg = ctypes.byref(self.tower._run_cfg(training=True))
    m8 = None if mask is None else mask.reshape(-1).to(torch.uint8).contiguous()
    grads = self.reducer.grads() if self.reducer is not None else self.grads
    self.grads = grads
    x = self._circular_pad(x, mask if mask is not None else (clicks >= 0))
    emb = self.positions_table
    st = _C.stream()
    _C.check(_C.lib.tfr_embedding_fwd(_C.ptr(self._pos), b * n, 1, _C.ptr(emb.flat.data),
                                      emb.vocab_size, 1, emb._combiner, 1, _C.ptr(self.exam), 1,
                                      None, st))
    self._forward(x, clicks, m8, cfg, True)
    self.loss.fused_fwd_bwd(clicks, self.exam, self.scores, sample_weight, self.dexam,
                            self.dscores, self.per_list, self.total2)
    self._backward(x, m8, cfg, grads)
    self._apply(grads)
    return self.total2[0]


class BilinearClickRankingTrainer(RankingTrainer):
  """Learns a relevance tower from position-biased clicks with the two-tower model of Yan et
  al., "Revisiting two tower models for unbiased learning to rank": a relevance tower and a
  position embedding interact through a keras.layers.Bilinear into the click logit, so the
  bias model is not restricted to click = examination x relevance.

      r = tower(x)                   [B * N, E]   tfr_mlp_fwd (tower.output_units = E)
      p = table[position]            [B * N, E]   tfr_embedding_fwd (one id per item, SUM)
      c = bilinear((r, p))           [B, N]       tfr_bilinear_fwd (K14), ln(1e-10) where
                                                  `mask` is 0
      loss, d c                                   the loss's fused kernel, clicks as labels
      d r, d p, bilinear gradients                tfr_bilinear_bwd
      tower gradients                             tfr_mlp_bwd with d scores = d r
      table gradient                              tfr_embedding_bwd (deterministic)
      optimizer                                   one launch over the shared flat buffer

  `tower`: a create_tower tower with output_units = bilinear.embedding_dim (the tower's output
  layer takes at most 8 units, so E <= 8); precision fp32, tf32x3 or tf32; BN is allowed, with
  circular padding as in the base class.  `bilinear`: a keras.layers.Bilinear(E, 1).  `loss`:
  a loss whose fused kernel takes [B, N] logits, e.g. keras.losses.SigmoidCrossEntropyLoss
  (not ClickEMLoss or MixtureEMLoss).  The position table is a
  keras.layers.TokenEmbedding(num_positions, E, combiner='sum') seeded with `seed`.  Table,
  bilinear and tower share one flat parameter buffer (_EmbeddingScorer), so checkpoints, the
  optimizer and the data-parallel reducer cover them.  The table's rows and the bilinear block
  are padded to multiples of 64 floats so that the tower's parameters keep the 256-byte
  alignment of a tower's own allocation; the padding is never read and keeps its value.
  Labels are clicks (>= 1 clicked, < 0 padding).  `predict` places every item at
  `serving_position` unless `positions` is given, so its scores rank by relevance and
  pipeline.fit / evaluate work unchanged."""

  _ALIGN = 64

  def __init__(self, tower, bilinear, loss, num_positions, serving_position=0, seed=None, **kw):
    from ranking_b200.keras import layers as keras_layers
    from ranking_b200.keras import losses as keras_losses
    if isinstance(loss, (keras_losses.ClickEMLoss, keras_losses.MixtureEMLoss)):
      raise ValueError('BilinearClickRankingTrainer needs a loss over [B, N] click logits '
                       '(e.g. SigmoidCrossEntropyLoss), not %s' % type(loss).__name__)
    if tower.precision not in ('fp32', 'tf32x3', 'tf32'):
      raise ValueError('the relevance tower must use precision fp32, tf32x3 or tf32')
    if tower.output_units != bilinear.embedding_dim:
      raise ValueError('the relevance tower has output_units %d, the bilinear layer takes '
                       'embedding_dim %d' % (tower.output_units, bilinear.embedding_dim))
    if bilinear.output_dim != 1:
      raise ValueError('the bilinear layer must have output_dim 1 (one click logit), got %d' %
                       bilinear.output_dim)
    if bilinear.flat.device != tower.flat.device:
      raise ValueError('the bilinear layer and the tower must live on the same device')
    num_positions = int(num_positions)
    if num_positions < 1:
      raise ValueError('num_positions must be >= 1')
    serving_position = int(serving_position)
    if not 0 <= serving_position < num_positions:
      raise ValueError('serving_position must lie in [0, %d)' % num_positions)
    e = bilinear.embedding_dim
    rows = num_positions
    while rows * e % self._ALIGN:
      rows += 1
    self.num_positions = num_positions
    self.serving_position = serving_position
    self.positions_table = keras_layers.TokenEmbedding(rows, e, combiner='sum', seed=seed,
                                                       device=tower.flat.device)
    self.bilinear = bilinear
    self.mlp = tower
    super().__init__(_EmbeddingScorer([self.positions_table], tower, middle=bilinear,
                                      middle_align=self._ALIGN), loss, **kw)
    self._pos = None

  def _new_workspace(self, b, n):
    dev, m, e = self.device, b * n, self.bilinear.embedding_dim
    self.rel = torch.empty(m, e, dtype=torch.float32, device=dev)
    self.pemb = torch.empty(m, e, dtype=torch.float32, device=dev)
    self.drel = torch.empty(m, e, dtype=torch.float32, device=dev)
    self.dpemb = torch.empty(m, e, dtype=torch.float32, device=dev)
    self._default_pos = torch.arange(n, device=dev).clamp(max=self.num_positions - 1).to(
        torch.int32).expand(b, n).contiguous()
    self._serving_pos = torch.full((b, n), self.serving_position, dtype=torch.int32, device=dev)
    emb = self.positions_table
    self._emb_ws = torch.empty(_C.lib.tfr_embedding_workspace_bytes(m, 1, emb.vocab_size, e),
                               dtype=torch.uint8, device=dev)
    self._bil_ws = torch.empty(_C.lib.tfr_bilinear_workspace_bytes(m, e, 1), dtype=torch.uint8,
                               device=dev)
    return self.mlp._new_workspace(m)

  def _set_positions(self, positions, b, n, default):
    if positions is None:
      self._pos = default
      return
    if tuple(positions.shape) != (b, n):
      raise ValueError('positions must have shape [batch_size, list_size] = %s, got %s' %
                       ((b, n), tuple(positions.shape)))
    pos = positions.to(self.device, torch.int32).contiguous()
    if bool(((pos < 0) | (pos >= self.num_positions)).any()):
      raise ValueError('positions must lie in [0, %d)' % self.num_positions)
    self._pos = pos

  def _forward(self, x, y_true, m8, cfg, training):
    b, n, _ = x.shape
    m, mlp, emb, bil = b * n, self.mlp, self.positions_table, self.bilinear
    e = bil.embedding_dim
    st = _C.stream()
    _C.check(_C.lib.tfr_mlp_fwd(_C.ptr(x), m, cfg, _C.ptr(mlp.flat.data), _C.ptr(m8),
                                _C.ptr(self.ws), _C.ptr(self.rel), mlp._precision, st))
    _C.check(_C.lib.tfr_embedding_fwd(_C.ptr(self._pos), m, 1, _C.ptr(emb.flat.data),
                                      emb.vocab_size, e, emb._combiner, 1, _C.ptr(self.pemb), e,
                                      None, st))
    _C.check(_C.lib.tfr_bilinear_fwd(_C.ptr(self.rel), _C.ptr(self.pemb), m, e, 1,
                                      _C.ptr(bil.flat.data), _C.ptr(m8), _C.ptr(self.scores), st))

  def _backward(self, x, m8, cfg, grads):
    b, n, _ = x.shape
    m, mlp, emb, bil, sc = b * n, self.mlp, self.positions_table, self.bilinear, self.tower
    e = bil.embedding_dim
    st = _C.stream()
    _C.check(_C.lib.tfr_bilinear_bwd(_C.ptr(self.rel), _C.ptr(self.pemb), m, e, 1,
                                      _C.ptr(bil.flat.data), _C.ptr(m8), _C.ptr(self.dscores),
                                      _C.ptr(self.drel), _C.ptr(self.dpemb),
                                      ctypes.c_void_p(grads.data_ptr() + 4 * sc.n_tables),
                                      _C.ptr(self._bil_ws), st))
    _C.check(_C.lib.tfr_mlp_bwd(_C.ptr(x), m, cfg, _C.ptr(mlp.flat.data), _C.ptr(self.drel),
                                _C.ptr(m8), _C.ptr(self.ws),
                                ctypes.c_void_p(grads.data_ptr() + 4 * sc.tower_offset),
                                mlp._precision, st))
    _C.check(_C.lib.tfr_embedding_bwd(_C.ptr(self._pos), m, 1, _C.ptr(self.dpemb), e, 1,
                                      emb.vocab_size, e, emb._combiner, 0, _C.ptr(self._emb_ws),
                                      _C.ptr(grads), None, st))

  def train_step(self, x, clicks, positions=None, sample_weight=None, mask=None):
    """x [B, N, D] (device, fp32), clicks [B, N] (>= 1 clicked, < 0 padding), positions
    ([B, N] int in [0, num_positions), optional: by default an item's position is its row
    in the list, clipped to num_positions - 1, i.e. the logged display order).  Returns the
    scalar loss as a 0-d device tensor."""
    b, n, _ = x.shape
    self._ensure(b, n)
    self._set_positions(positions, b, n, self._default_pos)
    return super().train_step(x, clicks, sample_weight=sample_weight, mask=mask)

  @torch.no_grad()
  def predict(self, x, mask=None, y_true=None, positions=None):
    """Click logits [B, N] with every item at `serving_position` (or at `positions`)."""
    b, n, _ = x.shape
    self._ensure(b, n)
    self._set_positions(positions, b, n, self._serving_pos)
    return super().predict(x, mask=mask, y_true=y_true)
