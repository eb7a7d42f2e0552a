"""A small fit / evaluate loop around `RankingTrainer` with checkpoint + resume: the
shape of the reference's `ModelFitPipeline.train_and_validate`
(keras/pipeline.py:561-650) for the fused CUDA step.
"""
import os

import torch
import torch.distributed as dist

from ranking_b200 import dp
from ranking_b200.keras import metrics as keras_metrics


def save_checkpoint(trainer, path, step):
  """Parameters, optimizer accumulator, BN moving statistics and the step counter (and
  AdamW's update count, and a TFR-BERT trainer's loss scale and good-step count).
  Data parallel: rank 0 alone writes (replicas hold identical parameters; BN statistics
  are per replica and rank 0's are the ones kept), every rank waits for the file."""
  tower = trainer.tower
  if dp.rank(trainer.group) == 0:
    tmp = '%s.tmp.%d' % (path, os.getpid())
    state = {'step': int(step), 'flat': tower.flat.detach().cpu(),
             'accum': trainer.accum.cpu(), 'bn_state': tower.bn_state.cpu(),
             'dims': list(tower.dims)}
    if hasattr(trainer, 'adam_step'):   # AdamW's update count t
      state['adam_step'] = int(trainer.adam_step)
    if hasattr(trainer, 'loss_scale'):   # TFR-BERT's fp16 loss scale and good-step count
      state['loss_scale'] = trainer.loss_scale.cpu()
      state['good_steps'] = trainer.good_steps.cpu()
    torch.save(state, tmp)
    os.replace(tmp, path)      # atomic: a crash never leaves a torn file
  if dp.world_size(trainer.group) > 1:
    dist.barrier(group=trainer.group)


def load_checkpoint(trainer, path):
  ckpt = torch.load(path, map_location='cpu', weights_only=True)
  tower = trainer.tower
  if list(ckpt['dims']) != list(tower.dims):
    raise ValueError('checkpoint was written for dims %s, tower has %s' %
                     (ckpt['dims'], tower.dims))
  with torch.no_grad():
    tower.flat.copy_(ckpt['flat'])
    trainer.accum.copy_(ckpt['accum'])
    if tower.bn_state.numel():
      tower.bn_state.copy_(ckpt['bn_state'])
  if 'adam_step' in ckpt:
    trainer.adam_step = int(ckpt['adam_step'])
  if hasattr(trainer, 'loss_scale'):   # a checkpoint without them: the initial scale, count 0
    if 'loss_scale' in ckpt:
      with torch.no_grad():
        trainer.loss_scale.copy_(ckpt['loss_scale'])
        trainer.good_steps.copy_(ckpt['good_steps'])
    else:
      trainer.reset_loss_scale()
  return int(ckpt['step'])


def _to_device(features, dev):
  return {k: v.to(dev, non_blocking=True) for k, v in features.items()}


def evaluate(trainer, batches, metric_group=None):
  """Scores every batch with the tower and accumulates `MetricGroup.default()`
  (all of `default_keras_metrics()`, one launch per batch)."""
  group = metric_group or keras_metrics.MetricGroup.default()
  group.reset_state()
  dev = trainer.device
  for batch in batches:
    y = batch[1].to(dev, non_blocking=True)
    if isinstance(batch[0], dict):   # ({input_word_ids, ...}, y): TFRBertRankingTrainer
      scores = trainer.predict(**_to_device(batch[0], dev), mask=(y >= 0))
      group.update_state(y, scores)
      continue
    x = batch[0].to(dev, non_blocking=True)
    if len(batch) > 2:     # (x, y, tokens): token features for EmbeddingRankingTrainer
      scores = trainer.predict(x, mask=(y >= 0), tokens=batch[2])
    else:
      scores = trainer.predict(x, mask=(y >= 0))
    group.update_state(y, scores)
  group.all_reduce(trainer.group)
  return group.result()


def fit(trainer, train_batches, num_steps, checkpoint_dir=None,
        steps_per_checkpoint=1000, eval_batches_fn=None, log_fn=print):
  """Runs `num_steps` fused training steps over `train_batches` (an iterator of host
  or device (x, y) pairs, or (x, y, tokens) triples whose token features go to an
  `EmbeddingRankingTrainer`).  With `checkpoint_dir`, resumes from `ckpt.pt` if it exists
  and rewrites it every `steps_per_checkpoint` steps and at the end."""
  step = 0
  ckpt = None
  if checkpoint_dir:
    os.makedirs(checkpoint_dir, exist_ok=True)
    ckpt = os.path.join(checkpoint_dir, 'ckpt.pt')
    if os.path.exists(ckpt):
      step = load_checkpoint(trainer, ckpt)
      log_fn('resumed from %s at step %d' % (ckpt, step))
  dev = trainer.device
  last = None
  for batch in train_batches:
    if step >= num_steps:
      break
    y = batch[1].to(dev, non_blocking=True)
    if isinstance(batch[0], dict):   # id tensors of TFRBertRankingTrainer
      last = trainer.train_step(**_to_device(batch[0], dev), y_true=y)
    elif len(batch) > 2:
      last = trainer.train_step(batch[0].to(dev, non_blocking=True), y, tokens=batch[2])
    else:
      last = trainer.train_step(batch[0].to(dev, non_blocking=True), y)
    step += 1
    if ckpt and step % steps_per_checkpoint == 0:
      save_checkpoint(trainer, ckpt, step)
      msg = 'step %d loss %.6f' % (step, float(last))
      if eval_batches_fn is not None:
        msg += ' ' + str(evaluate(trainer, eval_batches_fn()))
      log_fn(msg)
  if ckpt:
    save_checkpoint(trainer, ckpt, step)
  return step, (None if last is None else float(last))


# ----------------------------------------------------------------------------------------
# keras/pipeline.py:262-334, 372-650: PipelineHparams + ModelFitPipeline.train_and_validate
# ----------------------------------------------------------------------------------------
import dataclasses
from typing import Dict, Optional, Union


@dataclasses.dataclass
class PipelineHparams:
  """The reference's `PipelineHparams` (keras/pipeline.py:262-334), same field names.  Fields
  that select TF machinery (`strategy`, `cluster_resolver`, `variable_partitioner`, `tpu`,
  `steps_per_execution`) are accepted and ignored: data parallelism here is one process per
  GPU under torchrun (DESIGN.md §5).  `optimizer` must be one the fused step implements
  ('adagrad', 'sgd'); the reference's default 'adam' raises."""
  model_dir: str
  num_epochs: int
  steps_per_epoch: int
  validation_steps: int
  learning_rate: float
  loss: Union[str, Dict[str, str]]
  loss_reduction: str = 'auto'
  optimizer: str = 'adagrad'
  loss_weights: Optional[Union[float, Dict[str, float]]] = None
  steps_per_execution: int = 10
  automatic_reduce_lr: bool = False
  early_stopping_patience: int = 0
  early_stopping_min_delta: float = 0.0
  use_weighted_metrics: bool = False
  export_best_model: bool = False
  best_exporter_metric_higher_better: bool = False
  best_exporter_metric: str = 'loss'
  strategy: Optional[str] = None
  cluster_resolver: Optional[object] = None
  variable_partitioner: Optional[object] = None
  tpu: Optional[str] = ''

  def validate(self):
    if not isinstance(self.loss, str):
      raise ValueError('multi-task loss maps are not supported by the fused step')
    self.validate_loop()
    if self.loss_weights is not None and not isinstance(self.loss_weights, (int, float)):
      raise ValueError('loss_weights must be None or a scalar')

  def validate_loop(self):
    """The checks that do not depend on the loss: optimizer and loop lengths."""
    if self.optimizer not in ('adagrad', 'sgd'):
      raise ValueError("optimizer must be 'adagrad' or 'sgd', got %r" % (self.optimizer,))
    if self.num_epochs < 1 or self.steps_per_epoch < 1 or self.validation_steps < 0:
      raise ValueError('num_epochs / steps_per_epoch must be >= 1, validation_steps >= 0')


class ModelFitPipeline(object):
  """`ModelFitPipeline.train_and_validate` (keras/pipeline.py:561-632) over the fused CUDA
  step: `num_epochs` x (`steps_per_epoch` training steps, `validation_steps` evaluation
  batches), checkpoint + resume in `model_dir`, optional early stopping
  (`early_stopping_patience` / `_min_delta` on `best_exporter_metric`, keras/pipeline.py:
  474-496), ReduceLROnPlateau (`automatic_reduce_lr`: factor 0.1, patience = a third of the
  epochs, as build_callbacks does) and the best checkpoint (`export_best_model`).

  tower_fn()            -> ranking_b200.keras.layers.Tower (the model_builder's role)
  train_batches_fn()    -> iterable of (x, y) batches, restarted when exhausted
  valid_batches_fn()    -> the same for validation (may be None)
  """

  def __init__(self, tower_fn, train_batches_fn, valid_batches_fn, hparams,
               process_group=None, log_fn=print):
    self._validate_hparams(hparams)
    self._hparams = hparams
    self._tower_fn = tower_fn
    self._train_fn = train_batches_fn
    self._valid_fn = valid_batches_fn
    self._group = process_group
    self._log = log_fn
    self.history = []

  @staticmethod
  def _validate_hparams(hparams):
    hparams.validate()

  def build_loss(self):
    from ranking_b200.keras import losses as keras_losses
    kw = {}
    if self._hparams.loss_reduction not in (None, 'auto'):
      kw['reduction'] = self._hparams.loss_reduction
    return keras_losses.get(self._hparams.loss, **kw)

  def build_metrics(self):
    return keras_metrics.MetricGroup.default()

  def _monitor(self, logs):
    key = self._hparams.best_exporter_metric
    if key not in logs:
      raise ValueError('best_exporter_metric %r is not among %s' % (key, sorted(logs)))
    return logs[key]

  def _make_trainer(self, tower):
    from ranking_b200 import train as train_lib
    hp = self._hparams
    return train_lib.RankingTrainer(tower, self.build_loss(), optimizer=hp.optimizer,
                                    learning_rate=hp.learning_rate, process_group=self._group)

  def _train_step(self, trainer, batch, dev):
    x, y = batch
    return trainer.train_step(x.to(dev, non_blocking=True), y.to(dev, non_blocking=True))

  def _validation_logs(self, trainer, vb, dev):
    logs = evaluate(trainer, vb, self.build_metrics())
    vloss = 0.0
    loss_obj = trainer.loss
    for x, y in vb:
      xd, yd = x.to(dev), y.to(dev)
      vloss += float(loss_obj(yd, trainer.predict(xd, mask=(yd >= 0)).clone()))
    logs['loss'] = vloss / max(len(vb), 1)
    return logs

  def train_and_validate(self, verbose=0):
    hp = self._hparams
    tower = self._tower_fn()
    trainer = self._make_trainer(tower)
    os.makedirs(hp.model_dir, exist_ok=True)
    ckpt = os.path.join(hp.model_dir, 'ckpt.pt')
    best_dir = os.path.join(hp.model_dir, 'best_checkpoint')
    step = load_checkpoint(trainer, ckpt) if os.path.exists(ckpt) else 0
    first_epoch = step // hp.steps_per_epoch
    higher = hp.best_exporter_metric_higher_better
    best, bad_epochs, lr_bad = None, 0, 0
    train_it = iter(self._train_fn())
    dev = trainer.device
    for epoch in range(first_epoch, hp.num_epochs):
      loss_sum, n = 0.0, 0
      while step < (epoch + 1) * hp.steps_per_epoch:
        try:
          batch = next(train_it)
        except StopIteration:
          train_it = iter(self._train_fn())
          batch = next(train_it)
        loss = self._train_step(trainer, batch, dev)
        step += 1
        loss_sum += float(loss)
        n += 1
      logs = {'epoch': epoch + 1, 'step': step, 'train_loss': loss_sum / max(n, 1)}
      if self._valid_fn is not None and hp.validation_steps > 0:
        import itertools
        vb = list(itertools.islice(iter(self._valid_fn()), hp.validation_steps))
        logs.update(self._validation_logs(trainer, vb, dev))
      else:
        logs['loss'] = logs['train_loss']
      self.history.append(logs)
      if verbose:
        self._log(str(logs))
      save_checkpoint(trainer, ckpt, step)
      cur = self._monitor(logs)
      improved = best is None or (cur > best + hp.early_stopping_min_delta if higher
                                  else cur < best - hp.early_stopping_min_delta)
      if improved:
        best, bad_epochs, lr_bad = cur, 0, 0
        if hp.export_best_model:
          os.makedirs(best_dir, exist_ok=True)
          save_checkpoint(trainer, os.path.join(best_dir, 'ckpt.pt'), step)
      else:
        bad_epochs += 1
        lr_bad += 1
        if hp.automatic_reduce_lr and lr_bad >= max(1, hp.num_epochs // 3):
          trainer.lr *= 0.1        # ReduceLROnPlateau(factor=0.1), keras/pipeline.py:465-472
          lr_bad = 0
        if hp.early_stopping_patience > 0 and bad_epochs >= hp.early_stopping_patience:
          break
    self.trainer = trainer
    return self.history


class MultiTaskPipeline(ModelFitPipeline):
  """`MultiTaskPipeline` (keras/pipeline.py:733-824) over `MultiTaskRankingTrainer`, or over
  `trainer_cls` (`MultiTaskDINRankingTrainer`, `MultiTaskDASALCRankingTrainer`), which is
  called as trainer_cls(*parts, losses, ...) with `parts` what `tower_fn()` returns: a tower,
  or a tuple of model parts such as (din, tower) or (din, scorer).  `hparams.loss` maps each task to a loss key (dict order = the tower's output units) and
  `hparams.loss_weights` is None or a dict over those tasks.  The epoch loop, checkpoints,
  best checkpoint, early stopping and ReduceLROnPlateau are `ModelFitPipeline`'s.

  Batches are (x, labels {task: [B, N]}, mask, sample_weight or None), as
  `data.elwc_multilabel_batches` yields them, or (x, labels).  Validation logs use Keras'
  multi-output names: `loss` (sum_t w_t <task>_loss), `<task>_loss`, and
  `<task>_metric/ndcg_1`, `_5`, `_10`, `<task>_metric/ndcg`; with `use_weighted_metrics` also
  `<task>_weighted_metric/...` under the sample weights.  `best_exporter_metric` may name any
  of them."""

  TOPNS = (1, 5, 10, None)

  def __init__(self, tower_fn, train_batches_fn, valid_batches_fn, hparams,
               process_group=None, log_fn=print, trainer_cls=None):
    super().__init__(tower_fn, train_batches_fn, valid_batches_fn, hparams,
                     process_group=process_group, log_fn=log_fn)
    self.tasks = list(hparams.loss)
    self._trainer_cls = trainer_cls

  @staticmethod
  def _validate_hparams(hparams):
    # PipelineHparams.validate() refuses loss maps (the single-task step); the loop checks
    # are shared.
    if not isinstance(hparams.loss, dict) or not hparams.loss:
      raise ValueError('MultiTaskPipeline needs hparams.loss as a dict task -> loss key')
    if len(hparams.loss) > 8:
      raise ValueError('at most 8 tasks, got %d' % len(hparams.loss))
    weights = hparams.loss_weights
    if weights is not None:
      if not isinstance(weights, dict):
        raise ValueError('loss_weights must be None or a dict over the tasks')
      unknown = sorted(set(weights) - set(hparams.loss))
      if unknown:
        raise ValueError('loss_weights name unknown tasks %s' % unknown)
    hparams.validate_loop()

  def build_loss(self):
    from ranking_b200.keras import losses as keras_losses
    kw = {}
    if self._hparams.loss_reduction not in (None, 'auto'):
      kw['reduction'] = self._hparams.loss_reduction
    return {t: keras_losses.get(key, **kw) for t, key in self._hparams.loss.items()}

  def _make_trainer(self, tower):
    from ranking_b200 import train as train_lib
    hp = self._hparams
    cls = self._trainer_cls or train_lib.MultiTaskRankingTrainer
    parts = tower if isinstance(tower, tuple) else (tower,)
    return cls(*parts, self.build_loss(), loss_weights=hp.loss_weights, optimizer=hp.optimizer,
               learning_rate=hp.learning_rate, process_group=self._group)

  @staticmethod
  def _unpack(batch, dev, non_blocking=False):
    x, labels = batch[0], batch[1]
    mask = batch[2] if len(batch) > 2 else None
    weights = batch[3] if len(batch) > 3 else None
    mv = lambda t: None if t is None else t.to(dev, non_blocking=non_blocking)
    return mv(x), {t: mv(y) for t, y in labels.items()}, mv(mask), mv(weights)

  def _train_step(self, trainer, batch, dev):
    x, labels, mask, weights = self._unpack(batch, dev, non_blocking=True)
    return trainer.train_step(x, labels, sample_weight=weights, mask=mask)

  def _validation_logs(self, trainer, vb, dev):
    hp = self._hparams
    groups = {t: keras_metrics.MetricGroup(topns=self.TOPNS) for t in self.tasks}
    wgroups = {t: keras_metrics.MetricGroup(topns=self.TOPNS) for t in self.tasks} \
        if hp.use_weighted_metrics else {}
    tloss = {t: 0.0 for t in self.tasks}
    for batch in vb:
      x, labels, mask, weights = self._unpack(batch, dev)
      scores = trainer.predict(x, mask=mask, labels=labels)
      for t in self.tasks:
        s = scores[t].clone()
        groups[t].update_state(labels[t], s)
        if t in wgroups:
          wgroups[t].update_state(labels[t], s, weights)
        tloss[t] += float(trainer.losses[t](labels[t], s, weights))
    logs = {}
    total = 0.0
    for i, t in enumerate(self.tasks):
      for prefix, gs in (('_metric/', groups), ('_weighted_metric/', wgroups)):
        if t not in gs:
          continue
        gs[t].all_reduce(trainer.group)
        for key, v in gs[t].result().items():
          if key.startswith('metric/ndcg'):
            logs[t + prefix + key[len('metric/'):]] = v
      logs[t + '_loss'] = tloss[t] / max(len(vb), 1)
      total += trainer.loss_weights[i] * logs[t + '_loss']
    logs['loss'] = total
    return logs
