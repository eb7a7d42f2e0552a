"""Oracle restatement of the click-model losses and of a click EM training step:

  * ClickEMLoss (losses_impl.py:1324-1422) and MixtureEMLoss (:1472-1538), with the Keras
    wrappers (keras/losses.py:1344-1496): dense or ragged inputs, autograd gradients with
    `.detach()` where the reference has `stop_gradient`;
  * ClickEMTrainer: a relevance tower and a per-position examination table trained jointly
    with ClickEM, autograd and tf.keras Adagrad (the regression EM of Wang et al. 2018 run
    online).

Test infrastructure only (see oracle/__init__.py).  Plain torch on the CPU; fp32 or fp64 by
the dtype of the tensors passed in.
"""
import torch

from oracle import keras_losses
from oracle import losses_impl
from oracle import scorer
from oracle import utils


def _sce(labels, logits):
  """tf.nn.sigmoid_cross_entropy_with_logits: max(x, 0) - x z + log(1 + exp(-|x|))."""
  return torch.clamp(logits, min=0) - logits * labels + torch.log1p(torch.exp(-logits.abs()))


def ragged_to_dense(labels, logits, weights):
  """utils.py:421-443 for lists given as per-list sequences: labels pad -1, logits -1e6
  (trailing dims kept), per-item weights 0; returns (labels, logits, weights, mask)."""
  lab_rows = [torch.as_tensor(r, dtype=torch.float64) for r in labels]
  n = max([r.shape[0] for r in lab_rows] + [1])
  b = len(lab_rows)
  mask = torch.zeros(b, n, dtype=torch.bool)
  dense_labels = torch.full((b, n), -1., dtype=torch.float64)
  for i, r in enumerate(lab_rows):
    mask[i, :r.shape[0]] = True
    dense_labels[i, :r.shape[0]] = r
  dense_logits = None
  if logits is not None:
    rows = [torch.as_tensor(r, dtype=torch.float64) for r in logits]
    dense_logits = torch.full((b, n) + tuple(rows[0].shape[1:]), -1e6, dtype=torch.float64)
    for i, r in enumerate(rows):
      dense_logits[i, :r.shape[0]] = r
  if isinstance(weights, (list, tuple)) and all(
      torch.as_tensor(w).dim() >= 1 and torch.as_tensor(w).shape[0] == r.shape[0]
      for w, r in zip(weights, lab_rows)):
    dense_w = torch.zeros(b, n, dtype=torch.float64)
    for i, w in enumerate(weights):
      dense_w[i, :len(w)] = torch.as_tensor(w, dtype=torch.float64)
    weights = dense_w
  return dense_labels, dense_logits, weights, mask


class _Ragged(object):
  """ragged=True: inputs are lists of per-list sequences, densified first; the mask of
  the padding replaces the `mask` argument, as in the reference."""

  def _dense(self, labels, logits, weights, mask):
    if not self._ragged:
      return labels, logits, weights, mask
    return ragged_to_dense(labels, logits, weights)

  def compute(self, labels, logits, weights, reduction, mask=None):
    labels, logits, weights, mask = self._dense(labels, logits, weights, mask)
    return super().compute(labels, logits, weights, reduction, mask)

  def compute_per_list(self, labels, logits, weights, mask=None):
    labels, logits, weights, mask = self._dense(labels, logits, weights, mask)
    return super().compute_per_list(labels, logits, weights, mask)

  def compute_unreduced_loss(self, labels, logits, mask=None):
    labels, logits, _, mask = self._dense(labels, logits, None, mask)
    return super().compute_unreduced_loss(labels, logits, mask)

  def normalize_weights(self, labels, weights):
    labels, _, weights, _ = self._dense(labels, None, weights, None)
    return super().normalize_weights(labels, weights)


class ClickEMLoss(_Ragged, losses_impl._PointwiseLoss):
  """losses_impl.py:1324-1422: logits [B, N, 2] = (examination, relevance) logits."""

  def __init__(self, name=None, temperature=1.0, exam_loss_weight=1.0, rel_loss_weight=1.0,
               ragged=False):
    super().__init__(name, None, temperature)
    self._exam_loss_weight = exam_loss_weight
    self._rel_loss_weight = rel_loss_weight
    self._ragged = ragged

  def _compute_latent_prob(self, clicks, exam_logits, rel_logits):
    """E step (:1346-1391): posteriors from the stable logits e - softplus(r),
    r - softplus(e); 1 for clicked items; no gradient."""
    is_clicked = clicks >= 1.0
    exam_post = torch.sigmoid(exam_logits - torch.nn.functional.softplus(rel_logits))
    rel_post = torch.sigmoid(rel_logits - torch.nn.functional.softplus(exam_logits))
    one = torch.ones_like(exam_post)
    return (torch.where(is_clicked, one, exam_post).detach(),
            torch.where(is_clicked, one, rel_post).detach())

  def _compute_unreduced_loss_impl(self, labels, logits, mask=None):
    if logits.dim() != 3 or logits.shape[-1] != 2:
      raise ValueError('ClickEMLoss needs logits of shape [batch_size, list_size, 2]')
    if mask is None:
      mask = utils.is_label_valid(labels)
    labels = torch.where(mask, labels, torch.zeros_like(labels))
    exam_logits, rel_logits = logits.unbind(2)
    exam_logits = torch.where(mask, exam_logits, torch.zeros_like(exam_logits))
    rel_logits = torch.where(mask, rel_logits, torch.zeros_like(rel_logits))
    pe, pr = self._compute_latent_prob(labels, exam_logits, rel_logits)
    losses = (_sce(pe, exam_logits) * self._exam_loss_weight +
              _sce(pr, rel_logits) * self._rel_loss_weight)
    return losses, mask.to(logits.dtype)


class MixtureEMLoss(_Ragged, losses_impl._ListwiseLoss):
  """losses_impl.py:1472-1538: logits [B, N, model_num]."""

  def __init__(self, name=None, temperature=1.0, alpha=1.0, ragged=False):
    super().__init__(name, None, temperature)
    self._alpha = alpha
    self._ragged = ragged

  def _compute_unreduced_loss_impl(self, labels, logits, mask=None):
    if logits.dim() != 3:
      raise ValueError('MixtureEMLoss needs logits of shape [batch_size, list_size, M]')
    if mask is None:
      mask = utils.is_label_valid(labels)
    labels = torch.where(mask, labels, torch.zeros_like(labels))
    losses = _sce(labels.unsqueeze(2), logits)
    losses = torch.where(mask.unsqueeze(2), losses, torch.zeros_like(losses))
    per_list = losses.detach().sum(1, keepdim=True)                       # [B, 1, M]
    prob = torch.exp(-self._alpha * (per_list - per_list.min(2, keepdim=True).values))
    norm = prob.sum(2, keepdim=True)
    loss = (losses * prob / norm).sum((1, 2)).reshape(-1, 1)
    nonzero = labels.sum(1, keepdim=True) > 0
    return loss, nonzero.to(logits.dtype)


class _KerasLoss(keras_losses._RankingLoss):
  """keras/losses.py:247-285 with ragged inputs: densify, normalise the sample weight, then
  `call` (losses x loss weights) and the Keras reduction."""

  def __init__(self, reduction, name, ragged):
    super().__init__(reduction, name)
    self._ragged = ragged

  def __call__(self, y_true, y_pred, sample_weight=None):
    mask = None
    if self._ragged:
      y_true, y_pred, sample_weight, mask = ragged_to_dense(y_true, y_pred, sample_weight)
    y_pred = torch.as_tensor(y_pred)
    y_true = torch.as_tensor(y_true, dtype=y_pred.dtype)
    impl = self._loss
    sample_weight = losses_impl._RankingLoss.normalize_weights(impl, y_true, sample_weight)
    y_pred = impl.get_logits(y_pred)
    labels, logits, _, mask = impl._prepare_and_validate_params(y_true, y_pred, None, mask)
    losses, weights = impl._compute_unreduced_loss_impl(labels, logits, mask)
    return keras_losses._keras_compute_weighted_loss(losses * weights, sample_weight,
                                                     self.reduction)

  def get_config(self):
    return dict(self._config, reduction=self.reduction, name=self.name, ragged=self._ragged)

  @classmethod
  def from_config(cls, config):
    return cls(**config)


class KerasClickEMLoss(_KerasLoss):
  """keras/losses.py:1344-1418."""

  def __init__(self, reduction=keras_losses.Reduction.AUTO, name=None, exam_loss_weight=1.0,
               rel_loss_weight=1.0, ragged=False):
    super().__init__(reduction, name, ragged)
    self._config = dict(exam_loss_weight=exam_loss_weight, rel_loss_weight=rel_loss_weight)
    self._loss = ClickEMLoss(name, exam_loss_weight=exam_loss_weight,
                             rel_loss_weight=rel_loss_weight)


class KerasMixtureEMLoss(_KerasLoss):
  """keras/losses.py:1421-1496: lambda_weight and temperature are kept in the config only
  (the impl is built without them, :1484-1489)."""

  def __init__(self, reduction=keras_losses.Reduction.AUTO, name=None, lambda_weight=None,
               temperature=1.0, alpha=1.0, ragged=False):
    super().__init__(reduction, name, ragged)
    self._config = dict(lambda_weight=lambda_weight, temperature=temperature, alpha=alpha)
    self._loss = MixtureEMLoss(name, alpha=alpha)


class ClickEMTrainer(object):
  """One relevance tower (scorer.tower_forward over `params`) and an examination table
  [num_positions] trained jointly: exam logit = table[position], relevance logit =
  tower(x), Keras ClickEMLoss on (exam, rel), autograd, tf.keras Adagrad over the table
  and the tower parameters.  With BatchNormalization the padded slots of a list are filled
  circularly with its valid items before the tower (FlattenList(circular_padding=True))."""

  def __init__(self, params, table, activation='relu', use_batch_norm=False, bn_moving=None,
               exam_loss_weight=1.0, rel_loss_weight=1.0, learning_rate=0.001, epsilon=1e-7,
               initial_accumulator_value=0.1, reduction=keras_losses.Reduction.AUTO):
    self.params = params
    self.table = table
    self.activation = activation
    self.use_batch_norm = use_batch_norm
    self.bn_moving = bn_moving
    self.loss = KerasClickEMLoss(reduction, exam_loss_weight=exam_loss_weight,
                                 rel_loss_weight=rel_loss_weight)
    self.lr = learning_rate
    self.eps = epsilon
    self.leaves = [table]
    for w, b in zip(params['dense_w'], params['dense_b']):
      self.leaves += [w, b]
    for g, b in zip(params['bn_gamma'], params['bn_beta']):
      self.leaves += [g, b]
    for p in self.leaves:
      p.requires_grad_()
    self.accum = [torch.full_like(p, initial_accumulator_value) for p in self.leaves]

  def default_positions(self, b, n):
    p = torch.arange(n).clamp(max=self.table.shape[0] - 1)
    return p.unsqueeze(0).expand(b, n)

  def relevance(self, x, valid, training):
    b, n, d = x.shape
    if self.use_batch_norm and training:
      idx, _ = utils.padded_nd_indices(valid)
      x = torch.gather(x, 1, idx.unsqueeze(2).expand(-1, -1, d))
    rel = scorer.tower_forward(x.reshape(b * n, d), self.params, activation=self.activation,
                               use_batch_norm=self.use_batch_norm, training=training,
                               bn_moving=self.bn_moving)
    return rel.reshape(b, n)

  def train_step(self, x, clicks, positions=None, sample_weight=None):
    b, n, _ = x.shape
    if positions is None:
      positions = self.default_positions(b, n)
    for p in self.leaves:
      p.grad = None
    exam = self.table[torch.as_tensor(positions, dtype=torch.int64)]
    rel = self.relevance(x, clicks >= 0, True)
    loss = self.loss(clicks, torch.stack([exam, rel], 2), sample_weight)
    loss.backward()
    with torch.no_grad():
      for p, a in zip(self.leaves, self.accum):
        a.add_(p.grad * p.grad)
        p.sub_(self.lr * p.grad / (a.sqrt() + self.eps))
    return loss.detach()

  def flat_grad(self):
    return torch.cat([p.grad.reshape(-1) for p in self.leaves])

  def flat_params(self):
    return torch.cat([p.detach().reshape(-1) for p in self.leaves])

  def examination_propensity(self):
    return torch.sigmoid(self.table.detach())
