"""The `tfr.keras.losses` surface on torch tensors + fused CUDA kernels.

Mirrors tensorflow_ranking/python/keras/losses.py: `RankingLossKey`, `get`,
the serialisable LambdaWeight classes with their Keras defaults, and the loss
classes `__call__(y_true, y_pred, sample_weight=None) -> scalar` with the Keras
reduction semantics (AUTO / SUM_OVER_BATCH_SIZE -> sum / numel of the per-item
or per-list loss tensor; pairwise losses therefore divide by B*N,
keras/losses.py:324-335; listwise by B).  Losses are differentiable w.r.t.
`y_pred` through torch autograd.
"""
import torch

from ranking_b200 import _C
from ranking_b200 import losses_impl
from ranking_b200.keras import utils


class Reduction(object):
  """tf.keras.losses.Reduction."""
  AUTO = 'auto'
  NONE = 'none'
  SUM = 'sum'
  SUM_OVER_BATCH_SIZE = 'sum_over_batch_size'

  @classmethod
  def validate(cls, key):
    if key not in (cls.AUTO, cls.NONE, cls.SUM, cls.SUM_OVER_BATCH_SIZE):
      raise ValueError('Invalid Reduction Key: {}.'.format(key))


class RankingLossKey(object):
  """keras/losses.py:25-48 (keys of losses not on the hot path are listed so
  that `get` can say precisely what is unsupported)."""
  PAIRWISE_HINGE_LOSS = 'pairwise_hinge_loss'
  PAIRWISE_LOGISTIC_LOSS = 'pairwise_logistic_loss'
  PAIRWISE_SOFT_ZERO_ONE_LOSS = 'pairwise_soft_zero_one_loss'
  PAIRWISE_MSE_LOSS = 'pairwise_mse_loss'
  YETI_LOGISTIC_LOSS = 'yeti_logistic_loss'
  SOFTMAX_LOSS = 'softmax_loss'
  CALIBRATED_SOFTMAX_LOSS = 'calibrated_softmax_loss'
  UNIQUE_SOFTMAX_LOSS = 'unique_softmax_loss'
  SIGMOID_CROSS_ENTROPY_LOSS = 'sigmoid_cross_entropy_loss'
  MEAN_SQUARED_LOSS = 'mean_squared_loss'
  ORDINAL_LOSS = 'ordinal_loss'
  LIST_MLE_LOSS = 'list_mle_loss'
  APPROX_NDCG_LOSS = 'approx_ndcg_loss'
  APPROX_MRR_LOSS = 'approx_mrr_loss'
  GUMBEL_APPROX_NDCG_LOSS = 'gumbel_approx_ndcg_loss'
  COUPLED_RANKDISTIL_LOSS = 'coupled_rankdistil_loss'

  @classmethod
  def all_keys(cls):
    return [v for k, v in vars(cls).items() if k.isupper()]


# ---------------------------------------------------------------------------
# LambdaWeights with Keras defaults (keras/losses.py:114-244)
# ---------------------------------------------------------------------------
class LabelDiffLambdaWeight(losses_impl.LabelDiffLambdaWeight):

  def __init__(self, **kwargs):
    super().__init__()

  def get_config(self):
    return {}


class DCGLambdaWeight(losses_impl.DCGLambdaWeight):

  def __init__(self, topn=None, gain_fn=None, rank_discount_fn=None,
               normalized=False, smooth_fraction=0., **kwargs):
    super().__init__(topn, gain_fn or utils.identity,
                     rank_discount_fn or utils.inverse, normalized,
                     smooth_fraction)

  def get_config(self):
    return {
        'topn': self._topn,
        'gain_fn': self._gain_fn,
        'rank_discount_fn': self._rank_discount_fn,
        'normalized': self._normalized,
        'smooth_fraction': self._smooth_fraction,
    }


class NDCGLambdaWeight(DCGLambdaWeight):

  def __init__(self, topn=None, gain_fn=None, rank_discount_fn=None,
               smooth_fraction=0., **kwargs):
    super().__init__(topn, gain_fn or utils.pow_minus_1,
                     rank_discount_fn or utils.log2_inverse, normalized=True,
                     smooth_fraction=smooth_fraction)


class NDCGLambdaWeightV2(losses_impl.DCGLambdaWeightV2):

  def __init__(self, topn=None, gain_fn=None, rank_discount_fn=None, **kwargs):
    super().__init__(topn, gain_fn or utils.pow_minus_1,
                     rank_discount_fn or utils.log2_inverse, normalized=True)

  def get_config(self):
    return {
        'topn': self._topn,
        'gain_fn': self._gain_fn,
        'rank_discount_fn': self._rank_discount_fn,
    }


class YetiDCGLambdaWeight(losses_impl.YetiDCGLambdaWeight):

  def __init__(self, topn=None, gain_fn=None, rank_discount_fn=None,
               normalized=False, **kwargs):
    super().__init__(topn, gain_fn or utils.pow_minus_1,
                     rank_discount_fn or utils.log2_inverse,
                     normalized=normalized)

  def get_config(self):
    return {
        'topn': self._topn,
        'gain_fn': self._gain_fn,
        'rank_discount_fn': self._rank_discount_fn,
        'normalized': self._normalized,
    }


class PrecisionLambdaWeight(losses_impl.PrecisionLambdaWeight):

  def __init__(self, topn=None, positive_fn=None, **kwargs):
    super().__init__(topn, positive_fn or utils.is_greater_equal_1)

  def get_config(self):
    return {'topn': self._topn, 'positive_fn': self._positive_fn}


# ---------------------------------------------------------------------------
# losses
# ---------------------------------------------------------------------------
def _keras_reduce(losses, sample_weight, reduction):
  """tf.keras compute_weighted_loss: rank-align the weights, multiply, reduce."""
  if sample_weight is not None and not isinstance(sample_weight, float):
    sw = sample_weight
    if sw.dim() == losses.dim() + 1 and sw.shape[-1] == 1:
      sw = sw.squeeze(-1)
    elif sw.dim() == losses.dim() - 1:
      sw = sw.unsqueeze(-1)
    losses = losses * sw
  elif isinstance(sample_weight, float) and sample_weight != 1.0:
    losses = losses * sample_weight
  if reduction == Reduction.NONE:
    return losses
  total = losses.sum()
  if reduction == Reduction.SUM:
    return total
  return total / float(losses.numel())


class _RankingLoss(object):
  """keras/losses.py:247-285."""

  def __init__(self, reduction=Reduction.AUTO, name=None, ragged=False):
    Reduction.validate(reduction)
    self.reduction = reduction
    self.name = name
    self._loss = None
    self._ragged = ragged

  def __call__(self, y_true, y_pred, sample_weight=None):
    raise NotImplementedError

  def get_config(self):
    return {'reduction': self.reduction, 'name': self.name,
            'ragged': self._ragged}

  @classmethod
  def from_config(cls, config):
    return cls(**config)


class _PairwiseLoss(_RankingLoss):
  """keras/losses.py:288-335."""
  _impl = None

  def __init__(self, reduction=Reduction.AUTO, name=None, lambda_weight=None,
               temperature=1.0, ragged=False, **kwargs):
    super().__init__(reduction, name, ragged)
    self._lambda_weight = lambda_weight
    self._temperature = temperature
    self._loss = self._impl(name='{}_impl'.format(name) if name else None,
                            lambda_weight=lambda_weight,
                            temperature=temperature, ragged=ragged)

  def __call__(self, y_true, y_pred, sample_weight=None):
    # `normalize_weights` + `call` + the Keras reduction of the reference are
    # one kernel here: row sums already carry the item weights w_i.
    row = self._loss.compute_row_sums(y_true, y_pred, sample_weight)
    return _keras_reduce(row, None, self.reduction)

  def fused_fwd_bwd(self, y_true, y_pred, sample_weight, grad_out, per_list,
                    total2):
    """Training fast path: ONE launch writes d loss / d y_pred (already divided
    by the Keras normaliser) into `grad_out` and the per-list loss sums into
    `per_list[0]`; a second tiny launch reduces the scalar loss into `total2[0]`.
    No autograd graph, no intermediate tensors."""
    labels, logits = losses_impl._prep_2d(y_true, y_pred)
    w, wpi = losses_impl._prep_weights(sample_weight, logits)
    b, n = logits.shape
    scale = 1.0 if self.reduction == Reduction.SUM else 1.0 / float(b * n)
    cfg, keep = losses_impl._lambda_cfg(self._lambda_weight, labels)
    _C.check(_C.lib.tfr_pairwise_loss_fwd_bwd(
        _C.ptr(logits), _C.ptr(labels), _C.ptr(w), wpi, None, b, n,
        float(self._temperature), self._loss._phi, losses_impl._byref(cfg),
        scale, _C.ptr(grad_out), None, _C.ptr(per_list[0]), None, None, None,
        _C.stream()))
    del keep
    _C.check(_C.lib.tfr_weighted_sum(_C.ptr(per_list[0]), None, b, scale,
                                     _C.ptr(total2), _C.stream()))

  def get_config(self):
    config = super().get_config()
    config.update({'lambda_weight': self._lambda_weight,
                   'temperature': self._temperature})
    return config


class PairwiseHingeLoss(_PairwiseLoss):
  """keras/losses.py:338-402."""
  _impl = losses_impl.PairwiseHingeLoss


class PairwiseLogisticLoss(_PairwiseLoss):
  """keras/losses.py:405-469."""
  _impl = losses_impl.PairwiseLogisticLoss


class PairwiseSoftZeroOneLoss(_PairwiseLoss):
  """keras/losses.py:472-537."""
  _impl = losses_impl.PairwiseSoftZeroOneLoss


class PairwiseMSELoss(_PairwiseLoss):
  """keras/losses.py:540-606."""
  _impl = losses_impl.PairwiseMSELoss


class _ListwiseLoss(_RankingLoss):
  """keras/losses.py:721-755."""
  _impl = None
  _default_temperature = 1.0

  def __init__(self, reduction=Reduction.AUTO, name=None, lambda_weight=None,
               temperature=None, ragged=False, **kwargs):
    super().__init__(reduction, name, ragged)
    if temperature is None:
      temperature = self._default_temperature
    self._lambda_weight = lambda_weight
    self._temperature = temperature
    self._loss = self._impl(name='{}_impl'.format(name) if name else None,
                            lambda_weight=lambda_weight,
                            temperature=temperature, ragged=ragged)

  def __call__(self, y_true, y_pred, sample_weight=None):
    # losses [B] * loss weights [B] (already times the normalised sample
    # weight, losses_impl.py:1004-1015), then the Keras reduction over [B, 1].
    losses, weights = self._loss._run(y_true, y_pred, sample_weight, None,
                                      self._temperature)
    return _keras_reduce((losses * weights).unsqueeze(1), None, self.reduction)

  def fused_fwd_bwd(self, y_true, y_pred, sample_weight, grad_out, per_list,
                    total2):
    """Training fast path (see _PairwiseLoss.fused_fwd_bwd): per_list[0] = loss,
    per_list[1] = weight, total2[0] = reduced scalar loss."""
    labels, logits = losses_impl._prep_2d(y_true, y_pred)
    w, wpi = losses_impl._prep_weights(sample_weight, logits)
    b, n = logits.shape
    scale = 1.0 if self.reduction == Reduction.SUM else 1.0 / float(b)
    kind = self._loss._kind
    if kind == 'softmax':
      cfg, keep = losses_impl._lambda_cfg(self._lambda_weight, labels)
      _C.check(_C.lib.tfr_softmax_loss_fwd_bwd(
          _C.ptr(logits), _C.ptr(labels), _C.ptr(w), wpi, None, b, n,
          float(self._temperature), losses_impl._byref(cfg), scale, 1,
          _C.ptr(grad_out), _C.ptr(per_list[0]), _C.ptr(per_list[1]),
          _C.stream()))
      del keep
    else:
      _C.check(_C.lib.tfr_approx_loss_fwd_bwd(
          _C.ptr(logits), _C.ptr(labels), _C.ptr(w), wpi, None, b, n,
          float(self._temperature), 0 if kind == 'ndcg' else 1, scale, 1,
          _C.ptr(grad_out), _C.ptr(per_list[0]), _C.ptr(per_list[1]),
          _C.stream()))
    _C.check(_C.lib.tfr_weighted_sum(_C.ptr(per_list[0]), _C.ptr(per_list[1]), b,
                                     scale, _C.ptr(total2), _C.stream()))

  def get_config(self):
    config = super().get_config()
    config.update({'lambda_weight': self._lambda_weight,
                   'temperature': self._temperature})
    return config


class SoftmaxLoss(_ListwiseLoss):
  """keras/losses.py:758-832."""
  _impl = losses_impl.SoftmaxLoss

  def __call__(self, y_true, y_pred, sample_weight=None):
    losses, weights = self._loss.compute_per_list(y_true, y_pred, sample_weight)
    return _keras_reduce(losses * weights, None, self.reduction)


class CalibratedSoftmaxLoss(SoftmaxLoss):
  """keras/losses.py:836-943: softmax loss over the list plus one virtual item with
  score 0, label `virtual_label` and weight 1 (anchors the scores to zero)."""

  def __init__(self, reduction=Reduction.AUTO, name=None, lambda_weight=None,
               temperature=1.0, virtual_label=0.0, **kwargs):
    super().__init__(reduction, name, lambda_weight, temperature, False)
    assert virtual_label >= 0, 'Virtual label must be non-negative.'
    self._virtual_label = virtual_label

  def _augment(self, y_true, y_pred, sample_weight):
    labels, logits = losses_impl._prep_2d(y_true, y_pred)
    b = labels.shape[0]
    labels = torch.cat([labels, labels.new_full((b, 1), float(self._virtual_label))], 1)
    logits = torch.cat([logits, logits.new_zeros((b, 1))], 1)
    if sample_weight is not None and torch.is_tensor(sample_weight) and \
        sample_weight.dim() == 2 and sample_weight.shape[1] > 1:
      sample_weight = torch.cat([sample_weight, sample_weight.new_ones((b, 1))], 1)
    return labels, logits, sample_weight

  def __call__(self, y_true, y_pred, sample_weight=None):
    return super().__call__(*self._augment(y_true, y_pred, sample_weight))

  def fused_fwd_bwd(self, y_true, y_pred, sample_weight, grad_out, per_list,
                    total2):
    labels, logits, w = self._augment(y_true, y_pred, sample_weight)
    g = torch.empty_like(logits)
    super().fused_fwd_bwd(labels, logits, w, g, per_list, total2)
    grad_out.copy_(g[:, :-1])

  def get_config(self):
    config = super().get_config()
    config.update({'virtual_label': self._virtual_label})
    return config


class ApproxNDCGLoss(_ListwiseLoss):
  """keras/losses.py:1164-1237."""
  _impl = losses_impl.ApproxNDCGLoss
  _default_temperature = 0.1


class ApproxMRRLoss(_ListwiseLoss):
  """keras/losses.py:1093-1161."""
  _impl = losses_impl.ApproxMRRLoss
  _default_temperature = 0.1


class _GumbelMixin(object):
  """Losses evaluated on `sample_size` Gumbel-perturbed copies of every list
  (keras/losses.py:609-718, 1241-1341)."""

  def _init_gumbel(self, name, sample_size, gumbel_temperature, seed, ragged):
    self._sample_size = sample_size
    self._gumbel_temperature = gumbel_temperature
    self._seed = seed
    self._gumbel_sampler = losses_impl.GumbelSampler(
        name=name, sample_size=sample_size, temperature=gumbel_temperature, seed=seed,
        ragged=ragged)
    self._bufs = None

  def __call__(self, y_true, y_pred, sample_weight=None):
    gbl_labels, gbl_logits, gbl_weights = self._gumbel_sampler.sample(
        y_true, y_pred, weights=sample_weight)
    return super().__call__(gbl_labels, gbl_logits, gbl_weights)

  def fused_fwd_bwd(self, y_true, y_pred, sample_weight, grad_out, per_list,
                    total2):
    """sample -> base loss on [B * S, N] -> sampler backward; `per_list` (sized for
    B lists) receives the per-list means over the S samples."""
    labels, logits = losses_impl._prep_2d(y_true, y_pred)
    smp = self._gumbel_sampler
    s_ = smp._sample_size
    b, n = logits.shape
    ex_labels, ex_w = smp.expand(labels, sample_weight)
    if self._bufs is None or self._bufs[0].shape != (b * s_, n):
      dev = logits.device
      self._bufs = (torch.empty(b * s_, n, device=dev), torch.empty(b * s_, n, device=dev),
                    torch.zeros(2, b * s_, device=dev))
    sampled, g_ex, pl_ex = self._bufs
    seed = smp.next_seed()
    _C.check(_C.lib.tfr_gumbel_sample(
        _C.ptr(logits), _C.ptr(labels), b, n, s_, float(smp._temperature), seed, 0,
        _C.ptr(sampled), None, None, _C.stream()))
    super().fused_fwd_bwd(ex_labels, sampled, ex_w, g_ex, pl_ex, total2)
    _C.check(_C.lib.tfr_gumbel_sample(
        _C.ptr(logits), _C.ptr(labels), b, n, s_, float(smp._temperature), seed, 0, None,
        _C.ptr(g_ex), _C.ptr(grad_out), _C.stream()))
    per_list.copy_(pl_ex.reshape(2, b, s_).mean(2))

  def get_config(self):
    config = super().get_config()
    config.update({'sample_size': self._sample_size,
                   'gumbel_temperature': self._gumbel_temperature,
                   'seed': self._seed})
    return config


class YetiLogisticLoss(_GumbelMixin, PairwiseLogisticLoss):
  """keras/losses.py:609-718: pairwise logistic loss with YetiDCGLambdaWeight on
  Gumbel-sampled scores."""

  def __init__(self, reduction=Reduction.AUTO, name=None, lambda_weight=None,
               temperature=1.0, sample_size=8, gumbel_temperature=1.0, seed=None,
               ragged=False):
    lambda_weight = lambda_weight or YetiDCGLambdaWeight()
    PairwiseLogisticLoss.__init__(self, reduction, name, lambda_weight,
                                  temperature=temperature, ragged=ragged)
    self._init_gumbel(name, sample_size, gumbel_temperature, seed, ragged)


class GumbelApproxNDCGLoss(_GumbelMixin, ApproxNDCGLoss):
  """keras/losses.py:1241-1341."""

  def __init__(self, reduction=Reduction.AUTO, name=None, lambda_weight=None,
               temperature=0.1, sample_size=8, gumbel_temperature=1.0, seed=None,
               ragged=False):
    ApproxNDCGLoss.__init__(self, reduction, name, lambda_weight,
                            temperature=temperature, ragged=ragged)
    self._init_gumbel(name, sample_size, gumbel_temperature, seed, ragged)


class _MiscListwiseLoss(_ListwiseLoss):
  """Listwise losses served by K3b (tfr_misc_loss_fwd_bwd)."""

  def fused_fwd_bwd(self, y_true, y_pred, sample_weight, grad_out, per_list,
                    total2):
    labels, logits = losses_impl._prep_2d(y_true, y_pred)
    w, wpi = losses_impl._prep_weights(sample_weight, logits)
    b, n = logits.shape
    scale = 1.0 if self.reduction == Reduction.SUM else 1.0 / float(b)
    table = None
    if isinstance(self._lambda_weight, losses_impl.ListMLELambdaWeight):
      table = self._lambda_weight.rank_table(n, logits.device)
    # grad_out = scale * d loss_b / d s; the list weight multiplies on the host side
    # of the kernel only when weights are given (weight_b = 1 otherwise).
    _C.check(_C.lib.tfr_misc_loss_fwd_bwd(
        _C.ptr(logits), _C.ptr(labels), _C.ptr(w), wpi, None, b, n,
        float(self._temperature), losses_impl._MISC[self._loss._kind],
        _C.ptr(table), None, 0, scale, _C.ptr(grad_out), None, _C.ptr(per_list[0]),
        _C.ptr(per_list[1]), None, _C.stream()))
    if w is not None:
      grad_out.mul_(per_list[1].unsqueeze(1))
    _C.check(_C.lib.tfr_weighted_sum(_C.ptr(per_list[0]), _C.ptr(per_list[1]), b,
                                     scale, _C.ptr(total2), _C.stream()))


class UniqueSoftmaxLoss(_MiscListwiseLoss):
  """keras/losses.py:946-1005."""
  _impl = losses_impl.UniqueSoftmaxLoss


class ListMLELoss(_MiscListwiseLoss):
  """keras/losses.py:1008-1090."""
  _impl = losses_impl.ListMLELoss


class ListMLELambdaWeight(losses_impl.ListMLELambdaWeight):
  """keras/losses.py:233-244."""

  def __init__(self, rank_discount_fn=None, **kwargs):
    super().__init__(rank_discount_fn)

  def get_config(self):
    return {'rank_discount_fn': self._rank_discount_fn}


class _PointwiseLoss(_RankingLoss):
  """keras/losses.py:1499-1600: `call` returns loss_i * mask_i, `__call__` applies the
  normalised sample weight and the Keras reduction; one kernel launch here."""
  _impl = None

  def __call__(self, y_true, y_pred, sample_weight=None):
    rows = self._loss.compute_weighted_rows(y_true, y_pred, sample_weight)
    return _keras_reduce(rows, None, self.reduction)

  def fused_fwd_bwd(self, y_true, y_pred, sample_weight, grad_out, per_list,
                    total2):
    labels, logits = losses_impl._prep_2d(y_true, y_pred)
    w, wpi = losses_impl._prep_weights(sample_weight, logits)
    b, n = logits.shape
    scale = 1.0 if self.reduction == Reduction.SUM else 1.0 / float(b * n)
    _C.check(_C.lib.tfr_misc_loss_fwd_bwd(
        _C.ptr(logits), _C.ptr(labels), _C.ptr(w), wpi, None, b, n,
        float(self._loss._temperature), losses_impl._MISC[self._loss._kind], None,
        None, 0, scale, _C.ptr(grad_out), None, _C.ptr(per_list[0]), _C.ptr(per_list[1]),
        None, _C.stream()))
    _C.check(_C.lib.tfr_weighted_sum(_C.ptr(per_list[0]), None, b, scale,
                                     _C.ptr(total2), _C.stream()))


class SigmoidCrossEntropyLoss(_PointwiseLoss):
  """keras/losses.py:1499-1546."""

  def __init__(self, reduction=Reduction.AUTO, name=None, ragged=False):
    super().__init__(reduction, name, ragged)
    self._loss = losses_impl.SigmoidCrossEntropyLoss(
        name='{}_impl'.format(name) if name else None, ragged=ragged)


class MeanSquaredLoss(_PointwiseLoss):
  """keras/losses.py:1549-1600."""

  def __init__(self, reduction=Reduction.AUTO, name=None, ragged=False):
    super().__init__(reduction, name, ragged)
    self._loss = losses_impl.MeanSquaredLoss(
        name='{}_impl'.format(name) if name else None, ragged=ragged)


class CoupledRankDistilLoss(_RankingLoss):
  """keras/losses.py:1659-1750."""

  def __init__(self, reduction=Reduction.AUTO, name=None, ragged=False, sample_size=8,
               topk=None, temperature=1.):
    super().__init__(reduction, name, ragged)
    self._sample_size = sample_size
    self._topk = topk
    self._temperature = temperature
    self._loss = losses_impl.CoupledRankDistilLoss(
        name='{}_impl'.format(name) if name else None, sample_size=sample_size,
        topk=topk, temperature=temperature, ragged=ragged)

  def __call__(self, y_true, y_pred, sample_weight=None):
    losses, weights = self._loss._run(y_true, y_pred, sample_weight, None,
                                      self._temperature)
    return _keras_reduce((losses * weights).unsqueeze(1), None, self.reduction)

  def fused_fwd_bwd(self, *args, **kwargs):
    raise NotImplementedError('CoupledRankDistilLoss: use the autograd path')

  def get_config(self):
    config = super().get_config()
    config.update({'sample_size': self._sample_size, 'topk': self._topk,
                   'temperature': self._temperature})
    return config


class OrdinalLoss(_PointwiseLoss):
  """keras/losses.py:1603-1656: y_pred [B, N, ordinal_size]."""

  def __init__(self, reduction=Reduction.AUTO, name=None, ragged=False,
               ordinal_size=1, use_fraction_label=False):
    super().__init__(reduction, name, ragged)
    self._loss = losses_impl.OrdinalLoss(
        name='{}_impl'.format(name) if name else None, ordinal_size=ordinal_size,
        ragged=ragged, use_fraction_label=use_fraction_label)

  def fused_fwd_bwd(self, *args, **kwargs):
    raise NotImplementedError('OrdinalLoss needs a multi-head scorer; use autograd')


_KEY_TO_CLS = {
    RankingLossKey.COUPLED_RANKDISTIL_LOSS: CoupledRankDistilLoss,
    RankingLossKey.ORDINAL_LOSS: OrdinalLoss,
    RankingLossKey.APPROX_NDCG_LOSS: ApproxNDCGLoss,
    RankingLossKey.APPROX_MRR_LOSS: ApproxMRRLoss,
    RankingLossKey.SIGMOID_CROSS_ENTROPY_LOSS: SigmoidCrossEntropyLoss,
    RankingLossKey.MEAN_SQUARED_LOSS: MeanSquaredLoss,
    RankingLossKey.GUMBEL_APPROX_NDCG_LOSS: GumbelApproxNDCGLoss,
}
_KEY_TO_CLS_WITH_LAMBDA = {
    RankingLossKey.PAIRWISE_HINGE_LOSS: PairwiseHingeLoss,
    RankingLossKey.PAIRWISE_LOGISTIC_LOSS: PairwiseLogisticLoss,
    RankingLossKey.PAIRWISE_SOFT_ZERO_ONE_LOSS: PairwiseSoftZeroOneLoss,
    RankingLossKey.PAIRWISE_MSE_LOSS: PairwiseMSELoss,
    RankingLossKey.SOFTMAX_LOSS: SoftmaxLoss,
    RankingLossKey.CALIBRATED_SOFTMAX_LOSS: CalibratedSoftmaxLoss,
    RankingLossKey.UNIQUE_SOFTMAX_LOSS: UniqueSoftmaxLoss,
    RankingLossKey.LIST_MLE_LOSS: ListMLELoss,
    RankingLossKey.YETI_LOGISTIC_LOSS: YetiLogisticLoss,
}


def get(loss, reduction=Reduction.AUTO, lambda_weight=None, name=None, **kwargs):
  """keras/losses.py:51-111."""
  loss_kwargs = {'reduction': reduction, 'name': name}
  loss_kwargs.update(kwargs)
  if loss in _KEY_TO_CLS:
    return _KEY_TO_CLS[loss](**loss_kwargs)
  if loss in _KEY_TO_CLS_WITH_LAMBDA:
    return _KEY_TO_CLS_WITH_LAMBDA[loss](lambda_weight=lambda_weight,
                                         **loss_kwargs)
  if loss in RankingLossKey.all_keys():
    raise ValueError('unsupported loss: {} (not on the GPU hot path yet; see '
                     'DESIGN.md scope)'.format(loss))
  raise ValueError('unsupported loss: {}'.format(loss))
