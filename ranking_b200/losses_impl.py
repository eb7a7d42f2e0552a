"""Host-side mirror of tensorflow_ranking/python/losses_impl.py for the hot path.

Same class names, constructor arguments and method meaning as the reference
(`compute`, `compute_per_list`, `normalize_weights`, `get_logits`), but every
numeric step runs in the fused CUDA kernels behind the C ABI
(include/tfr_b200.h): no [B, N, N] tensor is ever created.  Gradients are
produced by the same kernel launch as the forward values (weights and ranks are
`stop_gradient` constants in the reference, losses_impl.py:882-883), and are
wired into torch autograd through `torch.autograd.Function`.
"""
import ctypes

import torch

from ranking_b200 import _C
from ranking_b200.keras import utils as keras_utils

_EPSILON = 1e-10


class Reduction(object):
  """tf.compat.v1.losses.Reduction values used by `compute` (losses.py:66-67)."""
  NONE = 'none'
  SUM = 'weighted_sum'
  MEAN = 'weighted_mean'
  SUM_OVER_BATCH_SIZE = 'weighted_sum_over_batch_size'
  SUM_BY_NONZERO_WEIGHTS = 'weighted_sum_by_nonzero_weights'


# ----------------------------------------------------------------------------
# tensor plumbing
# ----------------------------------------------------------------------------
def _as_f32(x, device=None, what='tensor'):
  if not torch.is_tensor(x):
    x = torch.as_tensor(x, dtype=torch.float32,
                        device=device if device is not None else 'cuda')
  _C.require_cuda(x, what)
  if x.dtype != torch.float32:
    x = x.float()
  return x.contiguous()


def _prep_2d(labels, logits):
  logits = _as_f32(logits, what='logits')
  labels = _as_f32(labels, logits.device, 'labels')
  if logits.dim() != 2 or labels.shape != logits.shape:
    raise ValueError('labels and logits must both have shape [batch_size, '
                     'list_size]; got %s and %s' % (tuple(labels.shape),
                                                    tuple(logits.shape)))
  return labels, logits


def _prep_weights(weights, like):
  """None | scalar | [B, 1] | [B] | [B, N] -> (tensor or None, w_per_item)."""
  if weights is None:
    return None, 0
  b, n = like.shape
  w = _as_f32(weights, like.device, 'weights')
  if w.dim() == 0:
    return w.expand(b).contiguous(), 0
  if w.dim() == 1 and w.shape[0] == b:
    return w, 0
  if w.dim() == 2 and w.shape == (b, 1):
    return w.reshape(b).contiguous(), 0
  if w.dim() == 2 and w.shape == (b, n):
    return w, 1
  if w.dim() == 2 and w.shape == (1, n):
    return w.expand(b, n).contiguous(), 1
  raise ValueError('weights must be a scalar, [batch_size, 1] or [batch_size, '
                   'list_size]; got %s' % (tuple(w.shape),))


def _prep_mask(mask, like):
  if mask is None:
    return None
  m = torch.as_tensor(mask, device=like.device)
  if m.shape != like.shape:
    raise ValueError('mask must have the shape of logits')
  return m.to(torch.uint8).contiguous()


def _safe_div(num, den):
  den_t = torch.as_tensor(den, dtype=num.dtype, device=num.device)
  return torch.where(den_t != 0, num / torch.where(den_t != 0, den_t,
                                                   torch.ones_like(den_t)),
                     torch.zeros_like(num))


# ----------------------------------------------------------------------------
# LambdaWeight family (losses_impl.py:170-454): configuration objects that
# select the in-kernel lambda; `pair_weights` materialises [B, N, N] for parity
# tests only (small N).
# ----------------------------------------------------------------------------
_GAIN_ENUM = {keras_utils.identity: _C.GAIN_IDENTITY,
              keras_utils.pow_minus_1: _C.GAIN_POW2_MINUS_1}
_DISC_ENUM = {keras_utils.inverse: _C.DISC_INVERSE,
              keras_utils.log2_inverse: _C.DISC_LOG2_INVERSE,
              keras_utils.log1p_inverse: _C.DISC_LOG1P_INVERSE}


class _LambdaWeight(object):
  _kind = _C.LAMBDA_NONE
  _topn = None
  _gain_fn = None
  _rank_discount_fn = None
  _normalized = False
  _smooth_fraction = 0.

  def _cfg(self, labels):
    """Builds the C struct for a [B, N] label tensor; returns (cfg, keepalive)."""
    keep = []
    cfg = _C.LambdaCfg()
    cfg.kind = self._kind
    cfg.topn = int(self._topn) if self._topn else 0
    cfg.normalized = 1 if self._normalized else 0
    cfg.smooth_fraction = float(self._smooth_fraction)
    cfg.gain_fn = _C.GAIN_IDENTITY
    cfg.disc_fn = _C.DISC_INVERSE
    cfg.gain_table = None
    cfg.disc_table = None
    n = labels.shape[1]
    if self._gain_fn is not None:
      if self._gain_fn in _GAIN_ENUM:
        cfg.gain_fn = _GAIN_ENUM[self._gain_fn]
      elif self._kind == _C.LAMBDA_PRECISION and \
          self._gain_fn is keras_utils.is_greater_equal_1:
        cfg.gain_fn = _C.GAIN_IDENTITY
      else:
        cleaned = torch.where(labels >= 0, labels, torch.zeros_like(labels))
        table = torch.as_tensor(self._gain_fn(cleaned)).to(
            torch.float32).contiguous()
        keep.append(table)
        cfg.gain_fn = _C.GAIN_TABLE
        cfg.gain_table = table.data_ptr()
    if self._rank_discount_fn is not None:
      if self._rank_discount_fn in _DISC_ENUM:
        cfg.disc_fn = _DISC_ENUM[self._rank_discount_fn]
      else:
        r = torch.arange(0, n + 2, dtype=torch.float32, device=labels.device)
        r[0] = 1.0   # d(0) is never used; avoid evaluating user code at 0
        table = torch.as_tensor(self._rank_discount_fn(r)).to(
            torch.float32).contiguous()
        keep.append(table)
        cfg.disc_fn = _C.DISC_TABLE
        cfg.disc_table = table.data_ptr()
    return cfg, keep

  def pair_weights(self, labels, ranks):
    """[B, N, N] lambda pair weights for given 1-based ranks (parity helper)."""
    labels = _as_f32(labels, what='labels')
    ranks = torch.as_tensor(ranks, device=labels.device).to(
        torch.int32).contiguous()
    b, n = labels.shape
    out = torch.empty(b, n, n, dtype=torch.float32, device=labels.device)
    cfg, keep = self._cfg(labels)
    _C.check(_C.lib.tfr_lambda_pair_weights(
        _C.ptr(labels), _C.ptr(ranks), b, n, ctypes.byref(cfg), _C.ptr(out),
        _C.stream()))
    del keep
    return out

  def individual_weights(self, labels, ranks):
    """losses_impl.py:195-207."""
    return labels


class LabelDiffLambdaWeight(_LambdaWeight):
  """losses_impl.py:210-216."""
  _kind = _C.LAMBDA_LABEL_DIFF


class AbstractDCGLambdaWeight(_LambdaWeight):
  """losses_impl.py:219-296."""

  def __init__(self, topn=None, gain_fn=None, rank_discount_fn=None,
               normalized=False):
    self._topn = topn
    self._gain_fn = gain_fn or keras_utils.identity
    self._rank_discount_fn = rank_discount_fn or keras_utils.inverse
    self._normalized = normalized


class DCGLambdaWeight(AbstractDCGLambdaWeight):
  """losses_impl.py:299-369."""
  _kind = _C.LAMBDA_DCG

  def __init__(self, topn=None, gain_fn=None, rank_discount_fn=None,
               normalized=False, smooth_fraction=0.):
    super().__init__(topn, gain_fn, rank_discount_fn, normalized)
    if not 0. <= smooth_fraction <= 1.:
      raise ValueError('smooth_fraction %s should be in range [0, 1].' %
                       smooth_fraction)
    self._smooth_fraction = smooth_fraction


class DCGLambdaWeightV2(AbstractDCGLambdaWeight):
  """losses_impl.py:372-394."""
  _kind = _C.LAMBDA_DCG_V2


class YetiDCGLambdaWeight(DCGLambdaWeightV2):
  """losses_impl.py:397-407."""
  _kind = _C.LAMBDA_YETI


class PrecisionLambdaWeight(_LambdaWeight):
  """losses_impl.py:410-454."""
  _kind = _C.LAMBDA_PRECISION

  def __init__(self, topn, positive_fn=None):
    self._topn = topn
    self._gain_fn = positive_fn or keras_utils.is_greater_equal_1
    self._positive_fn = self._gain_fn


def _lambda_cfg(lambda_weight, labels):
  if lambda_weight is None:
    return None, []
  if not isinstance(lambda_weight, _LambdaWeight):
    raise ValueError('lambda_weight must be a ranking_b200 LambdaWeight object')
  cfg, keep = lambda_weight._cfg(labels)
  return cfg, keep


def _byref(cfg):
  return ctypes.byref(cfg) if cfg is not None else None


# ----------------------------------------------------------------------------
# autograd bridges
# ----------------------------------------------------------------------------
class _PairwiseFn(torch.autograd.Function):
  """loss_sum[B], row_loss[B, N], w_sum[B], nnz[B] = K1(logits, ...)."""

  @staticmethod
  def forward(ctx, logits, labels, w, w_per_item, mask, temperature, phi,
              lambda_weight):
    b, n = logits.shape
    dev = logits.device
    grad = torch.empty_like(logits)
    row_loss = torch.empty_like(logits)
    loss_sum = torch.empty(b, dtype=torch.float32, device=dev)
    w_sum = torch.empty_like(loss_sum)
    nnz = torch.empty_like(loss_sum)
    cfg, keep = _lambda_cfg(lambda_weight, labels)
    _C.check(_C.lib.tfr_pairwise_loss_fwd_bwd(
        _C.ptr(logits), _C.ptr(labels), _C.ptr(w), w_per_item, _C.ptr(mask), b,
        n, float(temperature), phi, _byref(cfg), 1.0, _C.ptr(grad),
        _C.ptr(row_loss), _C.ptr(loss_sum), _C.ptr(w_sum), _C.ptr(nnz), None,
        _C.stream()))
    del keep
    ctx.set_materialize_grads(False)
    ctx.save_for_backward(grad, logits, labels, w, mask)
    ctx.args = (w_per_item, temperature, phi, lambda_weight)
    ctx.mark_non_differentiable(w_sum, nnz)
    return loss_sum, row_loss, w_sum, nnz

  @staticmethod
  def backward(ctx, g_sum, g_row, _gw, _gn):
    grad, logits, labels, w, mask = ctx.saved_tensors
    w_per_item, temperature, phi, lambda_weight = ctx.args
    out = None
    if g_row is None:
      if g_sum is not None:
        out = grad * g_sum.reshape(-1, 1)
    else:
      # Non-uniform upstream gradient per row (reduction NONE): rerun K1 with the
      # row weights scaled by the upstream gradient; W_ij is linear in w_i.
      b, n = logits.shape
      scale = g_row if g_sum is None else g_row + g_sum.reshape(-1, 1)
      if w is None:
        w_eff = scale.contiguous()
      else:
        w_eff = (scale * (w if w_per_item else w.reshape(-1, 1))).contiguous()
      out = torch.empty_like(logits)
      dummy = torch.empty(b, dtype=torch.float32, device=logits.device)
      cfg, keep = _lambda_cfg(lambda_weight, labels)
      _C.check(_C.lib.tfr_pairwise_loss_fwd_bwd(
          _C.ptr(logits), _C.ptr(labels), _C.ptr(w_eff), 1, _C.ptr(mask), b, n,
          float(temperature), phi, _byref(cfg), 1.0, _C.ptr(out), None,
          _C.ptr(dummy), None, None, None, _C.stream()))
      del keep
    return out, None, None, None, None, None, None, None


class _ListwiseFn(torch.autograd.Function):
  """loss[B], weight[B] = K2 / K3 (kind: 'ndcg' | 'mrr' | 'softmax')."""

  @staticmethod
  def forward(ctx, logits, labels, w, w_per_item, mask, temperature, kind,
              lambda_weight):
    b, n = logits.shape
    dev = logits.device
    grad = torch.empty_like(logits)
    loss = torch.empty(b, dtype=torch.float32, device=dev)
    weight = torch.empty_like(loss)
    if kind == 'softmax':
      cfg, keep = _lambda_cfg(lambda_weight, labels)
      _C.check(_C.lib.tfr_softmax_loss_fwd_bwd(
          _C.ptr(logits), _C.ptr(labels), _C.ptr(w), w_per_item, _C.ptr(mask),
          b, n, float(temperature), _byref(cfg), 1.0, 0, _C.ptr(grad),
          _C.ptr(loss), _C.ptr(weight), _C.stream()))
      del keep
    else:
      _C.check(_C.lib.tfr_approx_loss_fwd_bwd(
          _C.ptr(logits), _C.ptr(labels), _C.ptr(w), w_per_item, _C.ptr(mask),
          b, n, float(temperature), 0 if kind == 'ndcg' else 1, 1.0, 0,
          _C.ptr(grad), _C.ptr(loss), _C.ptr(weight), _C.stream()))
    ctx.set_materialize_grads(False)
    ctx.save_for_backward(grad)
    ctx.mark_non_differentiable(weight)
    return loss, weight

  @staticmethod
  def backward(ctx, g_loss, _gw):
    grad, = ctx.saved_tensors
    out = None if g_loss is None else grad * g_loss.reshape(-1, 1)
    return out, None, None, None, None, None, None, None


# ----------------------------------------------------------------------------
# _RankingLoss (losses_impl.py:652-860)
# ----------------------------------------------------------------------------
class _RankingLoss(object):

  def __init__(self, name=None, lambda_weight=None, temperature=1.0,
               ragged=False):
    self._name = name
    self._lambda_weight = lambda_weight
    self._temperature = temperature
    self._ragged = ragged

  @property
  def name(self):
    return self._name

  def _densify(self, labels, logits, weights, mask):
    """ragged=True: inputs are lists of per-list sequences (the torch stand-in for
    tf.RaggedTensor); they are padded the way utils.ragged_to_dense does
    (utils.py:421-443) and the mask argument is ignored, as in the reference."""
    if not self._ragged:
      return labels, logits, weights, mask
    from ranking_b200 import utils as tfr_utils
    return tfr_utils.ragged_to_dense(labels, logits, weights)

  def get_logits(self, logits):
    """losses_impl.py:773-785."""
    return _as_f32(logits, what='logits') / self._temperature

  def normalize_weights(self, labels, weights):
    """losses_impl.py:745-766."""
    if self._ragged:
      labels, _, weights, _ = self._densify(labels, None, weights, None)
    return self._normalize_weights_impl(_as_f32(labels, what='labels'), weights)

  def _normalize_weights_impl(self, labels, weights):
    return 1.0 if weights is None else weights


class _PairwiseLoss(_RankingLoss):
  """losses_impl.py:863-930."""
  _phi = None

  def _run(self, labels, logits, weights, mask, temperature):
    labels, logits, weights, mask = self._densify(labels, logits, weights, mask)
    labels, logits = _prep_2d(labels, logits)
    w, wpi = _prep_weights(weights, logits)
    m = _prep_mask(mask, logits)
    return _PairwiseFn.apply(logits, labels, w, wpi, m, temperature, self._phi,
                             self._lambda_weight)

  def compute(self, labels, logits, weights, reduction, mask=None):
    """losses_impl.py:787-814 over [B, N, N] pair losses, reduced per
    tf.compat.v1.losses.compute_weighted_loss."""
    loss_sum, _, w_sum, nnz = self._run(labels, logits, weights, mask,
                                        self._temperature)
    total = loss_sum.sum()
    if reduction == Reduction.SUM:
      return total
    if reduction == Reduction.MEAN:
      return _safe_div(total, w_sum.sum())
    if reduction == Reduction.SUM_BY_NONZERO_WEIGHTS:
      return _safe_div(total, nnz.sum())
    if reduction == Reduction.SUM_OVER_BATCH_SIZE:
      b, n = loss_sum.shape[0], torch.as_tensor(logits).shape[1]
      return total / float(b * n * n)
    raise ValueError('reduction %r is not supported for pairwise losses (the '
                     '[B, N, N] loss tensor is never materialised)' % (reduction,))

  def compute_per_list(self, labels, logits, weights, mask=None):
    """losses_impl.py:886-915 (no temperature, as in the reference)."""
    loss_sum, _, w_sum, _ = self._run(labels, logits, weights, mask, 1.0)
    return _safe_div(loss_sum, w_sum), w_sum

  def compute_row_sums(self, labels, logits, weights):
    """sum_j loss_ij * W_ij per item: what keras/losses.py:324-335 reduces."""
    return self._run(labels, logits, weights, None, self._temperature)[1]

  def _normalize_weights_impl(self, labels, weights):
    """losses_impl.py:917-930: [B, N, 1] row-item weights."""
    w = 1. if weights is None else _as_f32(weights, labels.device, 'weights')
    w = torch.where(labels >= 0, torch.ones_like(labels) * w,
                    torch.zeros_like(labels))
    return w.unsqueeze(2)


class PairwiseLogisticLoss(_PairwiseLoss):
  """losses_impl.py:933-940."""
  _phi = _C.PHI_LOGISTIC


class PairwiseHingeLoss(_PairwiseLoss):
  """losses_impl.py:943-948."""
  _phi = _C.PHI_HINGE


class PairwiseSoftZeroOneLoss(_PairwiseLoss):
  """losses_impl.py:951-958."""
  _phi = _C.PHI_SOFT_ZERO_ONE


class PairwiseMSELoss(_PairwiseLoss):
  """losses_impl.py:961-998."""
  _phi = _C.PHI_MSE


class _ListwiseLoss(_RankingLoss):
  """losses_impl.py:1001-1033."""
  _kind = None

  def _run(self, labels, logits, weights, mask, temperature):
    labels, logits, weights, mask = self._densify(labels, logits, weights, mask)
    labels, logits = _prep_2d(labels, logits)
    w, wpi = _prep_weights(weights, logits)
    m = _prep_mask(mask, logits)
    return _ListwiseFn.apply(logits, labels, w, wpi, m, temperature, self._kind,
                             self._lambda_weight)

  def compute(self, labels, logits, weights, reduction, mask=None):
    losses, w = self._run(labels, logits, weights, mask, self._temperature)
    return _reduce_lists(losses, w, reduction)

  def compute_per_list(self, labels, logits, weights, mask=None):
    """losses_impl.py:1017-1033 (no temperature, as in the reference)."""
    return self._run(labels, logits, weights, mask, 1.0)

  def _normalize_weights_impl(self, labels, weights):
    """losses_impl.py:1004-1015: sum(w * l) / sum(l) per list, [B, 1]."""
    if weights is None:
      return 1.0
    w = _as_f32(weights, labels.device, 'weights')
    lab = torch.where(labels >= 0, labels, torch.zeros_like(labels))
    return _safe_div((w * lab).sum(1, keepdim=True), lab.sum(1, keepdim=True))


def _reduce_lists(losses, weights, reduction):
  total = (losses * weights).sum()
  if reduction == Reduction.NONE:
    return losses * weights
  if reduction == Reduction.SUM:
    return total
  if reduction == Reduction.MEAN:
    return _safe_div(total, weights.sum())
  if reduction == Reduction.SUM_BY_NONZERO_WEIGHTS:
    return _safe_div(total, (weights != 0).to(losses.dtype).sum())
  if reduction == Reduction.SUM_OVER_BATCH_SIZE:
    return total / float(losses.numel())
  raise ValueError('bad reduction %r' % (reduction,))


class SoftmaxLoss(_ListwiseLoss):
  """losses_impl.py:1119-1197."""
  _kind = 'softmax'

  def compute_per_list(self, labels, logits, weights, mask=None):
    """losses_impl.py:1179-1189 (this one does apply the temperature)."""
    return self._run(labels, logits, weights, mask, self._temperature)


class ApproxNDCGLoss(_ListwiseLoss):
  """losses_impl.py:1579-1603."""
  _kind = 'ndcg'

  def __init__(self, name=None, lambda_weight=None, temperature=0.1,
               ragged=False):
    super().__init__(name, lambda_weight, temperature, ragged)


class ApproxMRRLoss(_ListwiseLoss):
  """losses_impl.py:1606-1632."""
  _kind = 'mrr'

  def __init__(self, name=None, lambda_weight=None, temperature=0.1,
               ragged=False):
    super().__init__(name, lambda_weight, temperature, ragged)


# ----------------------------------------------------------------------------
# Pointwise losses + UniqueSoftmax / ListMLE  (tfr_misc_loss_fwd_bwd, K3b)
# ----------------------------------------------------------------------------
_MISC = {'sigmoid_ce': 0, 'mean_squared': 1, 'unique_softmax': 2, 'list_mle': 3}


class _MiscFn(torch.autograd.Function):
  """(loss[B], weight[B], nonzero[B], row[B, N]) from one K3b launch.  Pointwise
  kinds: loss = sum_i row, row_i = loss_i * w_i.  Listwise kinds: row is None."""

  @staticmethod
  def forward(ctx, logits, labels, w, w_per_item, mask, temperature, kind,
              rank_weight, order_scores=None, topk=0):
    b, n = logits.shape
    dev = logits.device
    grad = torch.empty_like(logits)
    loss = torch.empty(b, dtype=torch.float32, device=dev)
    weight = torch.empty_like(loss)
    pointwise = kind in ('sigmoid_ce', 'mean_squared')
    nonzero = torch.empty_like(loss) if pointwise else None
    row = torch.empty_like(logits) if pointwise else None
    _C.check(_C.lib.tfr_misc_loss_fwd_bwd(
        _C.ptr(logits), _C.ptr(labels), _C.ptr(w), w_per_item, _C.ptr(mask), b, n,
        float(temperature), _MISC[kind], _C.ptr(rank_weight), _C.ptr(order_scores),
        int(topk or 0), 1.0, _C.ptr(grad), _C.ptr(row), _C.ptr(loss), _C.ptr(weight),
        _C.ptr(nonzero), _C.stream()))
    ctx.set_materialize_grads(False)
    ctx.save_for_backward(grad)
    ctx.mark_non_differentiable(weight)
    if pointwise:
      ctx.mark_non_differentiable(nonzero)
      return loss, weight, nonzero, row
    return loss, weight

  @staticmethod
  def backward(ctx, g_loss, _gw, *rest):
    grad, = ctx.saved_tensors
    out = None
    if g_loss is not None:
      out = grad * g_loss.reshape(-1, 1)
    if len(rest) == 2 and rest[1] is not None:     # d row_i / d s_i = grad_i
      out = grad * rest[1] if out is None else out + grad * rest[1]
    return out, None, None, None, None, None, None, None, None, None


class _PointwiseLoss(_RankingLoss):
  """losses_impl.py:1284-1321."""
  _kind = None

  def _run(self, labels, logits, weights, mask, temperature):
    labels, logits, weights, mask = self._densify(labels, logits, weights, mask)
    labels, logits = _prep_2d(labels, logits)
    w, wpi = _prep_weights(weights, logits)
    m = _prep_mask(mask, logits)
    return _MiscFn.apply(logits, labels, w, wpi, m, temperature, self._kind, None)

  def compute(self, labels, logits, weights, reduction, mask=None):
    loss, weight, nonzero, row = self._run(labels, logits, weights, mask,
                                           self._temperature)
    if reduction == Reduction.NONE:
      return row
    total = loss.sum()
    if reduction == Reduction.SUM:
      return total
    if reduction == Reduction.MEAN:
      return _safe_div(total, weight.sum())
    if reduction == Reduction.SUM_BY_NONZERO_WEIGHTS:
      return _safe_div(total, nonzero.sum())
    if reduction == Reduction.SUM_OVER_BATCH_SIZE:
      return total / float(row.numel())
    raise ValueError('bad reduction %r' % (reduction,))

  def compute_per_list(self, labels, logits, weights, mask=None):
    """losses_impl.py:1295-1321 (no temperature, as in the reference)."""
    loss, weight, _, _ = self._run(labels, logits, weights, mask, 1.0)
    return _safe_div(loss, weight), weight

  def compute_weighted_rows(self, labels, logits, weights):
    """[B, N] loss_i * mask_i * normalised weight: the Keras `call` x sample_weight."""
    return self._run(labels, logits, weights, None, self._temperature)[3]

  def _normalize_weights_impl(self, labels, weights):
    """losses_impl.py:1287-1293."""
    w = 1.0 if weights is None else _as_f32(weights, labels.device, 'weights')
    return torch.where(labels >= 0, torch.ones_like(labels) * w,
                       torch.zeros_like(labels))


class SigmoidCrossEntropyLoss(_PointwiseLoss):
  """losses_impl.py:1425-1446."""
  _kind = 'sigmoid_ce'

  def __init__(self, name=None, temperature=1.0, ragged=False):
    super().__init__(name, None, temperature, ragged)


class MeanSquaredLoss(_PointwiseLoss):
  """losses_impl.py:1449-1469 (temperature is not used)."""
  _kind = 'mean_squared'

  def __init__(self, name=None, ragged=False):
    super().__init__(name, None, 1.0, ragged)


class ListMLELambdaWeight(_LambdaWeight):
  """losses_impl.py:457-480."""

  def __init__(self, rank_discount_fn):
    self._rank_discount_fn = rank_discount_fn

  def individual_weights(self, labels, ranks):
    labels = torch.as_tensor(labels)
    return torch.ones_like(labels) * self._rank_discount_fn(
        torch.as_tensor(ranks).to(labels.dtype))

  def rank_table(self, n, device):
    """Discount of ranks 1..n as the [n] table the kernel reads."""
    r = torch.arange(1, n + 1, dtype=torch.float32, device=device)
    return (torch.ones_like(r) * self._rank_discount_fn(r)).float().contiguous()


class _MiscListwiseLoss(_ListwiseLoss):
  """UniqueSoftmax / ListMLE share the listwise plumbing of K2/K3."""

  def _run(self, labels, logits, weights, mask, temperature):
    labels, logits, weights, mask = self._densify(labels, logits, weights, mask)
    labels, logits = _prep_2d(labels, logits)
    w, wpi = _prep_weights(weights, logits)
    m = _prep_mask(mask, logits)
    table = None
    if self._kind == 'list_mle' and isinstance(self._lambda_weight,
                                               ListMLELambdaWeight):
      table = self._lambda_weight.rank_table(logits.shape[1], logits.device)
    return _MiscFn.apply(logits, labels, w, wpi, m, temperature, self._kind, table)


class UniqueSoftmaxLoss(_MiscListwiseLoss):
  """losses_impl.py:1250-1281."""
  _kind = 'unique_softmax'


class ListMLELoss(_MiscListwiseLoss):
  """losses_impl.py:1541-1576.  Label ties are ordered by index (the reference
  shuffles them randomly with a fixed op seed); invalid items come last."""
  _kind = 'list_mle'


# ----------------------------------------------------------------------------
# CircleLoss / NeuralSort losses  (tfr_extra_loss_fwd_bwd, K3c)
# ----------------------------------------------------------------------------
_EXTRA = {'circle': 0, 'neural_sort_ce': 1, 'neural_sort_ndcg': 2}


class _ExtraFn(torch.autograd.Function):
  """(loss[B], weight[B]) from one K3c launch; the gradient is produced by the same launch."""

  @staticmethod
  def forward(ctx, logits, labels, w, w_per_item, mask, temperature, kind, p0, p1):
    b, n = logits.shape
    grad = torch.empty_like(logits)
    loss = torch.empty(b, dtype=torch.float32, device=logits.device)
    weight = torch.empty_like(loss)
    _C.check(_C.lib.tfr_extra_loss_fwd_bwd(
        _C.ptr(logits), _C.ptr(labels), _C.ptr(w), w_per_item, _C.ptr(mask), b, n,
        float(temperature), _EXTRA[kind], float(p0), float(p1), 1.0, _C.ptr(grad),
        _C.ptr(loss), _C.ptr(weight), _C.stream()))
    ctx.set_materialize_grads(False)
    ctx.save_for_backward(grad)
    ctx.mark_non_differentiable(weight)
    return loss, weight

  @staticmethod
  def backward(ctx, g_loss, _gw):
    grad, = ctx.saved_tensors
    out = None if g_loss is None else grad * g_loss.reshape(-1, 1)
    return out, None, None, None, None, None, None, None, None


class _ExtraListwiseLoss(_ListwiseLoss):
  _p0 = 0.0
  _p1 = 0.0

  def _run(self, labels, logits, weights, mask, temperature):
    labels, logits, weights, mask = self._densify(labels, logits, weights, mask)
    labels, logits = _prep_2d(labels, logits)
    w, wpi = _prep_weights(weights, logits)
    m = _prep_mask(mask, logits)
    return _ExtraFn.apply(logits, labels, w, wpi, m, temperature, self._kind, self._p0,
                          self._p1)


class CircleLoss(_ExtraListwiseLoss):
  """losses_impl.py:1036-1116.  Scores are clipped to [0, 1] (`get_logits`, :1079-1082);
  a list without a valid pair has weight 0 / 0 = NaN, as in the reference."""
  _kind = 'circle'

  def __init__(self, name=None, lambda_weight=None, gamma=64, margin=0.25, ragged=False):
    super().__init__(name, lambda_weight, 1.0, ragged)
    self._gamma = gamma
    self._margin = margin
    self._p0 = float(gamma)
    self._p1 = float(margin)

  def get_logits(self, logits):
    return torch.clamp(logits, 0., 1.)


class NeuralSortCrossEntropyLoss(_ExtraListwiseLoss):
  """losses_impl.py:1635-1675."""
  _kind = 'neural_sort_ce'


class NeuralSortNDCGLoss(_ExtraListwiseLoss):
  """losses_impl.py:1678-1708 (PiRank NDCG)."""
  _kind = 'neural_sort_ndcg'


# ----------------------------------------------------------------------------
# GumbelSampler (losses_impl.py:540-649)
# ----------------------------------------------------------------------------
class _GumbelFn(torch.autograd.Function):

  @staticmethod
  def forward(ctx, logits, labels, sample_size, temperature, seed):
    b, n = logits.shape
    out = torch.empty(b * sample_size, n, dtype=torch.float32, device=logits.device)
    _C.check(_C.lib.tfr_gumbel_sample(
        _C.ptr(logits), _C.ptr(labels), b, n, sample_size, float(temperature), seed, 0,
        _C.ptr(out), None, None, _C.stream()))
    ctx.save_for_backward(logits, labels)
    ctx.cfg = (sample_size, float(temperature), seed)
    return out

  @staticmethod
  def backward(ctx, g_out):
    logits, labels = ctx.saved_tensors
    sample_size, temperature, seed = ctx.cfg
    b, n = logits.shape
    gin = torch.empty_like(logits)
    g_out = g_out.contiguous()
    _C.check(_C.lib.tfr_gumbel_sample(
        _C.ptr(logits), _C.ptr(labels), b, n, sample_size, temperature, seed, 0, None,
        _C.ptr(g_out), _C.ptr(gin), _C.stream()))
    return gin, None, None, None, None


class GumbelSampler(object):
  """losses_impl.py:540-645.  The uniforms are a counter hash of (seed, element)
  (include/tfr_b200.h, tfr_gumbel_sample); `seed=None` draws a fresh base seed and
  every `sample` call advances a counter, so consecutive calls differ like the
  reference's stateful `tf.random.uniform`."""

  def __init__(self, name=None, sample_size=8, temperature=1.0, seed=None,
               ragged=False):
    self._ragged = ragged
    self._name = name
    self._sample_size = int(sample_size)
    self._temperature = temperature
    self._seed = seed
    self._base = int(seed if seed is not None else torch.seed()) & 0xFFFFFFFF
    self._calls = 0

  def next_seed(self):
    self._calls += 1
    return (self._base << 32) | (self._calls & 0xFFFFFFFF)

  def expand(self, labels, weights):
    """Tiled labels [B*S, N] and weights ([B*S, 1] or [B*S, N])."""
    s = self._sample_size
    b, n = labels.shape
    ex_labels = labels.unsqueeze(1).expand(b, s, n).reshape(b * s, n).contiguous()
    ex_w = None
    if weights is not None:
      w = _as_f32(weights, labels.device, 'weights')
      if w.dim() == 0:
        w = w.expand(b)
      if w.dim() == 1:
        w = w.reshape(b, 1)
      ex_w = w.unsqueeze(1).expand(b, s, w.shape[1]).reshape(b * s, -1).contiguous()
    return ex_labels, ex_w

  def sample(self, labels, logits, weights=None):
    """With ragged=True the inputs are lists of per-list sequences and the outputs
    are DENSE padded tensors (label -1), which every loss here accepts."""
    if self._ragged:
      from ranking_b200 import utils as tfr_utils
      labels, logits, weights, _ = tfr_utils.ragged_to_dense(labels, logits, weights)
    labels, logits = _prep_2d(labels, logits)
    ex_labels, ex_w = self.expand(labels, weights)
    sampled = _GumbelFn.apply(logits, labels, self._sample_size, self._temperature,
                              self.next_seed())
    return ex_labels, sampled, ex_w


# ----------------------------------------------------------------------------
# OrdinalLoss (losses_impl.py:1850-1918)
# ----------------------------------------------------------------------------
class _OrdinalFn(torch.autograd.Function):

  @staticmethod
  def forward(ctx, logits, labels, w, w_per_item, mask, temperature, use_fraction):
    b, n, k = logits.shape
    dev = logits.device
    grad = torch.empty_like(logits)
    loss = torch.empty(b, dtype=torch.float32, device=dev)
    weight = torch.empty_like(loss)
    nonzero = torch.empty_like(loss)
    row = torch.empty(b, n, dtype=torch.float32, device=dev)
    _C.check(_C.lib.tfr_ordinal_loss_fwd_bwd(
        _C.ptr(logits), _C.ptr(labels), _C.ptr(w), w_per_item, _C.ptr(mask), b, n, k,
        float(temperature), int(bool(use_fraction)), 1.0, _C.ptr(grad), _C.ptr(row),
        _C.ptr(loss), _C.ptr(weight), _C.ptr(nonzero), _C.stream()))
    ctx.set_materialize_grads(False)
    ctx.save_for_backward(grad)
    ctx.mark_non_differentiable(weight, nonzero)
    return loss, weight, nonzero, row

  @staticmethod
  def backward(ctx, g_loss, _gw, _gn, g_row):
    grad, = ctx.saved_tensors
    out = None
    if g_loss is not None:
      out = grad * g_loss.reshape(-1, 1, 1)
    if g_row is not None:
      out = grad * g_row.unsqueeze(2) if out is None else out + grad * g_row.unsqueeze(2)
    return out, None, None, None, None, None, None


class OrdinalLoss(_PointwiseLoss):
  """losses_impl.py:1850-1918: logits [B, N, ordinal_size]."""

  def __init__(self, name=None, ordinal_size=1, temperature=1.0, ragged=False,
               use_fraction_label=False):
    super().__init__(name, None, temperature, ragged)
    self._ordinal_size = ordinal_size
    self._use_fraction_label = use_fraction_label

  def _run(self, labels, logits, weights, mask, temperature):
    labels, logits, weights, mask = self._densify(labels, logits, weights, mask)
    logits = _as_f32(logits, what='logits')
    if logits.dim() != 3:
      raise ValueError('Predictions for ordinal loss must have rank 3.')
    if logits.shape[-1] != self._ordinal_size:
      raise ValueError(
          'The last dimension of logits must be the number of ordinal levels '
          '{}, the actual dimension is {}.'.format(self._ordinal_size,
                                                   logits.shape[-1]))
    labels = _as_f32(labels, logits.device, 'labels')
    if labels.shape != logits.shape[:2]:
      raise ValueError('labels must have shape [batch_size, list_size]')
    w, wpi = _prep_weights(weights, labels)
    m = _prep_mask(mask, labels)
    return _OrdinalFn.apply(logits, labels, w, wpi, m, temperature,
                            self._use_fraction_label)


# ----------------------------------------------------------------------------
# ClickEMLoss / MixtureEMLoss  (tfr_click_em_loss_fwd_bwd / tfr_mixture_em_loss_fwd_bwd, K3d)
# ----------------------------------------------------------------------------
class _ClickEMFn(torch.autograd.Function):
  """(loss[B], weight[B], nonzero[B], row[B, N]) of ClickEM from one K3d launch over the
  [B, N, 2] logits (stride 2); the gradient is produced by the same launch."""

  @staticmethod
  def forward(ctx, logits, labels, w, w_per_item, mask, temperature, exam_w, rel_w):
    b, n, _ = logits.shape
    dev = logits.device
    grad = torch.empty_like(logits)
    loss = torch.empty(b, dtype=torch.float32, device=dev)
    weight = torch.empty_like(loss)
    nonzero = torch.empty_like(loss)
    row = torch.empty(b, n, dtype=torch.float32, device=dev)
    base = logits.data_ptr()
    gbase = grad.data_ptr()
    _C.check(_C.lib.tfr_click_em_loss_fwd_bwd(
        base, base + 4, 2, _C.ptr(labels), _C.ptr(w), w_per_item, _C.ptr(mask), b, n,
        float(temperature), float(exam_w), float(rel_w), 1.0, gbase, gbase + 4, _C.ptr(row),
        _C.ptr(loss), _C.ptr(weight), _C.ptr(nonzero), _C.stream()))
    ctx.set_materialize_grads(False)
    ctx.save_for_backward(grad)
    ctx.mark_non_differentiable(weight, nonzero)
    return loss, weight, nonzero, row

  @staticmethod
  def backward(ctx, g_loss, _gw, _gn, g_row):
    # d loss[b] / d logits = grad; d row[b, i] / d logits[b, i, :] = grad[b, i, :]
    grad, = ctx.saved_tensors
    out = None
    if g_loss is not None:
      out = grad * g_loss.reshape(-1, 1, 1)
    if g_row is not None:
      out = grad * g_row.unsqueeze(2) if out is None else out + grad * g_row.unsqueeze(2)
    return out, None, None, None, None, None, None, None


def _prep_3d(labels, logits, what):
  logits = _as_f32(logits, what='logits')
  if logits.dim() != 3:
    raise ValueError('Predictions for %s must have rank 3.' % what)
  labels = _as_f32(labels, logits.device, 'labels')
  if labels.shape != logits.shape[:2]:
    raise ValueError('labels must have shape [batch_size, list_size]; got %s for logits %s' %
                     (tuple(labels.shape), tuple(logits.shape)))
  return labels, logits


class ClickEMLoss(_PointwiseLoss):
  """losses_impl.py:1324-1422: logits [B, N, 2], [..., 0] the examination logits and
  [..., 1] the relevance logits; labels are clicks (>= 1 clicked, < 0 padding).
  `compute_unreduced_loss` returns losses that are 0 on invalid items (the reference's
  value there is finite but always multiplied by a zero weight)."""

  def __init__(self, name=None, temperature=1.0, exam_loss_weight=1.0, rel_loss_weight=1.0,
               ragged=False):
    super().__init__(name, None, temperature, ragged)
    self._exam_loss_weight = exam_loss_weight
    self._rel_loss_weight = rel_loss_weight

  def _run(self, labels, logits, weights, mask, temperature):
    labels, logits, weights, mask = self._densify(labels, logits, weights, mask)
    labels, logits = _prep_3d(labels, logits, 'click EM loss')
    if logits.shape[-1] != 2:
      raise ValueError('The last dimension of logits must be 2 (examination and relevance '
                       'logits), the actual dimension is {}.'.format(logits.shape[-1]))
    w, wpi = _prep_weights(weights, labels)
    m = _prep_mask(mask, labels)
    return _ClickEMFn.apply(logits, labels, w, wpi, m, temperature, self._exam_loss_weight,
                            self._rel_loss_weight)

  def compute_unreduced_loss(self, labels, logits, mask=None):
    """losses_impl.py:709-726: (losses [B, N], loss weights = mask [B, N])."""
    row = self._run(labels, logits, None, mask, 1.0)[3]
    if self._ragged:
      mask = self._densify(labels, None, None, None)[3]
    elif mask is None:
      mask = _as_f32(labels, row.device, 'labels') >= 0
    return row, torch.as_tensor(mask, device=row.device).to(torch.float32)


class _MixtureEMFn(torch.autograd.Function):
  """(loss[B], weight[B]) of MixtureEM from one K3d launch over [B, N, M] logits."""

  @staticmethod
  def forward(ctx, logits, labels, w, w_per_item, mask, temperature, alpha):
    b, n, m = logits.shape
    grad = torch.empty_like(logits)
    loss = torch.empty(b, dtype=torch.float32, device=logits.device)
    weight = torch.empty_like(loss)
    _C.check(_C.lib.tfr_mixture_em_loss_fwd_bwd(
        _C.ptr(logits), _C.ptr(labels), _C.ptr(w), w_per_item, _C.ptr(mask), b, n, m,
        float(temperature), float(alpha), 1.0, _C.ptr(grad), _C.ptr(loss), _C.ptr(weight),
        _C.stream()))
    ctx.set_materialize_grads(False)
    ctx.save_for_backward(grad)
    ctx.mark_non_differentiable(weight)
    return loss, weight

  @staticmethod
  def backward(ctx, g_loss, _gw):
    grad, = ctx.saved_tensors
    out = None if g_loss is None else grad * g_loss.reshape(-1, 1, 1)
    return out, None, None, None, None, None, None


class MixtureEMLoss(_ListwiseLoss):
  """losses_impl.py:1472-1538: logits [B, N, model_num] (1 <= model_num <= 32), one column
  per mixed click model; labels are clicks."""

  def __init__(self, name=None, temperature=1.0, alpha=1.0, ragged=False):
    super().__init__(name, None, temperature, ragged)
    self._alpha = alpha

  def _run(self, labels, logits, weights, mask, temperature):
    labels, logits, weights, mask = self._densify(labels, logits, weights, mask)
    labels, logits = _prep_3d(labels, logits, 'mixture EM loss')
    w, wpi = _prep_weights(weights, labels)
    m = _prep_mask(mask, labels)
    return _MixtureEMFn.apply(logits, labels, w, wpi, m, temperature, self._alpha)

  def compute_unreduced_loss(self, labels, logits, mask=None):
    """losses_impl.py:709-726: (losses [B, 1], loss weights [B, 1])."""
    loss, weight = self._run(labels, logits, None, mask, 1.0)
    return loss.unsqueeze(1), weight.unsqueeze(1)


# ----------------------------------------------------------------------------
# CoupledRankDistilLoss (losses_impl.py:1984-2116)
# ----------------------------------------------------------------------------
class CoupledRankDistilLoss(_ListwiseLoss):
  """Cross entropy between the top-k Plackett-Luce models of the labels (teacher) and
  the logits (student): `sample_size` permutations are drawn from the teacher with
  Gumbel noise (counter hash, see tfr_gumbel_sample mode 1) and each one is a top-k
  ListMLE term on the student scores (K3b with `order_scores`)."""
  _kind = 'list_mle'

  def __init__(self, name=None, sample_size=8, topk=None, temperature=1.,
               ragged=False):
    super().__init__(name, None, temperature, ragged)
    self._sample_size = int(sample_size)
    self._topk = topk
    self._base = int(torch.seed()) & 0xFFFFFFFF
    self._calls = 0

  def seed(self, base):
    """Fixes the noise stream (tests / reproducible runs)."""
    self._base = int(base) & 0xFFFFFFFF
    self._calls = 0

  def _run(self, labels, logits, weights, mask, temperature):
    labels, logits, weights, mask = self._densify(labels, logits, weights, mask)
    labels, logits = _prep_2d(labels, logits)
    w, wpi = _prep_weights(weights, logits)
    m = _prep_mask(mask, logits)
    b, n = logits.shape
    s_ = self._sample_size
    self._calls += 1
    seed = (self._base << 32) | (self._calls & 0xFFFFFFFF)
    # the teacher's validity is the loss mask: pass masked labels as -1
    t_labels = labels if m is None else torch.where(m != 0, labels,
                                                    torch.full_like(labels, -1.))
    teacher = torch.empty(b * s_, n, dtype=torch.float32, device=logits.device)
    _C.check(_C.lib.tfr_gumbel_sample(
        None, _C.ptr(t_labels.contiguous()), b, n, s_, 1.0, seed, 1, _C.ptr(teacher), None,
        None, _C.stream()))
    rep = lambda t: None if t is None else t.repeat_interleave(s_, dim=0).contiguous()
    ex_w = None if w is None else (w.repeat_interleave(s_, dim=0).contiguous())
    loss, weight = _MiscFn.apply(rep(logits), rep(labels), ex_w, wpi, rep(m), temperature,
                                 'list_mle', None, teacher, self._topk or 0)
    # mean over the samples (:2113); the list weight is the same for every sample
    return loss.reshape(b, s_).mean(1), weight.reshape(b, s_)[:, 0]
