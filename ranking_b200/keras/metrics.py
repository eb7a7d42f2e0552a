"""The `tfr.keras.metrics` surface (keras/metrics.py) for NDCG and MRR.

Each metric is a running weighted mean (tf.keras.metrics.Mean semantics,
keras/metrics.py:156-193): state = (sum v*w, sum w) kept on the device;
`update_state(y_true, y_pred, sample_weight=None)`, `result()`,
`reset_state()`.  `default_keras_metrics()`-style groups of NDCG@k / MRR can be
evaluated with ONE kernel launch through `MetricGroup`.
"""
import torch

from ranking_b200 import dp

from ranking_b200 import metrics_impl
from ranking_b200.keras import utils


class RankingMetricKey(object):
  """keras/metrics.py:34-66."""
  MRR = 'mrr'
  ARP = 'arp'
  NDCG = 'ndcg'
  DCG = 'dcg'
  PRECISION = 'precision'
  MAP = 'map'
  PRECISION_IA = 'precision_ia'
  ORDERED_PAIR_ACCURACY = 'ordered_pair_accuracy'
  ALPHA_DCG = 'alpha_dcg'
  HITS = 'hits'


class _RankingMetric(object):
  """keras/metrics.py:156-200."""

  def __init__(self, name=None, dtype=None, ragged=False, **kwargs):
    self.name = name
    self._dtype = dtype or torch.float32
    self._ragged = ragged
    self._metric = None
    self._state = None   # device tensor [2] = (sum v*w, sum w)

  def reset_state(self):
    self._state = None

  reset_states = reset_state

  def update_state(self, y_true, y_pred, sample_weight=None):
    v, w = self._metric.compute(y_true, y_pred, sample_weight)
    upd = torch.stack([(v * w).sum(), w.sum()])
    self._state = upd if self._state is None else self._state + upd

  def all_reduce(self, group=None):
    """Data-parallel evaluation: SUM the (sum v*w, sum w) pair across ranks."""
    if self._state is None:   # a rank that saw no batch still has to enter the collective
      dev = 'cuda' if torch.cuda.is_available() else 'cpu'
      self._state = torch.zeros(2, dtype=torch.float32, device=dev)
    dp.all_reduce_sum_(self._state, group)

  def result(self):
    if self._state is None:
      return torch.zeros((), dtype=torch.float32)
    s = self._state
    return torch.where(s[1] != 0, s[0] / torch.where(s[1] != 0, s[1],
                                                     torch.ones_like(s[1])),
                       torch.zeros_like(s[0]))

  def __call__(self, y_true, y_pred, sample_weight=None):
    self.update_state(y_true, y_pred, sample_weight)
    return self.result()

  def get_config(self):
    return {'name': self.name, 'dtype': self._dtype, 'ragged': self._ragged}


class MRRMetric(_RankingMetric):
  """keras/metrics.py:203-266."""

  def __init__(self, name=None, topn=None, dtype=None, ragged=False, **kwargs):
    super().__init__(name=name, dtype=dtype, ragged=ragged, **kwargs)
    self._topn = topn
    self._metric = metrics_impl.MRRMetric(name=name, topn=topn, ragged=ragged)

  def get_config(self):
    config = super().get_config()
    config.update({'topn': self._topn})
    return config


class NDCGMetric(_RankingMetric):
  """keras/metrics.py:709-796."""

  def __init__(self, name=None, topn=None, gain_fn=None, rank_discount_fn=None,
               dtype=None, ragged=False, **kwargs):
    super().__init__(name=name, dtype=dtype, ragged=ragged, **kwargs)
    self._topn = topn
    self._gain_fn = gain_fn or utils.pow_minus_1
    self._rank_discount_fn = rank_discount_fn or utils.log2_inverse
    self._metric = metrics_impl.NDCGMetric(
        name=name, topn=topn, gain_fn=self._gain_fn,
        rank_discount_fn=self._rank_discount_fn, ragged=ragged)

  def get_config(self):
    config = super().get_config()
    config.update({'topn': self._topn, 'gain_fn': self._gain_fn,
                   'rank_discount_fn': self._rank_discount_fn})
    return config


class _TopnMetric(_RankingMetric):
  _impl = None

  def __init__(self, name=None, topn=None, dtype=None, ragged=False, **kwargs):
    super().__init__(name=name, dtype=dtype, ragged=ragged, **kwargs)
    self._topn = topn
    self._metric = self._impl(name=name, topn=topn, ragged=ragged)

  def get_config(self):
    config = super().get_config()
    config.update({'topn': self._topn})
    return config


class HitsMetric(_TopnMetric):
  """keras/metrics.py:269-331."""
  _impl = metrics_impl.HitsMetric


class RecallMetric(_TopnMetric):
  """keras/metrics.py:417-482."""
  _impl = metrics_impl.RecallMetric


class PrecisionMetric(_TopnMetric):
  """keras/metrics.py:485-551."""
  _impl = metrics_impl.PrecisionMetric


class MeanAveragePrecisionMetric(_TopnMetric):
  """keras/metrics.py:554-640."""
  _impl = metrics_impl.MeanAveragePrecisionMetric


class ARPMetric(_RankingMetric):
  """keras/metrics.py:334-414."""

  def __init__(self, name=None, dtype=None, ragged=False, **kwargs):
    super().__init__(name=name, dtype=dtype, ragged=ragged, **kwargs)
    self._metric = metrics_impl.ARPMetric(name=name, ragged=ragged)


class OPAMetric(_RankingMetric):
  """keras/metrics.py:948-1010."""

  def __init__(self, name=None, dtype=None, ragged=False, **kwargs):
    super().__init__(name=name, dtype=dtype, ragged=ragged, **kwargs)
    self._metric = metrics_impl.OPAMetric(name=name, ragged=ragged)


class DCGMetric(_RankingMetric):
  """keras/metrics.py:799-877."""

  def __init__(self, name=None, topn=None, gain_fn=None, rank_discount_fn=None,
               dtype=None, ragged=False, **kwargs):
    super().__init__(name=name, dtype=dtype, ragged=ragged, **kwargs)
    self._topn = topn
    self._gain_fn = gain_fn or utils.pow_minus_1
    self._rank_discount_fn = rank_discount_fn or utils.log2_inverse
    self._metric = metrics_impl.DCGMetric(
        name=name, topn=topn, gain_fn=self._gain_fn,
        rank_discount_fn=self._rank_discount_fn, ragged=ragged)

  def get_config(self):
    config = super().get_config()
    config.update({'topn': self._topn, 'gain_fn': self._gain_fn,
                   'rank_discount_fn': self._rank_discount_fn})
    return config


class PrecisionIAMetric(_TopnMetric):
  """keras/metrics.py:643-706: y_true [B, N, subtopic_size]."""
  _impl = metrics_impl.PrecisionIAMetric


class AlphaDCGMetric(_RankingMetric):
  """keras/metrics.py:1013-1107: y_true [B, N, subtopic_size]."""

  def __init__(self, name='alpha_dcg_metric', topn=None, alpha=0.5,
               rank_discount_fn=None, seed=None, dtype=None, ragged=False, **kwargs):
    super().__init__(name=name, dtype=dtype, ragged=ragged, **kwargs)
    self._topn = topn
    self._alpha = alpha
    self._rank_discount_fn = rank_discount_fn or utils.log2_inverse
    self._seed = seed
    self._metric = metrics_impl.AlphaDCGMetric(
        name=name, topn=topn, alpha=alpha, rank_discount_fn=self._rank_discount_fn,
        seed=seed, ragged=ragged)

  def get_config(self):
    config = super().get_config()
    config.update({'topn': self._topn, 'alpha': self._alpha,
                   'rank_discount_fn': self._rank_discount_fn, 'seed': self._seed})
    return config


_KEY_TO_CLS = {
    RankingMetricKey.PRECISION_IA: PrecisionIAMetric,
    RankingMetricKey.ALPHA_DCG: AlphaDCGMetric,
    RankingMetricKey.MRR: MRRMetric, RankingMetricKey.NDCG: NDCGMetric,
    RankingMetricKey.ARP: ARPMetric, RankingMetricKey.DCG: DCGMetric,
    RankingMetricKey.PRECISION: PrecisionMetric,
    RankingMetricKey.MAP: MeanAveragePrecisionMetric,
    RankingMetricKey.ORDERED_PAIR_ACCURACY: OPAMetric,
    RankingMetricKey.HITS: HitsMetric,
}
_ALL_KEYS = [v for k, v in vars(RankingMetricKey).items() if k.isupper()]


def get(key, name=None, dtype=None, topn=None, **kwargs):
  """keras/metrics.py:69-128."""
  if not isinstance(key, str):
    raise ValueError('Input `key` needs to be string.')
  metric_kwargs = {'name': name, 'dtype': dtype}
  if topn:
    metric_kwargs.update({'topn': topn})
  metric_kwargs.update(kwargs)
  if key in _KEY_TO_CLS:
    return _KEY_TO_CLS[key](**metric_kwargs)
  if key in _ALL_KEYS:
    raise ValueError('Unsupported metric: {} (not on the GPU hot path yet; see '
                     'DESIGN.md scope)'.format(key))
  raise ValueError('Unsupported metric: {}'.format(key))


def default_keras_metrics(**kwargs):
  """keras/metrics.py:131-153: the same eleven metrics as the reference.  For
  evaluation loops prefer `MetricGroup.default()`, which gets all of them from one
  kernel launch per batch (one sort instead of eleven)."""
  list_kwargs = [
      dict(key='ndcg', topn=topn, name='metric/ndcg_{}'.format(topn), **kwargs)
      for topn in [1, 3, 5, 10]
  ] + [
      dict(key='arp', name='metric/arp', **kwargs),
      dict(key='ordered_pair_accuracy', name='metric/ordered_pair_accuracy',
           **kwargs),
      dict(key='mrr', name='metric/mrr', **kwargs),
      dict(key='precision', name='metric/precision', **kwargs),
      dict(key='map', name='metric/map', **kwargs),
      dict(key='dcg', name='metric/dcg', **kwargs),
      dict(key='ndcg', name='metric/ndcg', **kwargs),
  ]
  return [get(**kw) for kw in list_kwargs]


class MetricGroup(object):
  """NDCG@k for several k, plus MRR, from ONE K4 launch per update.

  `default_keras_metrics()` in the reference builds one object per cut-off and
  each re-sorts the batch (SURVEY.md §8a a19); this evaluates them together.
  """

  def __init__(self, topns=(1, 3, 5, 10, None), gain_fn=None,
               rank_discount_fn=None, ext=(), cross_replica_weights=False,
               process_group=None):
    # cross_replica_weights: take the batch-average list weight of lists without relevant
    # items (metrics_impl.py:101-113) over ALL replicas' batches (one 2-float all-reduce
    # per update) instead of per replica: data-parallel evaluation then equals a single
    # device on the concatenated batch.
    self._cross = bool(cross_replica_weights)
    self._group = process_group
    self.topns = tuple(topns)
    self._gain_fn = gain_fn
    self._rank_discount_fn = rank_discount_fn
    self._ext = tuple(ext)   # extra metrics from the same launch (see `default`)
    self._ext_state = None   # per ext metric: (sum v*w [T or 1], sum w)
    self._state = None    # [2T + 2]: sum ndcg_t*w (T), sum mrr_t*w (T), sum w_ndcg, sum w_mrr

  @classmethod
  def default(cls, **kwargs):
    """All of `default_keras_metrics()` (keras/metrics.py:131-153) from one launch."""
    return cls(topns=(1, 3, 5, 10, None),
               ext=('arp', 'opa', 'precision', 'map', 'dcg'), **kwargs)

  def reset_state(self):
    self._state = None
    self._ext_state = None

  def update_state(self, y_true, y_pred, sample_weight=None):
    o = metrics_impl.rank_metrics(y_true, y_pred, sample_weight, None,
                                  self.topns, self._gain_fn,
                                  self._rank_discount_fn, ext=self._ext)
    if self._cross:
      o['ndcg_w'] = dp.cross_replica_list_weights(o['raw'], 'ndcg', self._group)
      o['mrr_w'] = dp.cross_replica_list_weights(o['raw'], 'mrr', self._group)
    if self._ext:
      parts = []
      for key in self._ext:
        if key in ('arp', 'opa'):
          v, w = o[key][:, 0:1], o[key][:, 1]
        elif key == 'dcg':
          w = o['ndcg_w']
          v = metrics_impl._safe_div(o['dcg'], w.unsqueeze(1))
        else:
          v, w = o[key], o['mrr_w']
        parts.append(torch.cat([(v * w.unsqueeze(1)).sum(0), w.sum().reshape(1)]))
      upd_ext = torch.cat(parts)
      self._ext_state = upd_ext if self._ext_state is None else self._ext_state + upd_ext
    upd = torch.cat([
        (o['ndcg'] * o['ndcg_w'].unsqueeze(1)).sum(0),
        (o['mrr'] * o['mrr_w'].unsqueeze(1)).sum(0),
        o['ndcg_w'].sum().reshape(1), o['mrr_w'].sum().reshape(1)])
    self._state = upd if self._state is None else self._state + upd

  def _zero_state(self, device=None):
    """A rank that saw no batch still has a state of the right width (all zeros), so that
    every rank enters the same collectives and `result()` works on an empty evaluation."""
    t = len(self.topns)
    if device is None:
      device = torch.device('cuda', torch.cuda.current_device()) if \
          torch.cuda.is_available() else torch.device('cpu')
    if self._state is None:
      self._state = torch.zeros(2 * t + 2, dtype=torch.float32, device=device)
    if self._ext and self._ext_state is None:
      width = sum((1 if k in ('arp', 'opa') else t) + 1 for k in self._ext)
      self._ext_state = torch.zeros(width, dtype=torch.float32, device=device)

  def all_reduce(self, group=None):
    self._zero_state()
    dp.all_reduce_sum_(self._state, group)
    if self._ext_state is not None:
      dp.all_reduce_sum_(self._ext_state, group)

  def result(self):
    t = len(self.topns)
    self._zero_state()
    s = self._state.double().cpu()
    out = {}
    if self._ext_state is not None:
      e = self._ext_state.double().cpu()
      names = {'arp': 'arp', 'opa': 'ordered_pair_accuracy', 'precision': 'precision',
               'map': 'map', 'dcg': 'dcg', 'recall': 'recall', 'hits': 'hits'}
      pos = 0
      for key in self._ext:
        width = 1 if key in ('arp', 'opa') else t
        den = e[pos + width]
        for i in range(width):
          k = self.topns[i] if width > 1 else None
          suffix = '' if not k else '_{}'.format(k)
          out['metric/' + names[key] + suffix] = float(e[pos + i] / den) if den else 0.0
        pos += width + 1
    for i, k in enumerate(self.topns):
      suffix = '' if not k else '_{}'.format(k)
      out['metric/ndcg' + suffix] = float(s[i] / s[2 * t]) if s[2 * t] else 0.0
      out['metric/mrr' + suffix] = float(s[t + i] / s[2 * t + 1]) if s[
          2 * t + 1] else 0.0
    return out
