"""Known-answer tests of ClickEMLoss and MixtureEMLoss, transcribed from the reference's own
tests (losses_impl_test.py:1537-1660, keras/losses_test.py:327-372, 1378-1420) and the
docstring examples (keras/losses.py:1359-1371, 1435-1447).  Run against the CPU oracle
(oracle/click.py) and, under `-m gpu`, the CUDA kernels (csrc/loss_click.cu).  The last
test runs the click EM recovery experiment of tests/_click_refs.py through the oracle and
fixes the thresholds the GPU trainer is held to (tests/test_click_em_gpu.py)."""
import math

import numpy as np
import pytest
import torch

import _click_refs as CR

# Recovery thresholds, set from the oracle run below (measured: max |relative propensity -
# eta| = 0.038 over p = 1..9; NDCG@5 click EM 0.9996 vs naive 0.904, a gap of 0.095) with a
# margin of about 2x.
TAU = 0.08
DELTA = 0.05


def _impl(api, name):
  if api.name == 'oracle':
    from oracle import click
    return getattr(click, name)
  return getattr(api.losses_impl, name)


def _keras(api, name):
  if api.name == 'oracle':
    from oracle import click
    return getattr(click, 'Keras' + name)
  return getattr(api.keras_losses, name)


def _sce(labels, logits):
  """losses_impl_test.py:111-117."""
  return sum(max(x, 0) - x * z + math.log(1 + math.exp(-abs(x))) for z, x in zip(labels, logits))


def _logodds_prob(logodds, alpha=1.0):
  """losses_impl_test.py:120-123 for one list."""
  return [math.exp(-alpha * (v - min(logodds))) for v in logodds]


def _mix(l1, l2, alpha=1.0):
  p = _logodds_prob([l1, l2], alpha)
  return (l1 * p[0] + l2 * p[1]) / (p[0] + p[1])


def _close(actual, expected, places):
  assert abs(float(torch.as_tensor(actual).detach().cpu()) - expected) <= 1.5 * 10 ** -places, (
      float(actual), expected)


CLICKS = [[1., 0, 0, 0]]
EXAM = [[3., 3, 4, 100]]
REL = [[3., 2, 1, 100]]
PE = [1., 0.705384, 0.93624, 0.5]     # P(exam | click) of losses_impl_test.py:1550
PR = [1., 0.259496, 0.046613, 0.5]


def _stack(api, a, b):
  return torch.stack([api.t(a), api.t(b)], 2)


def test_click_em_loss(api):
  """losses_impl_test.py:1539-1568; the posteriors are checked through the gradient:
  d loss / d e_i = sigmoid(e_i) - P(exam | click)_i (SUM reduction, T = 1)."""
  R = api.Reduction
  logits = _stack(api, EXAM, REL).requires_grad_()
  loss = _impl(api, 'ClickEMLoss')(name=None).compute(api.t(CLICKS), logits, None, R.SUM)
  _close(loss, _sce(PE, EXAM[0]) + _sce(PR, REL[0]), 5)
  loss.backward()
  sig = lambda v: 1. / (1. + math.exp(-v))   # noqa: E731
  want_e = [sig(e) - p for e, p in zip(EXAM[0], PE)]
  want_r = [sig(r) - p for r, p in zip(REL[0], PR)]
  got = logits.grad.detach().cpu().double()
  torch.testing.assert_close(got[0, :, 0], torch.tensor(want_e, dtype=torch.float64), atol=1e-5,
                             rtol=0)
  torch.testing.assert_close(got[0, :, 1], torch.tensor(want_r, dtype=torch.float64), atol=1e-5,
                             rtol=0)
  weighted = _impl(api, 'ClickEMLoss')(name='weighted', exam_loss_weight=2.0,
                                       rel_loss_weight=5.0)
  _close(weighted.compute(api.t(CLICKS), _stack(api, EXAM, REL), None, R.SUM),
         _sce(PE, EXAM[0]) * 2.0 + _sce(PR, REL[0]) * 5.0, 4)


def test_click_em_loss_invalid_labels_and_mask(api):
  """losses_impl_test.py:1570-1602."""
  R = api.Reduction
  fn = _impl(api, 'ClickEMLoss')(name=None)
  want = _sce([1., 0.93624, 0.5], [3., 4., 100.]) + _sce([1., 0.046613, 0.5], [3., 1., 100.])
  _close(fn.compute(api.t([[1., -1., 0., 0.]]), _stack(api, EXAM, REL), None, R.SUM), want, 5)
  mask = torch.tensor([[True, False, True, True]], device=api.device)
  _close(fn.compute(api.t([[1., 1., 0., 0.]]), _stack(api, EXAM, REL), None, R.SUM, mask),
         want, 5)


def test_mixture_em_loss(api):
  """losses_impl_test.py:1605-1660."""
  R = api.Reduction
  fn = _impl(api, 'MixtureEMLoss')(name=None)
  l1, l2 = _sce(CLICKS[0], EXAM[0]), _sce(CLICKS[0], REL[0])
  _close(fn.compute(api.t(CLICKS), _stack(api, EXAM, REL), None, R.SUM), _mix(l1, l2), 4)
  l1, l2 = _sce([1., 0., 0.], [3., 4., 100.]), _sce([1., 0., 0.], [3., 1., 100.])
  _close(fn.compute(api.t([[1., -1., 0., 0.]]), _stack(api, EXAM, REL), None, R.SUM),
         _mix(l1, l2), 5)
  mask = torch.tensor([[True, False, True, True]], device=api.device)
  _close(fn.compute(api.t([[1., 1., 0., 0.]]), _stack(api, EXAM, REL), None, R.SUM, mask),
         _mix(l1, l2), 5)


def test_keras_click_and_mixture_em(api):
  """keras/losses_test.py:327-372."""
  loss = _keras(api, 'ClickEMLoss')()
  _close(loss(api.t(CLICKS), _stack(api, EXAM, REL)) * 4., _sce(PE, EXAM[0]) + _sce(PR, REL[0]),
         5)
  loss = _keras(api, 'ClickEMLoss')(exam_loss_weight=2.0, rel_loss_weight=5.0)
  _close(loss(api.t(CLICKS), _stack(api, EXAM, REL)) * 4.,
         _sce(PE, EXAM[0]) * 2.0 + _sce(PR, REL[0]) * 5.0, 4)
  l1, l2 = _sce(CLICKS[0], EXAM[0]), _sce(CLICKS[0], REL[0])
  for alpha in (1.0, 0.1):
    loss = _keras(api, 'MixtureEMLoss')(alpha=alpha)
    _close(loss(api.t(CLICKS), _stack(api, EXAM, REL)), _mix(l1, l2, alpha), 4)


@pytest.mark.parametrize('name,dense,ragged', [('ClickEMLoss', 1.1462884, 1.0770882),
                                               ('MixtureEMLoss', 1.3198698, 1.909512)])
def test_docstring_examples(api, name, dense, ragged):
  """keras/losses.py:1359-1371, 1435-1447."""
  cls = _keras(api, name)
  _close(cls()(api.t([[1., 0.]]), api.t([[[0.6, 0.9], [0.8, 0.2]]])), dense, 6)
  y_true = [[1., 0.], [0., 1., 0.]]
  y_pred = [[[0.6, 0.9], [0.8, 0.2]], [[0.5, 0.9], [0.8, 0.2], [0.4, 0.8]]]
  _close(cls(ragged=True)(y_true, y_pred), ragged, 6)


def test_config_round_trip(api):
  """keras/losses_test.py:1378-1420 for ClickEMLoss, dense and ragged; the MixtureEMLoss
  config keeps lambda_weight and temperature (keras/losses.py:1484-1496) without using them."""
  cls = _keras(api, 'ClickEMLoss')
  scores = api.t([[1., 3., 2.], [1., 2., 3.]])
  labels = api.t([[0., 0., 1.], [0., 1., 2.]])
  loss = cls(exam_loss_weight=2.0, rel_loss_weight=5.0)
  again = cls.from_config(loss.get_config())
  assert again.get_config() == loss.get_config()
  y = torch.stack([scores, scores], 2)
  assert float(loss(labels, y)) == float(again(labels, y))
  loss = cls(ragged=True)
  again = cls.from_config(loss.get_config())
  assert again.get_config() == loss.get_config()
  r_scores = [[[1., 1.], [2., 2.], [4., 4.]], [[0., 0.], [2., 2.]]]
  r_labels = [[0., 2., 1.], [1., 0.]]
  assert float(loss(r_labels, r_scores)) == float(again(r_labels, r_scores))
  mix = _keras(api, 'MixtureEMLoss')(temperature=0.5, alpha=0.3)
  cfg = mix.get_config()
  assert cfg['temperature'] == 0.5 and cfg['alpha'] == 0.3 and 'lambda_weight' in cfg
  y3 = torch.stack([scores, 2 * scores], 2)
  assert float(mix(labels, y3)) == pytest.approx(
      float(_keras(api, 'MixtureEMLoss')(alpha=0.3)(labels, y3)), rel=1e-6)


def test_reductions_per_list_and_unreduced(api):
  """Every Reduction of `compute`, `compute_per_list` (no temperature) and
  `compute_unreduced_loss` agree with the per-item / per-list values."""
  R = api.Reduction
  g = torch.Generator().manual_seed(3)
  labels = torch.tensor([[1., 0., 0., -1.], [0., 0., 1., 1.], [0., 0., 0., 0.]])
  logits2 = torch.randn(3, 4, 2, generator=g)
  logits3 = torch.randn(3, 4, 3, generator=g)
  w = torch.rand(3, 4, generator=g) + 0.5
  dev = api.device
  ce = _impl(api, 'ClickEMLoss')(name=None, temperature=2.0)
  losses, lw = ce.compute_unreduced_loss(labels.to(dev), logits2.to(dev) / 2.0)
  nw = ce.normalize_weights(labels.to(dev), w.to(dev))
  rows = (losses * lw * nw).cpu().double()
  total = float(rows.sum())
  wsum = float((lw * nw).sum())
  nnz = float(((lw * nw) != 0).sum())
  want = {R.SUM: total, R.MEAN: total / wsum, R.SUM_BY_NONZERO_WEIGHTS: total / nnz,
          R.SUM_OVER_BATCH_SIZE: total / 12.}
  for red, v in want.items():
    _close(ce.compute(labels.to(dev), logits2.to(dev), w.to(dev), red), v, 5)
  none = ce.compute(labels.to(dev), logits2.to(dev), w.to(dev), R.NONE)
  torch.testing.assert_close(none.cpu().double(), rows, atol=1e-5, rtol=1e-5)
  pl, pw = ce.compute_per_list(labels.to(dev), (logits2 / 2.0).to(dev), w.to(dev))
  torch.testing.assert_close(pw.cpu().double(), (lw * nw).cpu().double().sum(1))
  torch.testing.assert_close(pl.cpu().double() * pw.cpu().double(), rows.sum(1), atol=1e-5,
                             rtol=1e-5)
  mx = _impl(api, 'MixtureEMLoss')(name=None, temperature=2.0, alpha=0.5)
  losses, lw = mx.compute_unreduced_loss(labels.to(dev), logits3.to(dev) / 2.0)
  assert tuple(losses.shape) == (3, 1) and lw.reshape(-1).tolist() == [1., 1., 0.]
  pl, pw = mx.compute_per_list(labels.to(dev), (logits3 / 2.0).to(dev), None)
  torch.testing.assert_close(pl.cpu().double(), losses.reshape(-1).cpu().double(), atol=1e-6,
                             rtol=1e-6)
  per = (pl * pw).cpu().double()
  want = {R.SUM: float(per.sum()), R.MEAN: float(per.sum()) / 2.,
          R.SUM_BY_NONZERO_WEIGHTS: float(per.sum()) / 2., R.SUM_OVER_BATCH_SIZE: float(
              per.sum()) / 3.}
  for red, v in want.items():
    _close(mx.compute(labels.to(dev), logits3.to(dev), None, red), v, 5)


def test_rank_and_width_errors(api):
  R = api.Reduction
  labels = api.t([[1., 0.]])
  with pytest.raises(ValueError):
    _impl(api, 'ClickEMLoss')(name=None).compute(labels, api.t([[0.5, 0.2]]), None, R.SUM)
  with pytest.raises(ValueError):
    _impl(api, 'ClickEMLoss')(name=None).compute(labels, api.t([[[1., 2., 3.], [1., 2., 3.]]]),
                                                 None, R.SUM)
  with pytest.raises(ValueError):
    _impl(api, 'MixtureEMLoss')(name=None).compute(labels, api.t([[0.5, 0.2]]), None, R.SUM)


def test_click_em_recovery_oracle():
  """Click EM on position-biased clicks (tests/_click_refs.py) recovers the planted
  examination curve and ranks held-out lists better than a model trained naively on the
  clicks with sigmoid cross entropy, through the CPU oracle.  This run sets TAU and DELTA."""
  from oracle import click, keras_losses, scorer
  x, c, _ = CR.click_logs(CR.TRAIN_LISTS, seed=1)
  xt, _, p_rel = CR.click_logs(CR.TEST_LISTS, seed=2)
  em = click.ClickEMTrainer(scorer.init_tower_params(CR.D, [], 1, seed=3), torch.zeros(CR.N),
                            learning_rate=CR.LR)
  naive = scorer.init_tower_params(CR.D, [], 1, seed=3)
  leaves = naive['dense_w'] + naive['dense_b']
  for p in leaves:
    p.requires_grad_()
  accum = [torch.full_like(p, 0.1) for p in leaves]
  sce = keras_losses.SigmoidCrossEntropyLoss()
  for xb, cb in CR.batches(x, c):
    em.train_step(xb, cb)
    for p in leaves:
      p.grad = None
    sce(cb, scorer.tower_forward(xb.reshape(-1, CR.D), naive).reshape(cb.shape)).backward()
    with torch.no_grad():
      for p, a in zip(leaves, accum):
        a.add_(p.grad * p.grad)
        p.sub_(CR.LR * p.grad / (a.sqrt() + 1e-7))
  rel = CR.relative_propensity(em.examination_propensity())
  assert np.abs(rel - CR.eta())[1:].max() <= TAU, rel
  with torch.no_grad():
    s_em = em.relevance(xt, torch.ones(xt.shape[:2], dtype=torch.bool), False)
    s_naive = scorer.tower_forward(xt.reshape(-1, CR.D), naive).reshape(xt.shape[:2])
  assert CR.ndcg_at(s_em, p_rel, 5) >= CR.ndcg_at(s_naive, p_rel, 5) + DELTA
