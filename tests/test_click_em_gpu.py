"""K3d (csrc/loss_click.cu) and ClickEMRankingTrainer on the GPU against the fp64 oracle
(oracle/click.py), plus the argument checks of the two C entry points (no GPU needed)."""
import ctypes

import numpy as np
import pytest
import torch

import _click_refs as CR
from test_golden_click_losses import DELTA, TAU

U = 2.0 ** -24     # fp32 unit roundoff


def _lib():
  import __graft_entry__ as g
  g.build()
  from ranking_b200 import _C
  return _C


def test_click_loss_argument_validation_without_gpu():
  """NULL inputs, N outside 1..8192, M outside 1..32 and strides other than 1 / 2 are
  rejected with TFR_INVALID_ARGUMENT before any CUDA call."""
  _C = _lib()
  p = ctypes.c_void_p(256)    # never dereferenced: validation fails first
  ce = _C.lib.tfr_click_em_loss_fwd_bwd
  mx = _C.lib.tfr_mixture_em_loss_fwd_bwd

  def click(exam=p, n=4, stride=1):
    return ce(exam, p, stride, p, None, 0, None, 2, n, 1.0, 1.0, 1.0, 1.0, p, p, None, p, None,
              None, None)

  def mix(scores=p, n=4, m=2):
    return mx(scores, p, None, 0, None, 2, n, m, 1.0, 1.0, 1.0, p, p, None, None)

  for rc in (click(exam=None), click(n=0), click(n=8193), click(stride=0), click(stride=3),
             mix(scores=None), mix(n=0), mix(n=8193), mix(m=0), mix(m=33)):
    assert rc == 1, _C.last_error()


def _click_case(b, n, seed, extreme):
  g = torch.Generator().manual_seed(seed)
  logits = torch.randn(b, n, 2, generator=g) * 3.
  if extreme:
    vals = torch.tensor([100., -100., 1e4, -1e4])
    pick = torch.rand(b, n, 2, generator=g) < 0.2
    logits = torch.where(pick, vals[torch.randint(0, 4, (b, n, 2), generator=g)], logits)
  clicks = (torch.rand(b, n, generator=g) < 0.3).float()
  if n > 2:
    lens = torch.randint(1, n + 1, (b,), generator=g)
    clicks = torch.where(torch.arange(n)[None] < lens[:, None], clicks, torch.full_like(clicks, -1))
  clicks[0] = torch.where(clicks[0] >= 0, torch.zeros_like(clicks[0]), clicks[0])   # no click
  mask = torch.rand(b, n, generator=g) > 0.15
  return logits, clicks, mask


@pytest.mark.gpu
@pytest.mark.parametrize('n', [1, 2, 7, 64, 200, 1000, 8192])
@pytest.mark.parametrize('wkind', ['none', 'list', 'item'])
@pytest.mark.parametrize('kw,use_mask,extreme', [
    (dict(), False, False),
    (dict(temperature=0.7, exam_loss_weight=1.5, rel_loss_weight=0.5), True, False),
    (dict(), True, True)])
def test_click_em_loss_and_grad(cuda_api, oracle_api, n, wkind, kw, use_mask, extreme):
  """ClickEM MEAN loss and d loss / d logits against fp64 autograd.  Every item term
  max(x, 0) - x z + log1p(exp(-|x|)) is formed from fp32 operations of size at most
  |x| + 1, so the sum of the n terms is off by at most a few units of fp32 roundoff times
  S = sum_i w_i (ew (|e_i| + 1) + rw (|r_i| + 1)) / T; the posterior logit e - softplus(r)
  carries ~U (|e| + |r|) / T, which moves a gradient entry (bounded by its coefficient
  c_i = w_i max(ew, rw) / (T sum w)) by at most a quarter of that.  The per-list sums are
  about n / 256 + 10 additions deep (a serial run per thread, then a tree), each adding at
  most U S of rounding."""
  from oracle import click
  b = 5
  logits, clicks, mask = _click_case(b, n, 7 + n, extreme)
  t = kw.get('temperature', 1.0)
  ew, rw = kw.get('exam_loss_weight', 1.0), kw.get('rel_loss_weight', 1.0)
  g = torch.Generator().manual_seed(n)
  weights = {'none': None, 'list': torch.rand(b, 1, generator=g) + 0.5,
             'item': torch.rand(b, n, generator=g) + 0.5}[wkind]
  m = mask if use_mask else None
  fc = cuda_api.losses_impl.ClickEMLoss(name=None, **kw)
  fo = click.ClickEMLoss(name=None, **kw)
  lg = logits.cuda().requires_grad_()
  got = fc.compute(clicks.cuda(), lg, None if weights is None else weights.cuda(),
                   cuda_api.Reduction.MEAN, None if m is None else m.cuda())
  lr = logits.double().requires_grad_()
  ref = fo.compute(clicks.double(), lr, None if weights is None else weights.double(),
                   oracle_api.Reduction.MEAN, m)
  got.backward()
  ref.backward()
  assert torch.isfinite(got) and torch.isfinite(lg.grad).all()
  w = fo.normalize_weights(clicks.double(), None if weights is None else weights.double())
  w = w * (clicks >= 0 if m is None else (m & (clicks >= 0))).double()
  wsum = float(w.sum())
  if wsum == 0:
    assert float(got) == 0. and float(lg.grad.abs().max()) == 0.
    return
  mag = logits.double().abs() / t
  S = float((w * (ew * (mag[..., 0] + 1) + rw * (mag[..., 1] + 1))).sum()) / wsum
  assert abs(float(got) - float(ref)) <= 1e-6 * max(1., abs(float(ref))) + (
      n / 256 + 10) * U * S
  c = (w * max(ew, rw) / (t * wsum)).unsqueeze(2)
  tol = c * (16 * U + U * (mag[..., :1] + mag[..., 1:]))
  err = (lg.grad.double().cpu() - lr.grad).abs()
  assert bool((err <= tol + 1e-30).all()), float((err - tol).max())
  assert bool((lg.grad.cpu()[w == 0] == 0).all())   # invalid items: exact zeros


@pytest.mark.gpu
@pytest.mark.parametrize('n', [1, 2, 7, 64, 200, 1000, 8192])
@pytest.mark.parametrize('m_', [1, 2, 3, 8, 32])
@pytest.mark.parametrize('alpha', [0.1, 1., 10.])
@pytest.mark.parametrize('wkind', ['none', 'list', 'item'])
def test_mixture_em_loss_and_grad(cuda_api, oracle_api, n, m_, alpha, wkind):
  """MixtureEM SUM loss and gradient against fp64 autograd.  L_m sums fp32 item terms in
  fp64, each term off by at most ~4 U (|s| + 1) (T = 1); the +-100 / +-1e4 entries with
  labels in {0, 1} are formed exactly (max(x, 0) - x l is exact, log1p(exp(-|x|)) < 1e-43),
  so |dL_m| <= dL = 4 U sum over the other valid entries of (|s_i| + 1).
  The loss moves by at most (1 + M) dL (d loss / d L_k = q_k / Q (1 - alpha (L_k - loss)),
  and alpha x exp(-alpha x) <= 1 / e); q_m / Q moves relatively by at most 2 alpha dL, which
  bounds the gradient error by (q_m / Q) |sigmoid(s) - l| (2 alpha dL + 16 U) / T."""
  from oracle import click
  b = 4
  g = torch.Generator().manual_seed(100 * m_ + n)
  logits = torch.randn(b, n, m_, generator=g) * 2.
  if n >= 7:
    logits[1, :3] = torch.tensor([100., -1e4, 1e4])[:, None]
  clicks = (torch.rand(b, n, generator=g) < 0.3).float()
  if n > 2:
    clicks[:, -(n // 4 + 1):] = -1.
  clicks[2] = torch.where(clicks[2] >= 0, torch.zeros_like(clicks[2]), clicks[2])
  weights = {'none': None, 'list': torch.rand(b, 1, generator=g) + 0.5,
             'item': torch.rand(b, n, generator=g) + 0.5}[wkind]
  t = 1.0
  fc = cuda_api.losses_impl.MixtureEMLoss(name=None, temperature=t, alpha=alpha)
  fo = click.MixtureEMLoss(name=None, temperature=t, alpha=alpha)
  lg = logits.cuda().requires_grad_()
  got = fc.compute(clicks.cuda(), lg, None if weights is None else weights.cuda(),
                   cuda_api.Reduction.SUM)
  lr = logits.double().requires_grad_()
  ref = fo.compute(clicks.double(), lr, None if weights is None else weights.double(),
                   oracle_api.Reduction.SUM)
  got.backward()
  ref.backward()
  valid = (clicks >= 0).double()
  mod = (logits.abs() < 100).double() * valid.unsqueeze(2)
  dl = 4 * U * float(((logits.double().abs() + 1) * mod).sum((1, 2)).max())
  _, lw = fo.compute_per_list(clicks.double(), logits.double(),
                              None if weights is None else weights.double())
  assert abs(float(got) - float(ref)) <= float(lw.abs().sum()) * (1 + m_) * dl + 1e-6 * max(
      1., abs(float(ref)))
  gmax = (lr.grad.abs().amax((1, 2), keepdim=True) + 1e-30)
  err = (lg.grad.double().cpu() - lr.grad).abs()
  assert bool((err <= gmax * (2 * alpha * dl + 16 * U) + 1e-30).all())


@pytest.mark.gpu
def test_stride_and_determinism(cuda_api):
  """Stride 2 (the Keras [B, N, 2] tensor) and stride 1 (two planes) give identical bits;
  two identical calls of either kernel give identical bits."""
  from ranking_b200 import _C
  b, n = 64, 333
  logits, clicks, _ = _click_case(b, n, 5, True)
  logits, clicks = logits.cuda().contiguous(), clicks.cuda()
  w = (torch.rand(b, n) + 0.5).cuda()
  exam, rel = logits[..., 0].contiguous(), logits[..., 1].contiguous()

  def run(stride):
    out = [torch.empty(b, n, 2, device='cuda')] + [torch.empty(b, n, device='cuda')
                                                    for _ in range(3)] + [
        torch.empty(b, device='cuda') for _ in range(3)]
    g, de, dr, row, loss, weight, nz = out
    if stride == 2:
      args = (logits.data_ptr(), logits.data_ptr() + 4, 2)
      gp = (g.data_ptr(), g.data_ptr() + 4)
    else:
      args = (exam.data_ptr(), rel.data_ptr(), 1)
      gp = (de.data_ptr(), dr.data_ptr())
    _C.check(_C.lib.tfr_click_em_loss_fwd_bwd(
        *args, _C.ptr(clicks), _C.ptr(w), 1, None, b, n, 0.7, 1.5, 0.5, 0.25, *gp,
        _C.ptr(row), _C.ptr(loss), _C.ptr(weight), _C.ptr(nz), _C.stream()))
    if stride == 2:
      de.copy_(g[..., 0])
      dr.copy_(g[..., 1])
    return [de, dr, row, loss, weight, nz]

  a, a2, s1 = run(2), run(2), run(1)
  for x, y, z in zip(a, a2, s1):
    assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    assert torch.equal(x.view(torch.int32), z.view(torch.int32))
  scores = torch.randn(b, n, 5).cuda()
  mx = cuda_api.losses_impl.MixtureEMLoss(name=None, alpha=2.)
  outs = []
  for _ in range(2):
    s = scores.clone().requires_grad_()
    loss = mx.compute(clicks, s, w, cuda_api.Reduction.SUM)
    loss.backward()
    outs.append((loss.detach().view(torch.int32), s.grad.view(torch.int32)))
  assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


def _oracle_params(tower, bn):
  nl = len(tower.dims) - 1
  cp = lambda t: t.detach().cpu().double().clone()   # noqa: E731
  p = {'dense_w': [cp(tower.kernel(i)) for i in range(nl)],
       'dense_b': [cp(tower.bias(i)) for i in range(nl)], 'bn_gamma': [], 'bn_beta': [],
       'in_bn_gamma': None, 'in_bn_beta': None}
  if bn:
    for i in range(nl - 1):
      p['bn_gamma'].append(cp(tower.bn_gamma(i)))
      p['bn_beta'].append(cp(tower.bn_beta(i)))
  return p


def _rel_err(got, ref):
  got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
  return float((got - ref).abs().max() / (ref.abs().max() + 1e-30))


@pytest.mark.gpu
@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
@pytest.mark.parametrize('explicit_positions', [False, True])
@pytest.mark.parametrize('bn', [False, True])
def test_trainer_step_matches_oracle(precision, explicit_positions, bn):
  """One ClickEMRankingTrainer step against the oracle click trainer: loss, the flat
  gradient (position table and tower) and the parameters after Adagrad, on padded lists;
  then the same step again from the same state gives bitwise-identical parameters."""
  import ranking_b200 as tfr
  from oracle import click
  b, n, d, npos = 16, 30, 20, 12
  g = torch.Generator().manual_seed(11)
  x = torch.randn(b, n, d, generator=g)
  clicks = (torch.rand(b, n, generator=g) < 0.25).float()
  lens = torch.randint(n // 2, n + 1, (b,), generator=g)
  clicks = torch.where(torch.arange(n)[None] < lens[:, None], clicks, torch.full_like(clicks, -1))
  positions = torch.randint(0, npos, (b, n), generator=g) if explicit_positions else None
  torch.manual_seed(3)
  tower = tfr.keras.layers.create_tower([32, 16], 1, activation='relu', use_batch_norm=bn,
                                        dropout=0, input_dim=d, seed=3, precision=precision)
  with torch.no_grad():
    for i in range(len(tower.dims) - 1):
      tower.bias(i).uniform_(-0.2, 0.2)
  tr = tfr.train.ClickEMRankingTrainer(tower, tfr.keras.losses.ClickEMLoss(), npos, seed=4,
                                       learning_rate=0.05)
  rows = tr.positions_table.vocab_size
  params = _oracle_params(tower, bn)
  table = tr.positions_table.flat.detach()[:npos].cpu().double().clone()
  moving = None
  if bn:
    from oracle import scorer
    moving = scorer.init_bn_moving(d, [32, 16], use_batch_norm=True, dtype=torch.float64)
  ot = click.ClickEMTrainer(params, table, activation='relu', use_batch_norm=bn,
                            bn_moving=moving, learning_rate=0.05)
  state = (tr.tower.flat.detach().clone(), tr.accum.clone(), tower.bn_state.clone())
  got = tr.train_step(x.cuda(), clicks.cuda(),
                      positions=None if positions is None else positions.cuda())
  ref = ot.train_step(x.double(), clicks.double(), positions=positions)
  assert abs(float(got) - float(ref)) <= 1e-5 * max(1., abs(float(ref)))
  og = ot.flat_grad()
  pg = torch.cat([tr.grads[:npos], tr.grads[rows:]])
  assert _rel_err(pg, og) <= 5e-5
  assert float(tr.grads[npos:rows].abs().max()) == 0.
  flat = tr.tower.flat.detach()
  assert _rel_err(torch.cat([flat[:npos], flat[rows:]]), ot.flat_params()) <= 1e-5
  first = flat.clone()
  with torch.no_grad():
    tr.tower.flat.copy_(state[0])
    tr.accum.copy_(state[1])
    tower.bn_state.copy_(state[2])
  tr.train_step(x.cuda(), clicks.cuda(), positions=None if positions is None else positions.cuda())
  assert torch.equal(tr.tower.flat.detach().view(torch.int32), first.view(torch.int32))


@pytest.mark.gpu
def test_trainer_rejects_bad_positions_and_bf16():
  import ranking_b200 as tfr
  tower = tfr.keras.layers.create_tower([16], 1, use_batch_norm=False, dropout=0, input_dim=8,
                                        precision='fp32')
  tr = tfr.train.ClickEMRankingTrainer(tower, tfr.keras.losses.ClickEMLoss(), 5)
  x = torch.randn(2, 4, 8).cuda()
  y = torch.zeros(2, 4).cuda()
  for bad in (5, -1):
    pos = torch.zeros(2, 4, dtype=torch.int64)
    pos[1, 2] = bad
    with pytest.raises(ValueError):
      tr.train_step(x, y, positions=pos.cuda())
  tr.train_step(x, y)
  assert tuple(tr.examination_propensity().shape) == (5,)
  assert tuple(tr.predict(x).shape) == (2, 4)
  bf = tfr.keras.layers.create_tower([16], 1, use_batch_norm=False, dropout=0, input_dim=8,
                                     precision='bf16')
  with pytest.raises(ValueError):
    tfr.train.ClickEMRankingTrainer(bf, tfr.keras.losses.ClickEMLoss(), 5)
  with pytest.raises(ValueError):
    tfr.train.ClickEMRankingTrainer(tower, tfr.keras.losses.SigmoidCrossEntropyLoss(), 5)


@pytest.mark.gpu
def test_click_em_recovery():
  """The oracle experiment of test_golden_click_losses.py on the GPU trainer: relative
  propensities within TAU of the planted curve, NDCG@5 at least DELTA above a model trained
  naively on the clicks with sigmoid cross entropy."""
  import ranking_b200 as tfr
  x, c, _ = CR.click_logs(CR.TRAIN_LISTS, seed=1)
  xt, _, p_rel = CR.click_logs(CR.TEST_LISTS, seed=2)
  mk = lambda: tfr.keras.layers.create_tower([], 1, use_batch_norm=False, dropout=0,  # noqa
                                             input_dim=CR.D, seed=3, precision='fp32')
  em = tfr.train.ClickEMRankingTrainer(mk(), tfr.keras.losses.ClickEMLoss(), CR.N, seed=5,
                                       learning_rate=CR.LR)
  naive = tfr.train.RankingTrainer(mk(), tfr.keras.losses.SigmoidCrossEntropyLoss(),
                                   learning_rate=CR.LR)
  x, c = x.cuda(), c.cuda()
  for xb, cb in CR.batches(x, c):
    em.train_step(xb, cb)
    naive.train_step(xb, cb)
  rel = CR.relative_propensity(em.examination_propensity())
  assert np.abs(rel - CR.eta())[1:].max() <= TAU, rel
  xt = xt.cuda()
  s_em = em.predict(xt).clone()
  s_naive = naive.predict(xt).clone()
  assert CR.ndcg_at(s_em, p_rel, 5) >= CR.ndcg_at(s_naive, p_rel, 5) + DELTA
