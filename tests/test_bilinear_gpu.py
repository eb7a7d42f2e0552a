"""K14 Bilinear (csrc/bilinear.cu), keras.layers.Bilinear and train.BilinearClickRankingTrainer
on the GPU, against the fp64 restatements of oracle/bilinear.py.

Kernel tolerances are bounds on fp32 rounding for the kernel's summation order, as multiples of
U = 2^-24 times the oracle's sum of absolute terms S:
  y     s_j = sum_i a_i W'_ij (E + 1 terms), then sum_j c_j s_j (<= E + 4 terms)  -> (2E + 8) U S
  dv1   t_i = sum_j W'_ij c_j (E + 1 terms), then sum_k dy_k t_i,k (K terms)      -> (E + K + 4) U S
  dW    dy a (one rounding), a chain over the rows one thread sums (<= ceil(M / G) + 128, G the
        CTA count), at most 256 row slices and G CTA partials                     -> (ceil(M/G) + 1000) U S
with a' = [v1, 1], c' = [v2, 1] and W' the augmented weight (see the kernel's header)."""
import ctypes
import math

import numpy as np
import pytest
import torch

import _click_refs as CR
from test_golden_bilinear import DELTA, E_CLICK

U = 2.0 ** -24
LOG_EPS = float(np.float32(math.log(1e-10)))

SHAPES = [(1, 1), (3, 1), (16, 1), (64, 1), (100, 1), (128, 1), (8, 5), (64, 4), (32, 16), (16, 32),
          # limit edges: E = 128, K = 32, E^2 K at or just under 16384; (32, 16) and (24, 28)
          # keep one copy of W' in the backward (no room for the transposed one)
          (2, 32), (22, 32), (90, 2), (45, 8), (24, 28)]
ROWS = [1, 7, 255, 4097, 204800]


def _lib():
  import __graft_entry__ as g
  g.build()
  from ranking_b200 import _C
  return _C


def _case(m, e, k, seed, scale=1.0, masked=False):
  g = torch.Generator().manual_seed(seed)
  v1 = torch.randn(m, e, generator=g) * scale
  v2 = torch.randn(m, e, generator=g) * scale
  p = torch.randn(e * e * k + 2 * e * k + k, generator=g) / math.sqrt(e)
  dy = torch.randn(m, k, generator=g)
  mask = None
  if masked:
    mask = torch.rand(m, generator=g) > 0.3
    # masked rows carry garbage: the kernels must not read it into any result
    v1[~mask] = float('nan')
    v2[~mask] = float('inf')
    dy[~mask] = float('nan')
  return v1, v2, p, dy, mask


def _split(p, e, k):
  a, b, c = e * e * k, e * e * k + e * k, e * e * k + 2 * e * k
  return p[:a].view(e, e, k), p[a:b].view(e, k), p[b:c].view(e, k), p[c:]


def _oracle(v1, v2, p, dy, mask, e, k):
  """fp64 y, dv1, dv2, grads and their sums of absolute terms, in 1024-row chunks."""
  W, W1, W2, b = [t.double() for t in _split(p, e, k)]
  live = torch.ones(v1.shape[0], dtype=torch.bool) if mask is None else mask
  v1 = torch.where(live[:, None], v1, 0.).double()
  v2 = torch.where(live[:, None], v2, 0.).double()
  dy = torch.where(live[:, None], dy, 0.).double()
  Wf = W.reshape(e, e * k)
  aW, aW1, aW2, ab = W.abs(), W1.abs(), W2.abs(), b.abs()
  aWf = aW.reshape(e, e * k)
  out = {n: [] for n in ('y', 'sy', 'dv1', 'sdv1', 'dv2', 'sdv2')}
  gw = torch.zeros(e * k, e, dtype=torch.float64)
  sgw = torch.zeros_like(gw)
  for s in range(0, v1.shape[0], 1024):
    a, c, d = v1[s:s + 1024], v2[s:s + 1024], dy[s:s + 1024]
    t = (a @ Wf).view(-1, e, k)             # [m, j, k] = sum_i a_i W_ijk
    ta = (a.abs() @ aWf).view(-1, e, k)
    out['y'].append(torch.einsum('mjk,mj->mk', t, c) + a @ W1 + c @ W2 + b)
    out['sy'].append(torch.einsum('mjk,mj->mk', ta, c.abs()) + a.abs() @ aW1 + c.abs() @ aW2 + ab)
    out['dv2'].append(torch.einsum('mjk,mk->mj', t, d) + d @ W2.T)
    out['sdv2'].append(torch.einsum('mjk,mk->mj', ta, d.abs()) + d.abs() @ aW2.T)
    tw =torch.einsum('ijk,mk->mij', W, d)       # [m, i, j]
    out['dv1'].append(torch.einsum('mij,mj->mi', tw, c) + d @ W1.T)
    twa = torch.einsum('ijk,mk->mij', aW, d.abs())
    out['sdv1'].append(torch.einsum('mij,mj->mi', twa, c.abs()) + d.abs() @ aW1.T)
    du = torch.einsum('mi,mk->mik', a, d).reshape(-1, e * k)
    gw += du.T @ c
    sgw += torch.einsum('mi,mk->mik', a.abs(), d.abs()).reshape(-1, e * k).T @ c.abs()
  res = {n: torch.cat(v) for n, v in out.items()}
  dW = gw.view(e, k, e).permute(0, 2, 1)
  sdW = sgw.view(e, k, e).permute(0, 2, 1)
  res['grads'] = torch.cat([dW.reshape(-1), (v1.T @ dy).reshape(-1), (v2.T @ dy).reshape(-1),
                            dy.sum(0)])
  res['sgrads'] = torch.cat([sdW.reshape(-1), (v1.abs().T @ dy.abs()).reshape(-1),
                             (v2.abs().T @ dy.abs()).reshape(-1), dy.abs().sum(0)])
  return res


def _run(C, v1, v2, p, dy, mask, e, k):
  m = v1.shape[0]
  d = [t.cuda() for t in (v1, v2, p, dy)]
  m8 = None if mask is None else mask.to(torch.uint8).cuda()
  y = torch.empty(m, k, device='cuda')
  dv1, dv2 = torch.empty(m, e, device='cuda'), torch.empty(m, e, device='cuda')
  grads = torch.full_like(d[2], float('nan'))
  nws = C.lib.tfr_bilinear_workspace_bytes(m, e, k)
  ws = torch.empty(nws, dtype=torch.uint8, device='cuda')
  C.check(C.lib.tfr_bilinear_fwd(C.ptr(d[0]), C.ptr(d[1]), m, e, k, C.ptr(d[2]), C.ptr(m8),
                                 C.ptr(y), C.stream()))
  C.check(C.lib.tfr_bilinear_bwd(C.ptr(d[0]), C.ptr(d[1]), m, e, k, C.ptr(d[2]), C.ptr(m8),
                                 C.ptr(d[3]), C.ptr(dv1), C.ptr(dv2), C.ptr(grads), C.ptr(ws),
                                 C.stream()))
  torch.cuda.synchronize()
  ctas = nws // (4 * p.numel())
  return y.cpu(), dv1.cpu(), dv2.cpu(), grads.cpu(), ctas


def _within(got, ref, s, factor, what):
  got = got.double()
  err = (got - ref).abs()
  tol = factor * U * s + 1e-300
  bad = ~(err <= tol)
  assert not bool(bad.any()), '%s: %d of %d outside the bound, worst err/tol %.3g' % (
      what, int(bad.sum()), bad.numel(), float((err / tol)[bad].max()))


def _check(C, m, e, k, seed, scale=1.0, masked=False):
  v1, v2, p, dy, mask = _case(m, e, k, seed, scale, masked)
  y, dv1, dv2, grads, ctas = _run(C, v1, v2, p, dy, mask, e, k)
  r = _oracle(v1, v2, p, dy, mask, e, k)
  live = torch.ones(m, dtype=torch.bool) if mask is None else mask
  assert bool((y[~live] == LOG_EPS).all())
  assert bool((dv1[~live] == 0).all()) and bool((dv2[~live] == 0).all())
  _within(y[live], r['y'][live], r['sy'][live], 2 * e + 8, 'y')
  _within(dv1[live], r['dv1'][live], r['sdv1'][live], e + k + 4, 'dv1')
  _within(dv2[live], r['dv2'][live], r['sdv2'][live], e + k + 4, 'dv2')
  _within(grads, r['grads'], r['sgrads'], -(-m // ctas) + 1000, 'grads')


@pytest.mark.gpu
@pytest.mark.parametrize('m', ROWS)
@pytest.mark.parametrize('e,k', SHAPES)
def test_kernels_match_oracle(m, e, k):
  C = _lib()
  _check(C, m, e, k, seed=m * 131 + e * 7 + k)


@pytest.mark.gpu
@pytest.mark.parametrize('m', [7, 4097, 204800])
@pytest.mark.parametrize('e,k', [(1, 1), (16, 1), (100, 1), (128, 1), (8, 5), (22, 32)])
def test_kernels_row_mask(m, e, k):
  _check(_lib(), m, e, k, seed=m + e + k, masked=True)


@pytest.mark.gpu
@pytest.mark.parametrize('e,k', [(16, 1), (64, 4), (128, 1)])
def test_kernels_large_magnitude(e, k):
  _check(_lib(), 4097, e, k, seed=e * k, scale=3e3, masked=True)


@pytest.mark.gpu
def test_backward_is_deterministic():
  C = _lib()
  m, e, k = 204800, 16, 1
  v1, v2, p, dy, mask = _case(m, e, k, seed=9, masked=True)
  a = _run(C, v1, v2, p, dy, mask, e, k)
  b = _run(C, v1, v2, p, dy, mask, e, k)
  for x, y in zip(a[:4], b[:4]):
    assert torch.equal(x.view(torch.int32), y.view(torch.int32))


@pytest.mark.gpu
def test_layer_autograd_matches_oracle():
  import ranking_b200 as tfr
  from oracle import bilinear
  bsz, n, e, k = 6, 37, 12, 3
  layer = tfr.keras.layers.Bilinear(e, k, seed=2)
  with torch.no_grad():
    layer.const_term().copy_(torch.tensor([0.5, -1., 2.]))
  g = torch.Generator().manual_seed(1)
  v1 = torch.randn(bsz, n, e, generator=g)
  v2 = torch.randn(bsz, n, e, generator=g)
  w = torch.randn(bsz, n, k, generator=g)
  a, c = v1.cuda().requires_grad_(), v2.cuda().requires_grad_()
  out = layer((a, c))
  assert tuple(out.shape) == (bsz, n, k)
  (out * w.cuda()).sum().backward()
  ref_w = [t.detach().cpu().double().clone().requires_grad_() for t in
           (layer.bilinear_term(), layer.linear_term_1(), layer.linear_term_2(),
            layer.const_term())]
  ra, rc = v1.double().requires_grad_(), v2.double().requires_grad_()
  ref = bilinear.bilinear(ra, rc, *ref_w)
  (ref * w.double()).sum().backward()

  def rel(x, y):
    return float((x.detach().cpu().double() - y).abs().max() / (y.abs().max() + 1e-30))
  assert rel(out, ref.detach()) < 1e-5
  assert rel(a.grad, ra.grad) < 1e-5 and rel(c.grad, rc.grad) < 1e-5
  assert rel(layer.flat.grad, torch.cat([t.grad.reshape(-1) for t in ref_w])) < 1e-5
  with pytest.raises(ValueError):
    layer((a, c[:, :5]))
  with pytest.raises(ValueError):
    layer((a[..., :5], c[..., :5]))
  with pytest.raises(ValueError):
    tfr.keras.layers.Bilinear(64, 5)


def _oracle_tower(tower, bn):
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


def _make(precision, bn, e=8, npos=12, d=20, seed=3):
  import ranking_b200 as tfr
  torch.manual_seed(seed)
  tower = tfr.keras.layers.create_tower([32, 16], e, activation='relu', use_batch_norm=bn,
                                        dropout=0, input_dim=d, seed=seed, precision=precision)
  with torch.no_grad():
    for i in range(len(tower.dims) - 1):
      tower.bias(i).uniform_(-0.2, 0.2)
  bil = tfr.keras.layers.Bilinear(e, 1, seed=seed + 1)
  with torch.no_grad():
    bil.const_term().fill_(0.3)
  tr = tfr.train.BilinearClickRankingTrainer(tower, bil,
                                             tfr.keras.losses.SigmoidCrossEntropyLoss(), npos,
                                             seed=seed + 2, learning_rate=0.05)
  return tr, tower, bil


@pytest.mark.gpu
@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
@pytest.mark.parametrize('explicit_positions', [False, True])
@pytest.mark.parametrize('bn', [False, True])
@pytest.mark.parametrize('use_mask', [False, True])
def test_trainer_step_matches_oracle(precision, explicit_positions, bn, use_mask):
  """One BilinearClickRankingTrainer step against the oracle step: loss, the flat gradient
  (table, bilinear, tower), the parameters after Adagrad and `predict`; the padding of the
  table and of the bilinear block gets zero gradient; the same step again from the same state
  gives bitwise-identical parameters."""
  from oracle import bilinear
  b, n, d, npos, e = 16, 30, 20, 12, 8
  g = torch.Generator().manual_seed(11)
  x = torch.randn(b, n, d, generator=g)
  clicks = (torch.rand(b, n, generator=g) < 0.25).float()
  lens = torch.randint(n // 2, n + 1, (b,), generator=g)
  clicks = torch.where(torch.arange(n)[None] < lens[:, None], clicks, torch.full_like(clicks, -1))
  positions = torch.randint(0, npos, (b, n), generator=g) if explicit_positions else None
  # a mask shorter than the labelled prefix: masked items with labels >= 0 see ln(1e-10)
  # logits.  (A prefix, because predict circularly pads BN towers by the mask.)
  cut = lens - torch.randint(0, 4, (b,), generator=g)
  mask = (torch.arange(n)[None] < cut[:, None]) if use_mask else None
  tr, tower, bil = _make(precision, bn, e, npos, d)
  rows = tr.positions_table.vocab_size
  P = bil.flat.numel()
  off_b, off_t = rows * e, tr.tower.tower_offset
  assert off_b % 64 == 0 and off_t % 64 == 0 and off_t >= off_b + P
  table = tr.positions_table.table.detach()[:npos].cpu().double().clone()
  bw = [t.detach().cpu().double().clone() for t in (bil.bilinear_term(), bil.linear_term_1(),
                                                    bil.linear_term_2(), bil.const_term())]
  moving = None
  if bn:
    from oracle import scorer
    moving = scorer.init_bn_moving(d, [32, 16], use_batch_norm=True, dtype=torch.float64)
  ot = bilinear.BilinearClickTrainer(_oracle_tower(tower, bn), table, bw, activation='relu',
                                     use_batch_norm=bn, bn_moving=moving, learning_rate=0.05)
  state = (tr.tower.flat.detach().clone(), tr.accum.clone(), tower.bn_state.clone())
  cuda = lambda t: None if t is None else t.cuda()   # noqa: E731
  got = tr.train_step(x.cuda(), clicks.cuda(), positions=cuda(positions), mask=cuda(mask))
  ref = ot.train_step(x.double(), clicks.double(), positions=positions, mask=mask)
  assert abs(float(got) - float(ref)) <= 1e-5 * max(1., abs(float(ref)))
  pick = lambda f: torch.cat([f[:npos * e], f[off_b:off_b + P], f[off_t:]])   # noqa: E731
  assert _rel_err(pick(tr.grads), ot.flat_grad()) <= 5e-5
  assert float(tr.grads[npos * e:off_b].abs().max()) == 0.
  assert float(tr.grads[off_b + P:off_t].abs().max()) == 0.
  flat = tr.tower.flat.detach()
  assert _rel_err(pick(flat), ot.flat_params()) <= 1e-5
  got_p = tr.predict(x.cuda(), mask=cuda(mask)).clone()
  ref_p = ot.predict(x.double(), serving_position=0, mask=mask)
  assert _rel_err(got_p, ref_p) <= 1e-4
  if positions is not None:
    got_p = tr.predict(x.cuda(), mask=cuda(mask), positions=positions.cuda()).clone()
    assert _rel_err(got_p, ot.predict(x.double(), positions=positions, mask=mask)) <= 1e-4
  first = flat.clone()
  with torch.no_grad():
    tr.tower.flat.copy_(state[0])
    tr.accum.copy_(state[1])
    tower.bn_state.copy_(state[2])
  tr.train_step(x.cuda(), clicks.cuda(), positions=cuda(positions), mask=cuda(mask))
  assert torch.equal(tr.tower.flat.detach().view(torch.int32), first.view(torch.int32))


@pytest.mark.gpu
def test_trainer_errors():
  import ranking_b200 as tfr
  L = tfr.keras.layers
  sce = tfr.keras.losses.SigmoidCrossEntropyLoss()
  tower = L.create_tower([16], 4, use_batch_norm=False, dropout=0, input_dim=8, precision='fp32')
  bil = L.Bilinear(4, 1, seed=1)
  tr = tfr.train.BilinearClickRankingTrainer(tower, bil, sce, 5)
  x = torch.randn(2, 4, 8).cuda()
  y = torch.zeros(2, 4).cuda()
  for bad in (5, -1):
    pos = torch.zeros(2, 4, dtype=torch.int64)
    pos[1, 2] = bad
    with pytest.raises(ValueError):
      tr.train_step(x, y, positions=pos.cuda())
  with pytest.raises(ValueError):
    tr.train_step(x, y, positions=torch.zeros(2, 3, dtype=torch.int64).cuda())
  tr.train_step(x, y)
  assert tuple(tr.predict(x).shape) == (2, 4)
  mk = lambda out, prec='fp32': L.create_tower([16], out, use_batch_norm=False,  # noqa: E731
                                              dropout=0, input_dim=8, precision=prec)
  cases = [(mk(4, 'bf16'), L.Bilinear(4, 1), sce),
           (mk(3), L.Bilinear(4, 1), sce),
           (mk(4), L.Bilinear(4, 2), sce),
           (mk(4), L.Bilinear(4, 1), tfr.keras.losses.ClickEMLoss()),
           (mk(4), L.Bilinear(4, 1), tfr.keras.losses.MixtureEMLoss())]
  for t, b, loss in cases:
    with pytest.raises(ValueError):
      tfr.train.BilinearClickRankingTrainer(t, b, loss, 5)
  with pytest.raises(ValueError):
    tfr.train.BilinearClickRankingTrainer(mk(4), L.Bilinear(4, 1), sce, 5, serving_position=5)


@pytest.mark.gpu
def test_checkpoint_resumes_to_the_same_bits(tmp_path):
  import ranking_b200 as tfr
  g = torch.Generator().manual_seed(4)
  x = torch.randn(8, 10, 20, generator=g).cuda()
  clicks = (torch.rand(8, 10, generator=g) < 0.3).float().cuda()

  def steps(tr, k):
    for _ in range(k):
      tr.train_step(x, clicks)

  a, _, _ = _make('tf32x3', True)
  steps(a, 4)
  b, _, _ = _make('tf32x3', True)
  steps(b, 2)
  path = str(tmp_path / 'ckpt.pt')
  tfr.pipeline.save_checkpoint(b, path, 2)
  c, _, _ = _make('tf32x3', True, seed=9)
  tfr.pipeline.load_checkpoint(c, path)
  steps(c, 2)
  assert torch.equal(a.tower.flat.detach().view(torch.int32),
                     c.tower.flat.detach().view(torch.int32))
  assert torch.equal(a.accum.view(torch.int32), c.accum.view(torch.int32))


@pytest.mark.gpu
def test_bilinear_click_recovery():
  """The oracle experiment of test_golden_bilinear.py on the GPU trainer: NDCG@5 of held-out
  lists scored at position 0 at least DELTA above a model trained naively on the clicks."""
  import ranking_b200 as tfr
  x, c, _ = CR.click_logs(CR.TRAIN_LISTS, seed=1)
  xt, _, p_rel = CR.click_logs(CR.TEST_LISTS, seed=2)
  mk = lambda out: tfr.keras.layers.create_tower([], out, use_batch_norm=False,  # noqa: E731
                                                 dropout=0, input_dim=CR.D, seed=3,
                                                 precision='fp32')
  sce = tfr.keras.losses.SigmoidCrossEntropyLoss()
  two = tfr.train.BilinearClickRankingTrainer(mk(E_CLICK), tfr.keras.layers.Bilinear(
      E_CLICK, 1, seed=4), sce, CR.N, seed=5, learning_rate=CR.LR)
  naive = tfr.train.RankingTrainer(mk(1), sce, learning_rate=CR.LR)
  x, c = x.cuda(), c.cuda()
  for xb, cb in CR.batches(x, c):
    two.train_step(xb, cb)
    naive.train_step(xb, cb)
  xt = xt.cuda()
  got = CR.ndcg_at(two.predict(xt).clone(), p_rel, 5)
  base = CR.ndcg_at(naive.predict(xt).clone(), p_rel, 5)
  assert got >= base + DELTA, (got, base)
