"""The blocked fp64 references of tests/_list_refs.py against the oracle (CPU only).

test_list_size_sweep_gpu.py compares the CUDA kernels with these references above N = 2048,
where the oracle's [B, N, N] tensors no longer fit.  Here both are evaluated at N <= 512
with a small row block, so that lists span several blocks and end in a partial one:
values and score gradients, with tail padding, holes, an explicit mask, tied scores and
tied labels, lists without a relevant item, fully padded lists and all weight forms.
Both sides are fp64; they must agree to 1e-10.
"""
import pytest
import torch

import _list_refs as refs
from oracle import keras_losses as KO
from oracle import losses_impl as LO

TOL = 1e-10


@pytest.fixture(autouse=True)
def small_blocks(monkeypatch):
  monkeypatch.setattr(refs, 'ROW_BLOCK', 48)


def _case(b, n, seed, ties=True):
  g = torch.Generator().manual_seed(seed)
  scores = torch.randn(b, n, generator=g, dtype=torch.float64) * 2.
  if ties:
    scores[:, ::5] = torch.round(scores[:, ::5] * 2.) / 2.       # ties on a coarse grid
  labels = torch.multinomial(torch.tensor([.55, .25, .12, .06, .02]), b * n, replacement=True,
                             generator=g).reshape(b, n).double()
  lens = torch.randint((n + 1) // 2, n + 1, (b,), generator=g)
  labels = torch.where(torch.arange(n).unsqueeze(0) < lens.unsqueeze(1), labels,
                       torch.full_like(labels, -1.))
  labels = torch.where(torch.rand(b, n, generator=g) < 0.15, torch.full_like(labels, -1.),
                       labels)                                   # holes
  if b >= 4:
    labels[1] = torch.where(labels[1] >= 0, torch.zeros_like(labels[1]), labels[1])
    labels[2] = -1.
  item_w = torch.rand(b, n, generator=g, dtype=torch.float64) + 0.5
  list_w = torch.rand(b, 1, generator=g, dtype=torch.float64) + 0.5
  mask = (labels >= 0) & (torch.rand(b, n, generator=g) < 0.9)
  if b >= 4:
    mask[3, 0] = labels[3, 0] < 0                                # disagrees with labels >= 0
  return scores, labels, {'none': None, 'list': list_w, 'item': item_w}, mask


def _close(got, ref):
  scale = max(1.0, float(ref.abs().max()))
  assert float((got - ref).abs().max()) <= TOL * scale, float((got - ref).abs().max())


@pytest.mark.parametrize('mode,cls', [('ndcg', 'ApproxNDCGLoss'), ('mrr', 'ApproxMRRLoss')])
@pytest.mark.parametrize('wkind', ['none', 'list', 'item'])
@pytest.mark.parametrize('n,use_mask', [(1, False), (47, False), (130, True), (512, False)])
def test_approx_reference_matches_oracle(mode, cls, wkind, n, use_mask):
  scores, labels, weights, mask = _case(6, n, seed=n + len(wkind))
  w = weights[wkind]
  m = mask if use_mask else None
  s = scores.clone().requires_grad_()
  ref = getattr(LO, cls)(temperature=0.1).compute(labels, s, w, LO.Reduction.SUM, m)
  ref.backward()
  total, grad, _ = refs.approx_loss(labels, scores, w, m, temperature=0.1, mode=mode)
  _close(total, ref.detach())
  _close(grad, s.grad)


LAMBDAS = {
    'none': lambda: None,
    'ndcg': lambda: KO.NDCGLambdaWeight(),
    'dcg_smooth': lambda: KO.DCGLambdaWeight(topn=20, smooth_fraction=0.4),
    'precision_top3': lambda: KO.PrecisionLambdaWeight(topn=3),
}
PHI = {'logistic': 'PairwiseLogisticLoss', 'hinge': 'PairwiseHingeLoss',
       'soft_zero_one': 'PairwiseSoftZeroOneLoss', 'mse': 'PairwiseMSELoss'}


@pytest.mark.parametrize('phi', sorted(PHI))
@pytest.mark.parametrize('lam', sorted(LAMBDAS))
@pytest.mark.parametrize('wkind', ['none', 'list', 'item'])
@pytest.mark.parametrize('n', [1, 100, 300])
def test_pairwise_reference_matches_oracle(phi, lam, wkind, n):
  """The logistic loss is compared without tied scores: at z_i == z_j the reference (like
  the kernels) uses phi'(0) = -1/2, while autograd through the oracle's
  relu(-x) + log1p(exp(-|x|)) takes the subgradient 0 of both kinks."""
  scores, labels, weights, _ = _case(5, n, seed=3 * n + len(lam), ties=phi != 'logistic')
  w = weights[wkind]
  s = scores.clone().requires_grad_()
  ref = getattr(KO, PHI[phi])(reduction=KO.Reduction.SUM, lambda_weight=LAMBDAS[lam](),
                              temperature=0.7)(labels, s, w)
  ref.backward()
  total, grad = refs.pairwise_loss(labels, scores, w, phi, LAMBDAS[lam](), temperature=0.7)
  _close(total, ref.detach())
  _close(grad, s.grad)


def test_pairwise_reference_tail_copies():
  """Circular padding: the tail repeats the leading items with equal score and label."""
  scores, labels, weights, _ = _case(3, 64, seed=9, ties=False)
  labels[:, 40:] = labels[:, :24].clamp(min=0.)
  scores[:, 40:] = scores[:, :24]
  for lam in ('ndcg', 'precision_top3'):     # (a copy ties its original: no logistic here)
    s = scores.clone().requires_grad_()
    ref = KO.PairwiseHingeLoss(reduction=KO.Reduction.SUM,
                               lambda_weight=LAMBDAS[lam]())(labels, s, weights['item'])
    ref.backward()
    total, grad = refs.pairwise_loss(labels, scores, weights['item'], 'hinge',
                                     LAMBDAS[lam]())
    _close(total, ref.detach())
    _close(grad, s.grad)


@pytest.mark.parametrize('wkind', ['none', 'list', 'item'])
@pytest.mark.parametrize('n', [2, 100, 300])
def test_circle_reference_matches_oracle(wkind, n):
  """Scores straddle [0, 1] so that the clip passes some items and blocks others."""
  scores, labels, weights, _ = _case(5, n, seed=5 * n)
  scores = scores * 0.4 + 0.5
  labels[:, 0], labels[:, 1] = 2., 0.           # every list holds a valid pair
  s = scores.clone().requires_grad_()
  ref = LO.CircleLoss().compute(labels, s, weights[wkind], LO.Reduction.SUM)
  ref.backward()
  total, grad = refs.circle_loss(labels, scores, weights[wkind])
  _close(total, ref.detach())
  _close(grad, s.grad)


@pytest.mark.parametrize('n', [1, 100, 300])
def test_opa_reference_matches_oracle(n):
  from oracle import metrics_impl as MO
  scores, labels, weights, mask = _case(6, n, seed=n)
  w = weights['item'].clone()
  w[:, ::9] = 0.
  for ww, m in ((None, None), (w, None), (w, mask)):
    v, lw = refs.opa_metric(labels, scores, ww, m)
    rv, rw = MO.OPAMetric().compute(labels, scores, ww, m)
    _close(v, rv)
    _close(lw, rw)
