"""Per-list loss and metric kernels at every list-size dispatch boundary, up to the 8192-item
maximum (kMaxListSize, kMaxMetricListSize), against fp64 references.

Reference: the oracle up to N = 2048 (B <= 4).  Above that its [B, N, N] fp64 tensors are
replaced by the blocked restatements of tests/_list_refs.py (validated against the oracle by
tests/test_list_size_reference.py) for the approx and pairwise losses; sort-based metrics and
the O(N) losses stay on the oracle at every size.

Tolerances (those of test_parity_round2_gpu.py / test_parity_gpu.py):
  * losses: 1e-5 relative;
  * score gradients: per element |got - ref| <= 1e-5 |ref| + 1e-5 mean_list |ref|;
  * metrics: rtol 2e-5, atol 1e-6;
  * integer-valued outputs (ranks, MRR, Hits): exact.

Two bounds are looser, derived here:
  * approx-loss gradients: every entry is a sum of N terms (c_i - c_k) sigmoid'(z_k - z_i),
    each through ex2.approx and rcp.approx (about 2 ulp each).  An entry whose terms cancel
    can miss the per-element bound; as for the config-2 chunk of test_parity_round2_gpu.py,
    from N = 225 up, 1e-3 of the entries (the round-2 allowance), and never fewer than one
    entry, may miss it by at most 4x (measured: 1 entry in 900 .. 10240, by 1.04x .. 3.1x).
    Up to N = 224 the bound holds for every entry.
  * NeuralSort gradients at the largest accepted N (about 4000): the kernel forms every
    softmax exponent c_r s_k - D_k - max in fp64, so P is accurate to a few fp32 ulp; what is
    left is fp32 accumulation.  Each gradient entry is assembled from sequential fp32 sums of
    N terms (the column sums of the softmax backward, then sum_j H_j sign(s_j - s_m)), whose
    rounding error is at most (N - 1) 2^-24 times the sum of the terms' magnitudes, and those
    magnitudes are bounded by the largest gradient entry of the list times a small constant:
    rtol = N 2^-24 (2.4e-4 at N = 4005) against the largest entry, as test_parity_gpu.py
    measures gradients.
"""
import ctypes
import re

import pytest
import torch

import _list_refs as refs

pytestmark = pytest.mark.gpu

RTOL = 1e-5
ORACLE_MAX_N = 2048


def _batch(b, n, seed, pad=True, holes=False):
  g = torch.Generator().manual_seed(seed)
  scores = torch.randn(b, n, generator=g) * 2.0
  probs = torch.tensor([.55, .25, .12, .06, .02])
  labels = torch.multinomial(probs, b * n, replacement=True,
                             generator=g).reshape(b, n).float()
  if pad:
    lens = torch.randint((n + 1) // 2, n + 1, (b,), generator=g)
    labels = torch.where(torch.arange(n).unsqueeze(0) < lens.unsqueeze(1),
                         labels, torch.full_like(labels, -1.))
  if holes:   # padding in the middle of the list, not only at the tail
    drop = torch.rand(b, n, generator=g) < 0.2
    labels = torch.where(drop, torch.full_like(labels, -1.), labels)
  item_w = torch.rand(b, n, generator=g) + 0.5
  return scores, labels, item_w


def assert_grad_close(got, ref, rtol=RTOL, outliers=0.0):
  """Per element: |got - ref| <= rtol |ref| + rtol mean_list |ref|.  `outliers` > 0 lets that
  fraction of the entries miss the bound by up to 4x (full-size chunks: 12800 entries through
  MUFU-approximated exponentials)."""
  got = got.detach().double().cpu()
  ref = ref.detach().double().cpu()
  floor = rtol * ref.abs().mean(dim=-1, keepdim=True)
  ratio = (got - ref).abs() / (rtol * ref.abs() + floor + 1e-30)
  bad = ratio > 1
  msg = ('per-element gradient check failed on %d of %d entries; worst ratio %.2f, worst '
         '|d|=%.3e at ref=%.3e' %
         (int(bad.sum()), bad.numel(), float(ratio.max()), float((got - ref).abs().max()),
          float(ref.flatten()[(got - ref).abs().flatten().argmax()])))
  if outliers > 0:
    assert float(bad.double().mean()) <= outliers and float(ratio.max()) <= 4, msg
  else:
    assert not bool(bad.any()), msg


def _assert_loss_close(got, ref):
  got, ref = got.detach(), ref.detach()
  assert abs(float(got) - float(ref)) <= RTOL * max(1.0, abs(float(ref))), (
      float(got), float(ref))


def _check(cuda_loss, oracle_loss, scores, labels, weights):
  s_gpu = scores.cuda().requires_grad_()
  w_gpu = None if weights is None else weights.cuda()
  got = cuda_loss(labels.cuda(), s_gpu, w_gpu)
  got.backward()
  s_ref = scores.double().requires_grad_()
  w_ref = None if weights is None else weights.double()
  ref = oracle_loss(labels.double(), s_ref, w_ref)
  ref.backward()
  _assert_loss_close(got, ref)
  assert_grad_close(s_gpu.grad, s_ref.grad)


def _lists_for(n):
  """Lists per batch: the oracle's [B, N, N] tensors stay below ~1 GB."""
  return 4 if n <= 256 else 3 if n <= 1025 else 2 if n <= 4097 else 1


# ----------------------------------------------------------------------------
# ApproxNDCG / ApproxMRR: approx_loss_kernel<MODE, T>, T = ceil(N / 32) rounded up to
# 1, 2, 4, 7, 8, 16, 32; 224 threads for T <= 8, 256 above; T = 0 (generic loop) for N > 1024
# ----------------------------------------------------------------------------
APPROX_SIZES = {
    1: 'T1, 224 thr, one item', 32: 'T1 full', 33: 'T2 (first size with 2 col regs)',
    65: 'T4 (3 tiles in 4 regs)', 129: 'T7 (5 tiles)', 224: 'T7 full: N == threads',
    225: 'T8: N > threads (224)', 256: 'T8 full', 257: 'T16, 256 thr', 513: 'T32 (17 tiles)',
    1024: 'T32 full', 1025: 'T0 generic loop', 2048: 'T0, oracle at its limit',
    4097: 'T0, blocked reference', 8192: 'T0 at kMaxListSize'}


def _approx_case(mode, scores, labels, weights, mask, cuda_api, oracle_api):
  cls = 'ApproxNDCGLoss' if mode == 'ndcg' else 'ApproxMRRLoss'
  LC, LO = cuda_api.losses_impl, oracle_api.losses_impl
  s_gpu = scores.cuda().requires_grad_()
  got = getattr(LC, cls)(temperature=0.1).compute(
      labels.cuda(), s_gpu, None if weights is None else weights.cuda(), LC.Reduction.SUM,
      None if mask is None else mask.cuda())
  got.backward()
  n = scores.shape[1]
  if n <= ORACLE_MAX_N:
    s_ref = scores.double().requires_grad_()
    ref = getattr(LO, cls)(temperature=0.1).compute(
        labels.double(), s_ref, None if weights is None else weights.double(),
        LO.Reduction.SUM, mask)
    ref.backward()
    ref_grad = s_ref.grad
  else:
    ref, ref_grad, _ = refs.approx_loss(labels, scores, weights, mask, 0.1, mode)
  _assert_loss_close(got, ref)
  if n <= 224:
    assert_grad_close(s_gpu.grad, ref_grad)
  else:
    assert_grad_close(s_gpu.grad, ref_grad, outliers=max(1e-3, 1.0 / s_gpu.grad.numel()))


@pytest.mark.parametrize('n', sorted(APPROX_SIZES), ids=lambda n: '%d-%s' % (
    n, APPROX_SIZES[n].split(' ')[0].split(',')[0]))
@pytest.mark.parametrize('wkind', ['none', 'list', 'item'])
@pytest.mark.parametrize('mode', ['ndcg', 'mrr'])
def test_approx_sizes(cuda_api, oracle_api, mode, wkind, n):
  b = _lists_for(n)
  scores, labels, item_w = _batch(b, n, seed=7 * n + len(wkind))
  list_w = item_w[:, :1] + 0.25
  weights = {'none': None, 'list': list_w, 'item': item_w}[wkind]
  _approx_case(mode, scores, labels, weights, None, cuda_api, oracle_api)


@pytest.mark.parametrize('n', [200, 2048], ids=['T7', 'T0'])
@pytest.mark.parametrize('mode', ['ndcg', 'mrr'])
@pytest.mark.parametrize('use_mask', [False, True], ids=['labels', 'mask'])
def test_approx_edge_lists(cuda_api, oracle_api, mode, n, use_mask):
  """Holes inside lists; a list whose only valid item is its last; a fully padded list; a
  list with no positive label; with `mask`, a mask that disagrees with labels >= 0 (a padded
  label marked valid, valid labels masked out)."""
  scores, labels, item_w = _batch(5, n, seed=n + 1, holes=True)
  labels[1] = -1.
  labels[1, n - 1] = 2.                     # only the last item is valid
  labels[2] = -1.                           # fully padded
  labels[3] = torch.where(labels[3] >= 0, torch.zeros_like(labels[3]), labels[3])
  mask = None
  if use_mask:
    g = torch.Generator().manual_seed(n)
    mask = (labels >= 0) ^ (torch.rand(labels.shape, generator=g) < 0.1)
    mask[1] = False
    mask[1, n - 1] = True
  for weights in (None, item_w):
    _approx_case(mode, scores, labels, weights, mask, cuda_api, oracle_api)


# ----------------------------------------------------------------------------
# Pairwise losses: the both-ends pairwise_loss_kernel (N > 1024, and PairwiseMSELoss at any
# N); the triangular kernel (pairwise_tri.cu) at the first size of each packing
# ----------------------------------------------------------------------------
LAMBDAS = {
    'none': lambda K: None,
    'ndcg': lambda K: K.NDCGLambdaWeight(),
    'dcg_smooth': lambda K: K.DCGLambdaWeight(topn=20, smooth_fraction=0.4),
    'precision_top3': lambda K: K.PrecisionLambdaWeight(topn=3),
}
PHI = {'PairwiseLogisticLoss': 'logistic', 'PairwiseHingeLoss': 'hinge',
       'PairwiseSoftZeroOneLoss': 'soft_zero_one', 'PairwiseMSELoss': 'mse'}


def _pairwise_case(cls, lam, n, seed, cuda_api, oracle_api, temperature=0.8):
  b = _lists_for(n)
  scores, labels, item_w = _batch(b, n, seed=seed)
  KC, KO = cuda_api.keras_losses, oracle_api.keras_losses
  loss_c = getattr(KC, cls)(lambda_weight=LAMBDAS[lam](KC), temperature=temperature)
  if n <= ORACLE_MAX_N:
    loss_o = getattr(KO, cls)(lambda_weight=LAMBDAS[lam](KO), temperature=temperature)
    _check(loss_c, loss_o, scores, labels, item_w)
    return
  s_gpu = scores.cuda().requires_grad_()
  got = loss_c(labels.cuda(), s_gpu, item_w.cuda())
  got.backward()
  total, grad = refs.pairwise_loss(labels, scores, item_w, PHI[cls],
                                   LAMBDAS[lam](oracle_api.keras_losses), temperature)
  _assert_loss_close(got, total / (b * n))
  assert_grad_close(s_gpu.grad, grad / (b * n))


@pytest.mark.parametrize('n', [1025, 2048, 8192])
@pytest.mark.parametrize('lam', sorted(LAMBDAS))
@pytest.mark.parametrize('cls', ['PairwiseLogisticLoss', 'PairwiseHingeLoss',
                                 'PairwiseSoftZeroOneLoss'])
def test_pairwise_both_ends(cuda_api, oracle_api, cls, lam, n):
  _pairwise_case(cls, lam, n, 31 * n + len(lam), cuda_api, oracle_api)


@pytest.mark.parametrize('n', [1, 33, 257, 1024, 1025, 4096])
def test_pairwise_mse_both_ends(cuda_api, oracle_api, n):
  _pairwise_case('PairwiseMSELoss', 'none', n, n + 3, cuda_api, oracle_api)


@pytest.mark.parametrize('n', [65, 129, 256], ids=['65-64thr', '129-128thr', '256-256thr'])
@pytest.mark.parametrize('lam', ['none', 'ndcg', 'dcg_smooth'])
def test_pairwise_triangular_packing_boundaries(cuda_api, oracle_api, lam, n):
  _pairwise_case('PairwiseLogisticLoss', lam, n, 5 * n, cuda_api, oracle_api)


# ----------------------------------------------------------------------------
# The remaining per-list losses: one kernel each, shared memory grows with N
# ----------------------------------------------------------------------------
OTHER = {
    'softmax': lambda K: K.SoftmaxLoss(),
    'softmax_dcg': lambda K: K.SoftmaxLoss(lambda_weight=K.DCGLambdaWeight()),
    'list_mle': lambda K: K.ListMLELoss(),
    'sigmoid_ce': lambda K: K.SigmoidCrossEntropyLoss(),
    'mean_squared': lambda K: K.MeanSquaredLoss(),
    # [B, N, N] oracle and no blocked reference: UniqueSoftmax is checked up to N = 2048 only
    'unique_softmax': lambda K: K.UniqueSoftmaxLoss(),
}


@pytest.mark.parametrize('n', [1, 257, 1025, 4097, 8192])
@pytest.mark.parametrize('key', sorted(OTHER))
def test_other_losses_sizes(cuda_api, oracle_api, key, n):
  if key == 'unique_softmax' and n > ORACLE_MAX_N:
    pytest.skip('UniqueSoftmaxLoss has no reference above N = 2048 (oracle is [B, N, N])')
  scores, labels, item_w = _batch(2, n, seed=n + len(key), holes=True)
  _check(OTHER[key](cuda_api.keras_losses), OTHER[key](oracle_api.keras_losses), scores,
         labels, item_w)


@pytest.mark.parametrize('n', [1, 257, 1025, 4097, 8192])
def test_ordinal_loss_sizes(cuda_api, oracle_api, n):
  g = torch.Generator().manual_seed(n)
  scores = torch.randn(2, n, 3, generator=g)
  labels = torch.rand(2, n, generator=g) * 3.5
  labels[:, n // 2:] = torch.where(torch.rand(2, n - n // 2, generator=g) < 0.3,
                                   torch.full((2, n - n // 2), -1.), labels[:, n // 2:])
  item_w = torch.rand(2, n, generator=g) + 0.5
  _check(cuda_api.keras_losses.OrdinalLoss(ordinal_size=3),
         oracle_api.keras_losses.OrdinalLoss(ordinal_size=3), scores, labels, item_w)


def _neural_sort_limit():
  """The largest N the NeuralSort launcher accepts, from its own rejection message."""
  import ranking_b200 as tfr
  x = torch.zeros(1, 8192, device='cuda')
  with pytest.raises(ValueError) as e:
    tfr.losses_impl.NeuralSortCrossEntropyLoss().compute(x, x, None, tfr.losses_impl.Reduction.SUM)
  m = re.search(r'largest list_size accepted is (\d+)', str(e.value))
  assert m, str(e.value)
  return int(m.group(1))


@pytest.mark.parametrize('cls', ['NeuralSortCrossEntropyLoss', 'NeuralSortNDCGLoss'])
def test_neural_sort_at_its_limit(cuda_api, oracle_api, cls):
  """NeuralSort keeps 8 N floats of permutation rows in shared memory on top of the list:
  it runs at the largest N that fits the device's opt-in limit (values 1e-5, gradients see
  the module docstring)."""
  n_max = _neural_sort_limit()
  assert 1024 < n_max < 8192
  LC, LO = cuda_api.losses_impl, oracle_api.losses_impl
  scores, labels, item_w = _batch(1, n_max, seed=1)
  s_gpu = scores.cuda().requires_grad_()
  got = getattr(LC, cls)().compute(labels.cuda(), s_gpu, item_w.cuda(), LC.Reduction.SUM)
  got.backward()
  s_ref = scores.double().requires_grad_()
  ref = getattr(LO, cls)().compute(labels.double(), s_ref, item_w.double(), LO.Reduction.SUM)
  ref.backward()
  _assert_loss_close(got, ref)
  rtol = n_max * 2.0 ** -24
  err = float((s_gpu.grad.double().cpu() - s_ref.grad).abs().max() / s_ref.grad.abs().max())
  print('%s N=%d: gradient error %.2e of the largest entry (bound %.2e)' % (cls, n_max, err, rtol))
  assert err <= rtol, (err, rtol)


@pytest.mark.parametrize('cls', ['NeuralSortCrossEntropyLoss', 'NeuralSortNDCGLoss'])
def test_neural_sort_rejects_above_its_limit(cuda_api, cls):
  """N + 1 is an argument error that names the largest accepted N, raised before any launch."""
  import ranking_b200 as tfr
  n_max = _neural_sort_limit()
  over = torch.zeros(1, n_max + 1, device='cuda')
  LC = tfr.losses_impl
  with pytest.raises(ValueError, match='largest list_size accepted is %d' % n_max):
    getattr(LC, cls)().compute(over, over, None, LC.Reduction.SUM)


@pytest.mark.parametrize('n', [2, 257, 1025, 4097, 8192])
def test_circle_loss_sizes(cuda_api, oracle_api, n):
  """CircleLoss (gamma 64, margin 0.25): oracle up to 2048, the blocked reference above.
  N = 2 is the smallest list with a pair (a list without one has weight 0 / 0 = NaN).
  The pair sum S = sum e^(64 (alpha_i (1 - s_i - m) + alpha_j (s_j - m))) is formed in fp32,
  as in the reference, and overflows once a pair exponent passes ~88 - 2 ln N; scores are
  kept near 0.5 (pair exponents ~25) so that S is finite at N = 8192.  Two items per list sit
  outside [0, 1] so that the clip blocks their gradient; they carry the top and the bottom
  label, so that their large factors (e^60 at s = 0 as the higher item, at s = 1 as the lower)
  never enter a pair."""
  scores, labels, item_w = _batch(2, n, seed=n + 11, holes=True)
  scores = scores * 0.05 + 0.5
  labels[:, 0], labels[:, 1] = 2., 0.
  if n > 3:
    scores[:, 2], scores[:, 3] = 1.3, -0.2
    labels[:, 2], labels[:, 3] = 5., 0.
  LC, LO = cuda_api.losses_impl, oracle_api.losses_impl
  for w in (None, item_w):
    s_gpu = scores.cuda().requires_grad_()
    got = LC.CircleLoss().compute(labels.cuda(), s_gpu, None if w is None else w.cuda(),
                                  LC.Reduction.SUM)
    got.backward()
    if n <= ORACLE_MAX_N:
      s_ref = scores.double().requires_grad_()
      ref = LO.CircleLoss().compute(labels.double(), s_ref,
                                    None if w is None else w.double(), LO.Reduction.SUM)
      ref.backward()
      ref_grad = s_ref.grad
    else:
      ref, ref_grad = refs.circle_loss(labels, scores, w)
    _assert_loss_close(got, ref)
    assert_grad_close(s_gpu.grad, ref_grad)


def _hash_uniforms(seed, numel):
  """The uniforms of tfr_gumbel_sample (include/tfr_b200.h)."""
  import numpy as np
  with np.errstate(over='ignore'):
    idx = np.arange(numel, dtype=np.uint64)
    z = np.uint64(seed) + np.uint64(0x9E3779B97F4A7C15) * (idx + np.uint64(1))
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z = z ^ (z >> np.uint64(31))
  return torch.from_numpy((z >> np.uint64(40)).astype(np.float32) *
                          np.float32(1.0 / 16777216.0))


@pytest.mark.parametrize('n', [1, 257, 1025, 4097, 8192])
def test_gumbel_sampler_sizes(cuda_api, oracle_api, n):
  """Sampled logits and their backward against the oracle on the same uniforms (tolerances
  of test_parity_gpu.py::test_gumbel_sampler)."""
  b, s_ = 2, 3
  scores, labels, item_w = _batch(b, n, seed=40 + n, holes=True)
  smp = cuda_api.losses_impl.GumbelSampler(sample_size=s_, temperature=0.7, seed=123)
  sc = scores.cuda().requires_grad_()
  el, sl, ew = smp.sample(labels.cuda(), sc, item_w.cuda())
  u = _hash_uniforms((123 << 32) | 1, b * s_ * n).reshape(b, s_, n)
  so = scores.double().requires_grad_()
  rl, rs, rw = oracle_api.losses_impl.GumbelSampler(sample_size=s_, temperature=0.7).sample(
      labels.double(), so, item_w.double(), uniforms=u.double())
  assert torch.equal(el.cpu().double(), rl)
  torch.testing.assert_close(ew.cpu().double(), rw)
  valid = rl >= 0
  torch.testing.assert_close(sl.detach().cpu().double()[valid], rs.detach()[valid],
                             rtol=1e-5, atol=2e-5)
  up = torch.randn(b * s_, n, generator=torch.Generator().manual_seed(n)).double() * valid
  (sl * up.float().cuda()).sum().backward()
  (rs * up).sum().backward()
  err = float((sc.grad.double().cpu() - so.grad).abs().max() / (so.grad.abs().max() + 1e-30))
  assert err <= 2e-5 or float(so.grad.abs().max()) < 1e-12, err


# ----------------------------------------------------------------------------
# Metrics: bitonic sort over P = next power of two >= N, 13-bit index field in the sort key
# ----------------------------------------------------------------------------
METRIC_SIZES = [1, 2, 255, 256, 257, 1024, 1025, 4096, 4097, 5715, 5716, 8192]
EXT_CLASSES = ['HitsMetric', 'RecallMetric', 'PrecisionMetric', 'MeanAveragePrecisionMetric',
               'DCGMetric', 'BPrefMetric']


def _metric_batch(n, seed):
  scores, labels, item_w = _batch(2, n, seed=seed)
  labels[1] = 0.
  labels[1, n - 1] = 1.            # the only relevant item is the last: index bit 12 at 8192
  return scores, labels, item_w


def _metric_close(got, ref):
  torch.testing.assert_close(got.cpu().double(), ref.double(), rtol=2e-5, atol=1e-6)


@pytest.mark.parametrize('n', METRIC_SIZES, ids=lambda n: '%d-P%d' % (n, 1 << (n - 1).bit_length()))
def test_rank_metrics_sizes(cuda_api, oracle_api, n):
  """NDCG / MRR (plain launch) and every extended output, each with topns beyond N."""
  MC, MO = cuda_api.metrics_impl, oracle_api.metrics_impl
  scores, labels, item_w = _metric_batch(n, seed=n)
  topns = (1, 3, 10, n, n + 5, None)
  yc, sc, wc = labels.cuda(), scores.cuda(), item_w.cuda()
  y64, s64, w64 = labels.double(), scores.double(), item_w.double()
  for t, topn in enumerate(topns):
    for cls in ['NDCGMetric', 'MRRMetric'] + EXT_CLASSES:
      v, w = getattr(MC, cls)(topn=topn).compute(yc, sc, wc)
      rv, rw = getattr(MO, cls)(topn=topn).compute(y64, s64, w64)
      _metric_close(v, rv)
      _metric_close(w, rw)
      if cls == 'MRRMetric':     # 1 / rank of an exact position
        assert torch.equal(v.cpu(), rv.float()), (topn, v.cpu(), rv)
  for cls in ('ARPMetric', 'OPAMetric'):
    v, w = getattr(MC, cls)().compute(yc, sc, wc)
    if cls == 'OPAMetric' and n > ORACLE_MAX_N:   # the oracle's OPA materialises [B, N, N]
      rv, rw = refs.opa_metric(y64, s64, w64)
    else:
      rv, rw = getattr(MO, cls)().compute(y64, s64, w64)
    _metric_close(v, rv)
    torch.testing.assert_close(w.cpu().double(), rw, rtol=2e-5, atol=1e-5)
  # one launch with every extended output equals the single-output launches
  allx = MC.rank_metrics(yc, sc, wc, None, topns, ext=MC._EXT_KEYS)
  for key, cls in (('hits', 'HitsMetric'), ('recall', 'RecallMetric'),
                   ('precision', 'PrecisionMetric'), ('map', 'MeanAveragePrecisionMetric')):
    for t, topn in enumerate(topns):
      v, _ = getattr(MC, cls)(topn=topn).compute(yc, sc, wc)
      assert torch.equal(allx[key][:, t], v[:, 0]), (key, topn)
  plain = MC.rank_metrics(yc, sc, wc, None, topns)
  assert torch.equal(allx['ndcg'], plain['ndcg']) and torch.equal(allx['mrr'], plain['mrr'])


@pytest.mark.parametrize('n', METRIC_SIZES, ids=lambda n: '%d-P%d' % (n, 1 << (n - 1).bit_length()))
def test_diversity_metrics_sizes(cuda_api, oracle_api, n):
  g = torch.Generator().manual_seed(n)
  s_ = 3
  scores = torch.randn(2, n, generator=g)
  labels = (torch.rand(2, n, s_, generator=g) < 0.2).float()
  labels[:, -max(1, n // 7):] = -1.
  labels[1] = 0.
  labels[1, n - 1, 1] = 1.
  item_w = torch.rand(2, n, generator=g) + 0.2
  MC, MO = cuda_api.metrics_impl, oracle_api.metrics_impl
  for topn in (1, 10, n + 5, None):
    for cls, kw in (('PrecisionIAMetric', {}), ('AlphaDCGMetric', dict(alpha=0.3))):
      v, lw = getattr(MC, cls)(topn=topn, **kw).compute(labels.cuda(), scores.cuda(),
                                                        item_w.cuda())
      rv, rw = getattr(MO, cls)(topn=topn, **kw).compute(labels.double(), scores.double(),
                                                         item_w.double())
      _metric_close(v, rv)
      _metric_close(lw, rw)


def test_sorted_ranks_at_max_list_size(cuda_api, oracle_api):
  scores, labels, _ = _batch(2, 8192, seed=3, holes=True)
  got = cuda_api.utils.sorted_ranks(scores.cuda(), labels.cuda())
  ref = oracle_api.losses_impl._compute_ranks(scores.double(), labels >= 0)
  assert torch.equal(got.cpu().long(), ref)


# ----------------------------------------------------------------------------
# Ties: integer-valued outputs follow the oracle's index-stable order exactly
# ----------------------------------------------------------------------------
def _tied_batch(n, kind, seed):
  scores, labels, item_w = _batch(2, n, seed=seed)
  if kind == 'grid':
    scores = torch.round(scores * 2.) / 2.
  elif kind == 'signed_zero':
    g = torch.Generator().manual_seed(seed)
    z = torch.where(torch.rand(2, n, generator=g) < 0.5, torch.tensor(-0.0), torch.tensor(0.0))
    scores = torch.where(torch.rand(2, n, generator=g) < 0.6, z, scores)
  else:   # circular padding: the tail repeats the leading items, score and label
    k = max(1, n // 3)
    labels = labels.clamp(min=0.)
    labels[:, n - k:] = labels[:, :k]
    scores[:, n - k:] = scores[:, :k]
  return scores, labels, item_w


@pytest.mark.parametrize('n', [100, 1025, 8192])
@pytest.mark.parametrize('kind', ['grid', 'signed_zero', 'tail_copies'])
def test_ties_exact(cuda_api, oracle_api, kind, n):
  scores, labels, item_w = _tied_batch(n, kind, seed=n)
  yc, sc = labels.cuda(), scores.cuda()
  got = cuda_api.utils.sorted_ranks(sc, yc)
  ref = oracle_api.losses_impl._compute_ranks(scores.double(), labels >= 0)
  assert torch.equal(got.cpu().long(), ref)
  MC, MO = cuda_api.metrics_impl, oracle_api.metrics_impl
  for topn in (1, 3, None):
    v, _ = MC.MRRMetric(topn=topn).compute(yc, sc, None)
    rv, _ = MO.MRRMetric(topn=topn).compute(labels.double(), scores.double(), None)
    assert torch.equal(v.cpu(), rv.float()), (topn, v.cpu(), rv)
    v, _ = MC.HitsMetric(topn=topn).compute(yc, sc, None)
    rv, _ = MO.HitsMetric(topn=topn).compute(labels.double(), scores.double(), None)
    assert torch.equal(v.cpu(), rv.float()), (topn, v.cpu(), rv)
    v, _ = MC.NDCGMetric(topn=topn).compute(yc, sc, item_w.cuda())
    rv, _ = MO.NDCGMetric(topn=topn).compute(labels.double(), scores.double(),
                                             item_w.double())
    _metric_close(v, rv)


# ----------------------------------------------------------------------------
# Error state: a failed CUDA call must not be reported again by the next launch
# ----------------------------------------------------------------------------
def test_failed_cuda_call_does_not_poison_next_launch(cuda_api, oracle_api):
  """tfr_dp_free on a host address fails inside the runtime (cudaFree rejects it).  The very
  next CUDA work is a tfr launch of a different kernel, on tensors prepared before the failing
  call, so its own launch check is the one that would see a stale error: it must return 0 and
  the ranks must be right."""
  from ranking_b200 import _C
  scores, labels, _ = _batch(3, 300, seed=2)
  s, l = scores.cuda().contiguous(), labels.cuda().contiguous()
  ranks = torch.zeros(3, 300, dtype=torch.int32, device='cuda')
  torch.cuda.synchronize()
  host = ctypes.create_string_buffer(64)
  assert _C.lib.tfr_dp_free(ctypes.cast(host, ctypes.c_void_p)) != 0
  assert 'cudaFree' in _C.last_error()
  rc = _C.lib.tfr_sorted_ranks(_C.ptr(s), _C.ptr(l), None, 3, 300, _C.ptr(ranks), _C.stream())
  assert rc == 0, _C.last_error()
  ref = oracle_api.losses_impl._compute_ranks(scores.double(), labels >= 0)
  assert torch.equal(ranks.cpu().long(), ref)
