"""GPU parity tests: CUDA path (through the C ABI) vs the CPU oracle on the same
seeded inputs.  Tolerance for floating point: 1e-5 relative (the north_star
bar) on losses and on gradients relative to the largest gradient entry of the
batch; ranks and NDCG permutations must agree exactly on tie-free scores.
"""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

RTOL = 1e-5


def _batch(b, n, seed, pad=True, zero_rows=True):
  g = torch.Generator().manual_seed(seed)
  scores = torch.randn(b, n, generator=g) * 2.0
  probs = torch.tensor([.55, .25, .12, .06, .02])
  labels = torch.multinomial(probs, b * n, replacement=True,
                             generator=g).reshape(b, n).float()
  if pad:
    lens = torch.randint((n + 1) // 2, n + 1, (b,), generator=g)
    labels = torch.where(torch.arange(n).unsqueeze(0) < lens.unsqueeze(1),
                         labels, torch.full_like(labels, -1.))
  if zero_rows and b >= 4:
    labels[1] = torch.where(labels[1] >= 0, torch.zeros_like(labels[1]),
                            labels[1])       # a list without relevant items
    labels[2] = -1.                          # a fully padded list
  item_w = torch.rand(b, n, generator=g) + 0.5
  list_w = torch.rand(b, 1, generator=g) + 0.5
  return scores, labels, item_w, list_w


def _rel_err(got, ref):
  got = got.detach().double().cpu()
  ref = ref.detach().double().cpu()
  return float((got - ref).abs().max() / (ref.abs().max() + 1e-30))


def _check_loss_and_grad(cuda_loss, oracle_loss, scores, labels, weights):
  s_gpu = scores.cuda().requires_grad_()
  w_gpu = None if weights is None else weights.cuda()
  got = cuda_loss(labels.cuda(), s_gpu, w_gpu)
  got.backward()
  s_ref = scores.double().requires_grad_()
  w_ref = None if weights is None else weights.double()
  ref = oracle_loss(labels.double(), s_ref, w_ref)
  ref.backward()
  assert abs(float(got.detach()) - float(ref.detach())) <= RTOL * max(
      1.0, abs(float(ref.detach()))), (float(got.detach()), float(ref.detach()))
  if float(s_ref.grad.abs().max()) > 0:
    err = _rel_err(s_gpu.grad, s_ref.grad)
    assert err <= RTOL, err
  else:
    assert float(s_gpu.grad.abs().max()) <= 1e-6


LAMBDAS = {
    'none': lambda K: None,
    'label_diff': lambda K: K.LabelDiffLambdaWeight(),
    'dcg': lambda K: K.DCGLambdaWeight(),
    'ndcg': lambda K: K.NDCGLambdaWeight(),
    'ndcg_smooth_top5': lambda K: K.NDCGLambdaWeight(topn=5, smooth_fraction=0.25),
    'ndcg_v2_top5': lambda K: K.NDCGLambdaWeightV2(topn=5),
    'yeti': lambda K: K.YetiDCGLambdaWeight(topn=4, normalized=True),
    'precision_top3': lambda K: K.PrecisionLambdaWeight(topn=3),
}


@pytest.mark.parametrize('cls', ['PairwiseLogisticLoss', 'PairwiseHingeLoss',
                                 'PairwiseSoftZeroOneLoss', 'PairwiseMSELoss'])
@pytest.mark.parametrize('lam', sorted(LAMBDAS))
@pytest.mark.parametrize('wkind', ['none', 'list', 'item'])
def test_pairwise_loss_and_grad(cuda_api, oracle_api, cls, lam, wkind):
  scores, labels, item_w, list_w = _batch(6, 37, seed=11)
  weights = {'none': None, 'list': list_w, 'item': item_w}[wkind]
  KC, KO = cuda_api.keras_losses, oracle_api.keras_losses
  loss_c = getattr(KC, cls)(lambda_weight=LAMBDAS[lam](KC), temperature=0.7)
  loss_o = getattr(KO, cls)(lambda_weight=LAMBDAS[lam](KO), temperature=0.7)
  _check_loss_and_grad(loss_c, loss_o, scores, labels, weights)


@pytest.mark.parametrize('cls', ['ApproxNDCGLoss', 'ApproxMRRLoss', 'SoftmaxLoss'])
@pytest.mark.parametrize('wkind', ['none', 'list', 'item'])
@pytest.mark.parametrize('n', [1, 5, 64, 200])
def test_listwise_loss_and_grad(cuda_api, oracle_api, cls, wkind, n):
  scores, labels, item_w, list_w = _batch(8, n, seed=5 + n)
  weights = {'none': None, 'list': list_w, 'item': item_w}[wkind]
  loss_c = getattr(cuda_api.keras_losses, cls)()
  loss_o = getattr(oracle_api.keras_losses, cls)()
  _check_loss_and_grad(loss_c, loss_o, scores, labels, weights)


@pytest.mark.parametrize('cls', ['UniqueSoftmaxLoss', 'ListMLELoss',
                                 'SigmoidCrossEntropyLoss', 'MeanSquaredLoss'])
@pytest.mark.parametrize('wkind', ['none', 'list', 'item'])
@pytest.mark.parametrize('n', [1, 5, 64, 200, 700])
def test_more_losses_and_grad(cuda_api, oracle_api, cls, wkind, n):
  """K3b: the remaining RankingLossKey members against the oracle (values and
  gradients, Keras SUM_OVER_BATCH_SIZE reduction)."""
  scores, labels, item_w, list_w = _batch(6, n, seed=17 + n)
  weights = {'none': None, 'list': list_w, 'item': item_w}[wkind]
  loss_c = getattr(cuda_api.keras_losses, cls)()
  loss_o = getattr(oracle_api.keras_losses, cls)()
  _check_loss_and_grad(loss_c, loss_o, scores, labels, weights)


def test_list_mle_lambda_weight_and_temperature(cuda_api, oracle_api):
  scores, labels, item_w, _ = _batch(5, 40, seed=23)
  KC, KO = cuda_api.keras_losses, oracle_api.keras_losses
  disc = lambda r: 1. / torch.log1p(r)
  _check_loss_and_grad(
      KC.ListMLELoss(lambda_weight=KC.ListMLELambdaWeight(rank_discount_fn=disc),
                     temperature=0.5),
      KO.ListMLELoss(lambda_weight=KO.ListMLELambdaWeight(rank_discount_fn=disc),
                     temperature=0.5), scores, labels, item_w)
  _check_loss_and_grad(KC.UniqueSoftmaxLoss(temperature=2.0),
                       KO.UniqueSoftmaxLoss(temperature=2.0), scores, labels, None)
  for w in (None, item_w, item_w[:, :1]):
    _check_loss_and_grad(KC.CalibratedSoftmaxLoss(virtual_label=0.7),
                         KO.CalibratedSoftmaxLoss(virtual_label=0.7), scores, labels, w)


@pytest.mark.parametrize('key', ['unique_softmax_loss', 'list_mle_loss',
                                 'sigmoid_cross_entropy_loss', 'mean_squared_loss'])
def test_fused_train_step_more_losses(oracle_api, key):
  """RankingTrainer with the K3b losses: one Adagrad step equals the oracle's."""
  import ranking_b200 as tfr
  b, n, d, hidden = 8, 10, 16, [24]
  tower, params = _tower_and_params(tfr, d, hidden, 1, seed=5)
  trainer = tfr.train.RankingTrainer(tower, tfr.keras.losses.get(key),
                                     optimizer='sgd', learning_rate=0.1)
  g = torch.Generator().manual_seed(4)
  x = torch.randn(b, n, d, generator=g)
  y = torch.randint(0, 4, (b, n), generator=g).float()
  y[:, -3:] = -1.0
  w = torch.rand(b, 1, generator=g) + 0.5
  got = float(trainer.train_step(x.cuda(), y.cuda(), sample_weight=w.cuda()))
  flat = oracle_api.scorer.tower_forward(x.double().reshape(b * n, d), params,
                                         activation='relu')
  logits = oracle_api.scorer.restore_list(flat, y >= 0)
  ol = oracle_api.keras_losses.get(key)(y.double(), logits, w.double())
  ol.backward()
  assert got == pytest.approx(float(ol.detach()), rel=2e-5, abs=1e-6)
  want = torch.cat([torch.cat([(wt - 0.1 * wt.grad).reshape(-1),
                               (bs - 0.1 * bs.grad).reshape(-1)])
                    for wt, bs in zip(params['dense_w'], params['dense_b'])])
  assert _rel_err(tower.flat.detach(), want.detach()) <= 1e-5


@pytest.mark.parametrize('frac', [False, True])
def test_ordinal_loss_and_grad(cuda_api, oracle_api, frac):
  b, n, k = 5, 33, 4
  g = torch.Generator().manual_seed(3)
  scores = torch.randn(b, n, k, generator=g)
  labels = torch.rand(b, n, generator=g) * 4.5
  labels[:, -4:] = -1.0
  item_w = torch.rand(b, n, generator=g) + 0.5
  for w in (None, item_w, item_w[:, :1]):
    lc = cuda_api.keras_losses.OrdinalLoss(ordinal_size=k, use_fraction_label=frac)
    lo = oracle_api.keras_losses.OrdinalLoss(ordinal_size=k, use_fraction_label=frac)
    _check_loss_and_grad(lc, lo, scores, labels, w)


# ------------------------------ ragged=True ----------------------------------
@pytest.mark.parametrize('cls,expected_losses,expected_weights', [
    ('SigmoidCrossEntropyLoss', [1.3644443, -0.8190755], [9., 2.]),
    ('MeanSquaredLoss', [3.6666667, 1.], [9., 2.]),
    ('PairwiseHingeLoss', [1., 0.], [8., 1.]),
    ('PairwiseLogisticLoss', [0.813262, 0.126928], [8., 1.]),
    ('PairwiseSoftZeroOneLoss', [0.5, 0.119203], [8., 1.]),
    ('ListMLELoss', [3.534534, 0.126928], [4., 1.]),
    ('SoftmaxLoss', [1.407606, 0.126928], [4., 2.]),
    ('UniqueSoftmaxLoss', [1.407606, 0.380784], [4., 1.]),
    ('ApproxNDCGLoss', [-0.63093, -0.922917], [4., 1.]),
    ('ApproxMRRLoss', [-0.5, -0.893493], [4., 1.]),
])
def test_compute_per_list_with_ragged_inputs(cuda_api, cls, expected_losses,
                                             expected_weights):
  """losses_impl_test.py:556-578 with true ragged inputs (lists of sequences stand in
  for tf.RaggedTensor)."""
  scores = [[1., 3., 2.], [1., 3.]]
  labels = [[0., 0., 1.], [0., 2.]]
  per_item_weights = [[2., 3., 4.], [1., 1.]]
  loss_fn = getattr(cuda_api.losses_impl, cls)(name=None, ragged=True)
  losses, weights = loss_fn.compute_per_list(labels, scores, per_item_weights)
  torch.testing.assert_close(losses.cpu().double().reshape(-1),
                             torch.tensor(expected_losses, dtype=torch.float64),
                             rtol=1e-5, atol=1e-5)
  torch.testing.assert_close(weights.cpu().double().reshape(-1),
                             torch.tensor(expected_weights, dtype=torch.float64),
                             rtol=1e-5, atol=1e-5)


def test_metrics_with_ragged_inputs(cuda_api):
  """metrics_impl_test.py: the *_should_handle_ragged_inputs cases."""
  M = cuda_api.metrics_impl
  log2p1 = lambda x: math.log2(1. + x)

  def check(metric, labels, scores, want, want_w=None):
    v, w = metric.compute(labels, scores)
    torch.testing.assert_close(v.cpu().double(), torch.tensor(want, dtype=torch.float64),
                               rtol=1e-5, atol=1e-6)
    if want_w is not None:
      torch.testing.assert_close(w.cpu().double(),
                                 torch.tensor(want_w, dtype=torch.float64),
                                 rtol=1e-5, atol=1e-6)

  check(M.MRRMetric(topn=None, ragged=True), [[0., 1., 0.], [0., 1.]],
        [[1., 2., 3.], [1., 2.]], [[0.5], [1.]])
  check(M.HitsMetric(topn=1, ragged=True), [[0., 1., 0.], [0., 1.]],
        [[1., 2., 3.], [1., 2.]], [[0.], [1.]])
  check(M.ARPMetric(ragged=True), [[0., 0., 1., 0.], [0., 1., 2.]],
        [[1., 3., 2., 4.], [1., 2., 3.]], [[3.], [((1. * 2.) + (2. * 1.)) / (2. + 1.)]])
  check(M.PrecisionMetric(topn=None, ragged=True), [[0., 0., 1., 0.], [1., 0., 2.]],
        [[1., 3., 2., 4.], [1., 2., 3.]], [[1. / 4.], [2. / 3.]])
  check(M.MeanAveragePrecisionMetric(topn=None, ragged=True),
        [[0., 0., 1., 0.], [1., 1., 0.]], [[1., 4., 3., 2.], [1., 3., 2.]],
        [[(1. / 2.) / 1.], [(1. / 1. + 2. / 3.) / 2.]])
  check(M.DCGMetric(topn=None, ragged=True), [[0., 1., 0.], [1., 1., 0., 0.]],
        [[3., 2., 1.], [4., 1., 2., 3.]],
        [[1. / log2p1(2.)], [1. / log2p1(1.) + 1. / log2p1(4.)]])
  check(M.OPAMetric(ragged=True), [[0., 1., 0.], [1., 0., 1., 0.]],
        [[3., 2., 1.], [4., 1., 2., 3.]], [[1. / 2.], [3. / 4.]], [[2.], [4.]])
  # Keras objects (keras/losses.py docstrings :620-627, 1611-1618)
  K = cuda_api.keras_losses
  got = K.OrdinalLoss(ordinal_size=2, ragged=True)(
      [[2., 1.], [0.]], [[[0.6, 0.2], [0.8, 0.3]], [[0., -0.2]]])
  assert abs(float(got) - 0.88809216) < 1e-5


def _hash_uniforms(seed, numel):
  """The uniforms of tfr_gumbel_sample / dropout (include/tfr_b200.h)."""
  import numpy as np
  with np.errstate(over='ignore'):
    idx = np.arange(numel, dtype=np.uint64)
    z = np.uint64(seed) + np.uint64(0x9E3779B97F4A7C15) * (idx + np.uint64(1))
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z = z ^ (z >> np.uint64(31))
  return torch.from_numpy((z >> np.uint64(40)).astype(np.float32) *
                          np.float32(1.0 / 16777216.0))


@pytest.mark.parametrize('n', [1, 9, 200])
def test_gumbel_sampler(cuda_api, oracle_api, n):
  b, s_ = 5, 3
  scores, labels, item_w, _ = _batch(b, n, seed=40 + n)
  smp = cuda_api.losses_impl.GumbelSampler(sample_size=s_, temperature=0.7, seed=123)
  sc = scores.cuda().requires_grad_()
  el, sl, ew = smp.sample(labels.cuda(), sc, item_w.cuda())
  seed = (123 << 32) | 1
  u = _hash_uniforms(seed, b * s_ * n).reshape(b, s_, n)
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
  assert _rel_err(sc.grad, so.grad) <= 2e-5 or float(so.grad.abs().max()) < 1e-12


@pytest.mark.parametrize('key', ['yeti_logistic_loss', 'gumbel_approx_ndcg_loss'])
@pytest.mark.parametrize('wkind', ['none', 'list', 'item'])
def test_gumbel_losses(cuda_api, oracle_api, key, wkind):
  """YetiLogisticLoss / GumbelApproxNDCGLoss (keras/losses.py:609-718, 1241-1341) with
  the oracle fed the same uniforms; autograd path and fused training path."""
  b, n, s_ = 6, 30, 4
  scores, labels, item_w, list_w = _batch(b, n, seed=61)
  weights = {'none': None, 'list': list_w, 'item': item_w}[wkind]
  lc = cuda_api.keras_losses.get(key, sample_size=s_, seed=7)
  lo = oracle_api.keras_losses.get(key, sample_size=s_, seed=7)
  u = _hash_uniforms((7 << 32) | 1, b * s_ * n).reshape(b, s_, n).double()
  sc = scores.cuda().requires_grad_()
  wc = None if weights is None else weights.cuda()
  got = lc(labels.cuda(), sc, wc)
  got.backward()
  so = scores.double().requires_grad_()
  ref = lo(labels.double(), so, None if weights is None else weights.double(), uniforms=u)
  ref.backward()
  assert abs(float(got.detach()) - float(ref.detach())) <= 2e-5 * max(1., abs(float(ref.detach())))
  assert _rel_err(sc.grad, so.grad) <= 5e-5
  # fused path: same seed -> same numbers without autograd
  lc._gumbel_sampler._calls = 0
  grad = torch.empty(b, n, device='cuda')
  per_list = torch.empty(2, b, device='cuda')
  total2 = torch.zeros(2, device='cuda')
  lc.fused_fwd_bwd(labels.cuda(), scores.cuda(), wc, grad, per_list, total2)
  assert abs(float(total2[0]) - float(ref.detach())) <= 2e-5 * max(1., abs(float(ref.detach())))
  assert _rel_err(grad, so.grad) <= 5e-5


@pytest.mark.parametrize('topk', [None, 3])
@pytest.mark.parametrize('wkind', ['none', 'list', 'item'])
def test_coupled_rank_distil_loss(cuda_api, oracle_api, topk, wkind):
  """CoupledRankDistilLoss (keras/losses.py:1659-1750): teacher permutations from the
  counter-hash Gumbel noise, replayed through the oracle."""
  b, n, s_ = 5, 17, 3
  scores, labels, item_w, list_w = _batch(b, n, seed=71)
  labels[2] = torch.where(labels[2] >= 0, torch.zeros_like(labels[2]), labels[2])  # weight 0
  weights = {'none': None, 'list': list_w, 'item': item_w}[wkind]
  lc = cuda_api.keras_losses.CoupledRankDistilLoss(sample_size=s_, topk=topk, temperature=0.8)
  lo = oracle_api.keras_losses.CoupledRankDistilLoss(sample_size=s_, topk=topk,
                                                     temperature=0.8)
  lc._loss.seed(5)
  lo._loss.uniforms = _hash_uniforms((5 << 32) | 1, b * s_ * n).reshape(b, s_, n).double()
  _check_loss_and_grad(lc, lo, scores, labels, weights)


def test_softmax_with_dcg_lambda(cuda_api, oracle_api):
  scores, labels, item_w, _ = _batch(8, 50, seed=3)
  KC, KO = cuda_api.keras_losses, oracle_api.keras_losses
  _check_loss_and_grad(KC.SoftmaxLoss(lambda_weight=KC.NDCGLambdaWeight(topn=10)),
                       KO.SoftmaxLoss(lambda_weight=KO.NDCGLambdaWeight(topn=10)),
                       scores, labels, item_w)


def test_custom_gain_and_discount_tables(cuda_api, oracle_api):
  """User callables travel as tables (SURVEY.md §7 hard parts)."""
  scores, labels, _, _ = _batch(4, 21, seed=9)
  gain = lambda l: l * l + 0.5 * l
  disc = lambda r: 1. / (r + 3.)
  KC, KO = cuda_api.keras_losses, oracle_api.keras_losses
  _check_loss_and_grad(
      KC.PairwiseLogisticLoss(lambda_weight=KC.DCGLambdaWeight(
          gain_fn=gain, rank_discount_fn=disc, normalized=True,
          smooth_fraction=0.5)),
      KO.PairwiseLogisticLoss(lambda_weight=KO.DCGLambdaWeight(
          gain_fn=gain, rank_discount_fn=disc, normalized=True,
          smooth_fraction=0.5)), scores, labels, None)


@pytest.mark.parametrize('n', [32, 256, 1024])
def test_pairwise_logistic_list_size_sweep(cuda_api, oracle_api, n):
  """BASELINE config 5 sizes, checked on a few lists (the oracle materialises
  [B, N, N])."""
  scores, labels, _, _ = _batch(4, n, seed=n, zero_rows=False)
  _check_loss_and_grad(cuda_api.keras_losses.PairwiseLogisticLoss(),
                       oracle_api.keras_losses.PairwiseLogisticLoss(), scores,
                       labels, None)


def test_lambda_loss_config3_shape(cuda_api, oracle_api):
  """BASELINE config 3 list size (N=512) with NDCGLambdaWeight, few lists."""
  scores, labels, _, _ = _batch(3, 512, seed=21, zero_rows=False)
  KC, KO = cuda_api.keras_losses, oracle_api.keras_losses
  _check_loss_and_grad(KC.PairwiseLogisticLoss(lambda_weight=KC.NDCGLambdaWeight()),
                       KO.PairwiseLogisticLoss(lambda_weight=KO.NDCGLambdaWeight()),
                       scores, labels, None)


def test_reduction_none_and_row_gradients(cuda_api, oracle_api):
  scores, labels, item_w, _ = _batch(5, 19, seed=2)
  KC, KO = cuda_api.keras_losses, oracle_api.keras_losses
  up = torch.rand(5, 19)
  s_gpu = scores.cuda().requires_grad_()
  out = KC.PairwiseLogisticLoss(reduction=KC.Reduction.NONE)(
      labels.cuda(), s_gpu, item_w.cuda())
  (out * up.cuda()).sum().backward()
  s_ref = scores.double().requires_grad_()
  ref = KO.PairwiseLogisticLoss(reduction=KO.Reduction.NONE)(
      labels.double(), s_ref, item_w.double())
  (ref * up.double()).sum().backward()
  assert _rel_err(out, ref) <= RTOL
  assert _rel_err(s_gpu.grad, s_ref.grad) <= RTOL


def test_estimator_reductions(cuda_api, oracle_api):
  scores, labels, item_w, _ = _batch(6, 23, seed=4)
  LC, LO = cuda_api.losses_impl, oracle_api.losses_impl
  for red in ['SUM', 'MEAN', 'SUM_BY_NONZERO_WEIGHTS', 'SUM_OVER_BATCH_SIZE']:
    for cls in ['PairwiseLogisticLoss', 'ApproxNDCGLoss', 'SoftmaxLoss']:
      got = getattr(LC, cls)(name=None).compute(
          labels.cuda(), scores.cuda(), item_w.cuda(),
          getattr(LC.Reduction, red))
      ref = getattr(LO, cls)(name=None).compute(
          labels.double(), scores.double(), item_w.double(),
          getattr(LO.Reduction, red))
      assert abs(float(got) - float(ref)) <= RTOL * max(1., abs(float(ref))), (
          red, cls, float(got), float(ref))


def test_sorted_ranks_exact(cuda_api, oracle_api):
  scores, labels, _, _ = _batch(16, 100, seed=8)
  ranks = cuda_api.utils.sorted_ranks(scores.cuda(), labels.cuda())
  ref = oracle_api.losses_impl._compute_ranks(scores.double(), labels >= 0)
  assert torch.equal(ranks.cpu().long(), ref)
  # ties are broken by index
  tie = torch.tensor([[1., 2., 1., 2., 0.]])
  assert cuda_api.utils.sorted_ranks(tie.cuda()).tolist() == [[3, 1, 4, 2, 5]]


@pytest.mark.parametrize('n', [1, 7, 200, 777])
def test_rank_metrics(cuda_api, oracle_api, n):
  scores, labels, item_w, _ = _batch(16, n, seed=n)
  topns = (1, 3, 5, 10, None)
  for weights in (None, item_w):
    out = cuda_api.metrics_impl.rank_metrics(
        labels.cuda(), scores.cuda(), None if weights is None else weights.cuda(),
        None, topns)
    for t, topn in enumerate(topns):
      w64 = None if weights is None else weights.double()
      nd, ndw = oracle_api.metrics_impl.NDCGMetric(topn=topn).compute(
          labels.double(), scores.double(), w64)
      mr, mrw = oracle_api.metrics_impl.MRRMetric(topn=topn).compute(
          labels.double(), scores.double(), w64)
      torch.testing.assert_close(out['ndcg'][:, t].cpu().double(), nd[:, 0],
                                 rtol=1e-5, atol=1e-6)
      torch.testing.assert_close(out['mrr'][:, t].cpu().double(), mr[:, 0],
                                 rtol=1e-6, atol=0)  # 1/rank of an exact position
      torch.testing.assert_close(out['ndcg_w'].cpu().double(), ndw[:, 0],
                                 rtol=1e-5, atol=1e-6)
      torch.testing.assert_close(out['mrr_w'].cpu().double(), mrw[:, 0],
                                 rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize('n', [1, 7, 64, 200, 1000])
def test_rank_metrics_extended(cuda_api, oracle_api, n):
  """K4's extended outputs (Hits, ARP, Recall, Precision, MAP, DCG, OPA) on random
  batches with padding, ties, item weights (some zero) and an explicit mask."""
  scores, labels, item_w, _ = _batch(12, n, seed=100 + n)
  g = torch.Generator().manual_seed(n)
  item_w = torch.where(torch.rand(item_w.shape, generator=g) < 0.1,
                       torch.zeros_like(item_w), item_w)
  mask = (labels >= 0) & (torch.rand(labels.shape, generator=g) < 0.9)
  MO, MC = oracle_api.metrics_impl, cuda_api.metrics_impl
  for weights, m in ((None, None), (item_w, None), (item_w, mask)):
    w64 = None if weights is None else weights.double()
    wc = None if weights is None else weights.cuda()
    mc = None if m is None else m.cuda()
    for topn in (1, 5, None):
      for cls in ('HitsMetric', 'RecallMetric', 'PrecisionMetric',
                  'MeanAveragePrecisionMetric', 'DCGMetric'):
        v, w = getattr(MC, cls)(topn=topn).compute(labels.cuda(), scores.cuda(), wc, mc)
        rv, rw = getattr(MO, cls)(topn=topn).compute(labels.double(), scores.double(),
                                                     w64, m)
        torch.testing.assert_close(v.cpu().double(), rv, rtol=2e-5, atol=1e-6)
        torch.testing.assert_close(w.cpu().double(), rw, rtol=2e-5, atol=1e-6)
    for cls in ('ARPMetric', 'OPAMetric'):
      v, w = getattr(MC, cls)().compute(labels.cuda(), scores.cuda(), wc, mc)
      rv, rw = getattr(MO, cls)().compute(labels.double(), scores.double(), w64, m)
      torch.testing.assert_close(v.cpu().double(), rv, rtol=2e-5, atol=1e-6)
      torch.testing.assert_close(w.cpu().double(), rw, rtol=2e-5, atol=1e-5)


@pytest.mark.parametrize('n,s_', [(1, 1), (9, 3), (150, 7), (700, 2)])
def test_diversity_metrics(cuda_api, oracle_api, n, s_):
  g = torch.Generator().manual_seed(n + s_)
  b = 6
  scores = torch.randn(b, n, generator=g)
  scores = torch.round(scores * 4) / 4          # ties, broken by index on both sides
  labels = (torch.rand(b, n, s_, generator=g) < 0.3).float()
  labels[:, -max(1, n // 5):] = -1.0
  labels[1] = torch.where(labels[1] >= 0, torch.zeros_like(labels[1]), labels[1])  # no relevance
  item_w = torch.rand(b, n, generator=g) + 0.2
  MO, MC = oracle_api.metrics_impl, cuda_api.metrics_impl
  for w in (None, item_w):
    for topn in (1, 5, None):
      for cls, kw in (('PrecisionIAMetric', {}), ('AlphaDCGMetric', dict(alpha=0.3))):
        v, lw = getattr(MC, cls)(topn=topn, **kw).compute(
            labels.cuda(), scores.cuda(), None if w is None else w.cuda())
        rv, rw = getattr(MO, cls)(topn=topn, **kw).compute(
            labels.double(), scores.double(), None if w is None else w.double())
        torch.testing.assert_close(v.cpu().double(), rv, rtol=2e-5, atol=1e-6)
        torch.testing.assert_close(lw.cpu().double(), rw, rtol=2e-5, atol=1e-6)


def test_default_keras_metrics_one_launch(cuda_api, oracle_api):
  """`MetricGroup.default()` (one launch per batch) equals the eleven separate
  `default_keras_metrics()` objects (keras/metrics.py:131-153)."""
  MC = __import__('ranking_b200').keras.metrics
  scores, labels, item_w, _ = _batch(24, 50, seed=8)
  objs = MC.default_keras_metrics()
  assert [o.name for o in objs] == [
      'metric/ndcg_1', 'metric/ndcg_3', 'metric/ndcg_5', 'metric/ndcg_10', 'metric/arp',
      'metric/ordered_pair_accuracy', 'metric/mrr', 'metric/precision', 'metric/map',
      'metric/dcg', 'metric/ndcg']
  grp = MC.MetricGroup.default()
  for lo in (0, 12):
    y, s_, w = labels[lo:lo + 12].cuda(), scores[lo:lo + 12].cuda(), item_w[lo:lo + 12].cuda()
    for o in objs:
      o.update_state(y, s_, w)
    grp.update_state(y, s_, w)
  res = grp.result()
  for o in objs:
    assert abs(res[o.name] - float(o.result())) <= 1e-5 * max(1.0, abs(float(o.result()))), o.name


def test_keras_metric_objects(cuda_api, oracle_api):
  scores, labels, _, _ = _batch(32, 40, seed=77)
  MC = __import__('ranking_b200').keras.metrics
  m = MC.NDCGMetric(topn=10)
  m.update_state(labels[:16].cuda(), scores[:16].cuda())
  m.update_state(labels[16:].cuda(), scores[16:].cuda())
  ref = oracle_api.metrics_impl.KerasMean(
      oracle_api.metrics_impl.NDCGMetric(topn=10))
  ref.update_state(labels[:16].double(), scores[:16].double())
  ref.update_state(labels[16:].double(), scores[16:].double())
  assert abs(float(m.result()) - ref.result()) <= 1e-6
  # docstring example keras/metrics.py:729-733
  got = MC.NDCGMetric()(torch.tensor([[0., 1., 1.]]).cuda(),
                        torch.tensor([[3., 1., 2.]]).cuda())
  assert abs(float(got) - 0.6934264) < 1e-6
  grp = MC.MetricGroup()
  grp.update_state(labels.cuda(), scores.cuda())
  res = grp.result()
  m10 = MC.NDCGMetric(topn=10)
  m10.update_state(labels.cuda(), scores.cuda())
  assert abs(res['metric/ndcg_10'] - float(m10.result())) < 1e-6


# ------------------------------ scorer tower --------------------------------
def _tower_and_params(tfr, d, hidden, out, seed, activation='relu',
                      precision='fp32'):
  torch.manual_seed(seed)
  tower = tfr.keras.layers.create_tower(hidden, out, activation=activation,
                                        use_batch_norm=False, dropout=0,
                                        input_dim=d, seed=seed,
                                        precision=precision)
  with torch.no_grad():
    for i in range(len(tower.dims) - 1):
      tower.bias(i).uniform_(-0.2, 0.2)
  nl = len(tower.dims) - 1
  params = {
      'dense_w': [tower.kernel(i).detach().cpu().double().clone().requires_grad_()
                  for i in range(nl)],
      'dense_b': [tower.bias(i).detach().cpu().double().clone().requires_grad_()
                  for i in range(nl)]}
  return tower, params


def _flat_grad(params):
  return torch.cat([torch.cat([w.grad.reshape(-1), b.grad.reshape(-1)])
                    for w, b in zip(params['dense_w'], params['dense_b'])])


@pytest.mark.parametrize('shape', [
    (300, 136, [256, 128, 64], 1, 'relu'),
    (1000, 17, [33, 9], 1, 'relu'),
    (257, 40, [], 1, None),          # linear scorer, no hidden layer
    (513, 24, [48], 2, None),        # two outputs (groupwise scoring), identity act
    (4100, 136, [256, 128, 64], 1, 'relu'),   # crosses the row-split boundary
])
def test_tower_forward_backward(oracle_api, shape):
  import ranking_b200 as tfr
  m, d, hidden, out, act = shape
  tower, params = _tower_and_params(tfr, d, hidden, out, seed=m, activation=act)
  g = torch.Generator().manual_seed(m)
  x = torch.randn(m, d, generator=g)
  up = torch.randn(m, out, generator=g)
  y = tower(x.cuda())
  (y * up.cuda()).sum().backward()
  ref = oracle_api.scorer.tower_forward(x.double(), params, activation=act)
  (ref * up.double()).sum().backward()
  assert _rel_err(y, ref) <= RTOL
  assert _rel_err(tower.flat.grad, _flat_grad(params)) <= 5e-5


@pytest.mark.parametrize('precision,tol_fwd,tol_bwd', [('tf32x3', 1e-5, 5e-5),
                                                       ('tf32', 5e-3, 0.15)])
@pytest.mark.parametrize('shape', [
    (300, 136, [256, 128, 64], 1, 'relu'),
    (4100, 136, [256, 128, 64], 1, 'relu'),    # several row splits
    (1000, 16, [32, 8], 1, 'relu'),
    (513, 24, [48], 2, None),
    # N tile > 256 columns.  Identity activation: with ReLU a pre-activation within
    # rounding distance of 0 flips its mask and moves one dW entry by ~1e-3, which
    # says nothing about the GEMMs (3.3M hidden units here).
    (6400, 256, [512, 64], 1, None),
])
def test_tower_tensor_core_path(oracle_api, shape, precision, tol_fwd, tol_bwd):
  """Tensor-core scorer path: 3xTF32 must stay fp32-faithful (1e-5), TF32 is looser.

  With ReLU, a hidden pre-activation that lies within rounding distance of zero
  can take the other branch than in the fp64 oracle; that moves a handful of
  gradient entries by O(1e-3) and is a property of ReLU, not of the GEMMs.  The
  gradient check therefore uses the relative L2 error for ReLU towers and the
  max-norm error for identity towers."""
  import ranking_b200 as tfr
  torch.manual_seed(1234)
  m, d, hidden, out, act = shape
  tower, params = _tower_and_params(tfr, d, hidden, out, seed=m, activation=act,
                                    precision=precision)
  g = torch.Generator().manual_seed(m)
  x = torch.randn(m, d, generator=g)
  up = torch.randn(m, out, generator=g)
  y = tower(x.cuda())
  (y * up.cuda()).sum().backward()
  ref = oracle_api.scorer.tower_forward(x.double(), params, activation=act)
  (ref * up.double()).sum().backward()
  assert _rel_err(y, ref) <= tol_fwd, _rel_err(y, ref)
  got, want = tower.flat.grad.detach().cpu().double(), _flat_grad(params)
  if act is None:
    assert _rel_err(got, want) <= tol_bwd, _rel_err(got, want)
  else:
    l2 = float((got - want).norm() / want.norm())
    assert l2 <= tol_bwd, l2
    assert _rel_err(got, want) <= max(100 * tol_bwd, 5e-3)


# ---------------------- BatchNormalization / Dropout ------------------------
def _bn_tower_and_params(tfr, d, hidden, out, seed, activation, precision,
                         input_bn, use_bn, dropout=0.0, moment=0.9):
  tower = tfr.keras.layers.create_tower(
      hidden, out, activation=activation, input_batch_norm=input_bn,
      use_batch_norm=use_bn, batch_norm_moment=moment, dropout=dropout,
      input_dim=d, seed=seed, precision=precision)
  g = torch.Generator().manual_seed(seed + 7)
  with torch.no_grad():
    for i in range(len(tower.dims) - 1):
      tower.bias(i).copy_(torch.rand(tower.dims[i + 1], generator=g) * 0.4 - 0.2)
    for key in tower.bn_offsets:
      w = tower.bn_offsets[key][2]
      tower.bn_gamma(key).copy_(torch.rand(w, generator=g) + 0.5)
      tower.bn_beta(key).copy_(torch.rand(w, generator=g) * 0.6 - 0.3)
  nl = len(tower.dims) - 1
  dbl = lambda t: t.detach().cpu().double().clone().requires_grad_()
  params = {'dense_w': [dbl(tower.kernel(i)) for i in range(nl)],
            'dense_b': [dbl(tower.bias(i)) for i in range(nl)],
            'bn_gamma': [], 'bn_beta': [], 'in_bn_gamma': None, 'in_bn_beta': None}
  if input_bn:
    params['in_bn_gamma'] = dbl(tower.bn_gamma('input'))
    params['in_bn_beta'] = dbl(tower.bn_beta('input'))
  if use_bn:
    params['bn_gamma'] = [dbl(tower.bn_gamma(i)) for i in range(len(hidden))]
    params['bn_beta'] = [dbl(tower.bn_beta(i)) for i in range(len(hidden))]
  return tower, params


def _bn_flat_grad(params, zero=False):
  parts = []
  for w, b in zip(params['dense_w'], params['dense_b']):
    parts += [w.grad.reshape(-1), b.grad.reshape(-1)]
  if params['in_bn_gamma'] is not None:
    parts += [params['in_bn_gamma'].grad, params['in_bn_beta'].grad]
  for g_, b_ in zip(params['bn_gamma'], params['bn_beta']):
    parts += [g_.grad, b_.grad]
  return torch.cat(parts)


@pytest.mark.parametrize('precision,tol', [('fp32', 2e-5), ('tf32x3', 5e-5)])
@pytest.mark.parametrize('shape', [
    # m, d, hidden, out, act, input_bn, use_bn
    (700, 136, [256, 128, 64], 1, 'relu', True, True),     # reference defaults
    (700, 136, [256, 128, 64], 1, 'relu', False, True),
    (1300, 24, [48, 16], 1, None, True, False),
    (515, 40, [], 1, None, True, False),                    # linear scorer + input BN
    (4200, 64, [128], 2, None, True, True),
])
def test_tower_batch_norm_training(oracle_api, shape, precision, tol):
  """create_tower with BatchNormalization in training mode
  (keras/layers.py:67-72): batch statistics, parameter gradients of Dense and
  BN layers, and the moving-average update."""
  import ranking_b200 as tfr
  m, d, hidden, out, act, input_bn, use_bn = shape
  tower, params = _bn_tower_and_params(tfr, d, hidden, out, m, act, precision,
                                       input_bn, use_bn)
  g = torch.Generator().manual_seed(m)
  x = torch.randn(m, d, generator=g) * 1.5 + 0.3
  up = torch.randn(m, out, generator=g)
  moving = oracle_api.scorer.init_bn_moving(d, hidden, input_bn, use_bn,
                                            dtype=torch.float64)
  tower.train()
  y = tower(x.cuda())
  (y * up.cuda()).sum().backward()
  ref = oracle_api.scorer.tower_forward(
      x.double(), params, activation=act, use_batch_norm=use_bn and bool(hidden),
      input_batch_norm=input_bn, training=True, bn_moving=moving, momentum=0.9)
  (ref * up.double()).sum().backward()
  assert _rel_err(y, ref) <= tol, _rel_err(y, ref)
  got, want = tower.flat.grad.detach().cpu().double(), _bn_flat_grad(params)
  if act is None:
    assert _rel_err(got, want) <= 10 * tol, _rel_err(got, want)
  else:
    # One ReLU input within rounding distance of 0 may take the other branch than in
    # the fp64 oracle; through BN's batch coupling a single flip moves the whole
    # gradient by O(1/sqrt(M)) of one column (measured 3e-3 at M = 700).  The
    # identity-activation cases above pin the BN arithmetic to 1e-4.
    l2 = float((got - want).norm() / want.norm())
    assert l2 <= 1e-2, l2
  for key, (mean, var) in moving.items():
    gm, gv = tower.bn_moving(key)
    assert _rel_err(gm, mean) <= 1e-5
    assert _rel_err(gv, var) <= 1e-5


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
def test_tower_batch_norm_inference(oracle_api, precision):
  """eval(): moving statistics normalise, nothing is updated; gradients flow
  through the frozen statistics."""
  import ranking_b200 as tfr
  m, d, hidden = 600, 32, [64, 16]
  tower, params = _bn_tower_and_params(tfr, d, hidden, 1, 3, None, precision,
                                       True, True)
  g = torch.Generator().manual_seed(5)
  moving = oracle_api.scorer.init_bn_moving(d, hidden, True, True,
                                            dtype=torch.float64)
  with torch.no_grad():
    for key, (mean, var) in moving.items():
      mean.copy_(torch.randn(mean.shape, generator=g) * 0.3)
      var.copy_(torch.rand(var.shape, generator=g) + 0.5)
      gm, gv = tower.bn_moving(key)
      gm.copy_(mean.float())
      gv.copy_(var.float())
  state_before = tower.bn_state.clone()
  x = torch.randn(m, d, generator=g)
  up = torch.randn(m, 1, generator=g)
  tower.eval()
  y = tower(x.cuda())
  (y * up.cuda()).sum().backward()
  ref = oracle_api.scorer.tower_forward(
      x.double(), params, activation=None, use_batch_norm=True,
      input_batch_norm=True, training=False, bn_moving=moving)
  (ref * up.double()).sum().backward()
  assert torch.equal(tower.bn_state, state_before)
  assert _rel_err(y, ref) <= 5e-5
  assert _rel_err(tower.flat.grad, _bn_flat_grad(params)) <= 5e-4


def _dropout_keep_mask(seed, layer, m, n, rate):
  """The mask tfr_mlp_fwd draws (include/tfr_b200.h, "dropout mask"): element i of
  hidden layer `layer` is dropped iff u < rate, u = top 24 bits of
  splitmix64(seed * 0x100000001B3 + layer + 1 + 0x9E3779B97F4A7C15 * (i + 1))."""
  import numpy as np
  with np.errstate(over='ignore'):
    s = np.uint64(seed) * np.uint64(0x100000001B3) + np.uint64(layer + 1)
    idx = np.arange(m * n, dtype=np.uint64)
    z = s + np.uint64(0x9E3779B97F4A7C15) * (idx + np.uint64(1))
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z = z ^ (z >> np.uint64(31))
  u = (z >> np.uint64(40)).astype(np.float32) * np.float32(1.0 / 16777216.0)
  keep = ~(u < np.float32(rate))
  return torch.from_numpy(keep.reshape(m, n))


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
@pytest.mark.parametrize('act,use_bn', [('relu', False), (None, False), ('relu', True)])
def test_tower_dropout(oracle_api, precision, act, use_bn):
  """Dropout after every hidden activation (keras/layers.py:74-75).  The reference's
  mask is random; ours is a documented counter hash of (seed, layer, element), so
  the test replays exactly that mask through the oracle, and checks the drop rate,
  the 1/(1-p) scale, determinism under a fixed seed, and eval()."""
  import ranking_b200 as tfr
  m, d, hidden, p = 2048, 32, [64, 32], 0.3
  tower, params = _bn_tower_and_params(tfr, d, hidden, 1, 11, act, precision,
                                       False, use_bn, dropout=p)
  g = torch.Generator().manual_seed(9)
  x = torch.randn(m, d, generator=g)
  up = torch.randn(m, 1, generator=g)
  tower.train()
  tower._dropout_calls = 0
  y = tower(x.cuda())
  (y * up.cuda()).sum().backward()
  seed = (tower._dropout_base << 32) | 1
  keeps = [_dropout_keep_mask(seed, i, m, h, p) for i, h in enumerate(hidden)]
  for k in keeps:
    assert abs(1.0 - float(k.double().mean()) - p) < 0.02
  ref = oracle_api.scorer.tower_forward(
      x.double(), params, activation=act, use_batch_norm=use_bn,
      keep_masks=[k.double() / (1 - p) for k in keeps])
  (ref * up.double()).sum().backward()
  assert _rel_err(y, ref) <= 1e-4, _rel_err(y, ref)
  got, want = tower.flat.grad.detach().cpu().double(), _bn_flat_grad(params)
  l2 = float((got - want).norm() / want.norm())
  assert l2 <= 1e-3, l2
  # same seed and call index -> same mask; next call -> another mask
  tower._dropout_calls = 0
  y2 = tower(x.cuda())
  assert torch.equal(y2, y)
  y3 = tower(x.cuda())
  assert not torch.equal(y3, y)
  # eval(): dropout is the identity
  tower.eval()
  ye = tower(x.cuda())
  moving = None
  if use_bn:
    moving = {i: [t.detach().cpu().double() for t in tower.bn_moving(i)]
              for i in range(len(hidden))}
  refe = oracle_api.scorer.tower_forward(x.double(), params, activation=act,
                                         use_batch_norm=use_bn, training=False,
                                         bn_moving=moving)
  assert _rel_err(ye, refe) <= 1e-4


def test_fused_train_step_with_batch_norm(oracle_api):
  """RankingTrainer over a BN tower: three Adagrad steps stay on the oracle's
  trajectory (BN parameters are part of the flat buffer / single all-reduce)."""
  import ranking_b200 as tfr
  b, n, d, hidden = 16, 12, 24, [32, 16]
  tower, params = _bn_tower_and_params(tfr, d, hidden, 1, 21, 'relu', 'fp32',
                                       True, True)
  loss = tfr.keras.losses.get('approx_ndcg_loss')
  trainer = tfr.train.RankingTrainer(tower, loss, optimizer='adagrad',
                                     learning_rate=0.05)
  oloss = oracle_api.keras_losses.get('approx_ndcg_loss')
  leaves = (params['dense_w'] + params['dense_b'] +
            [params['in_bn_gamma'], params['in_bn_beta']] +
            params['bn_gamma'] + params['bn_beta'])
  accum = [torch.full_like(t, 0.1) for t in leaves]
  g = torch.Generator().manual_seed(2)
  for step in range(3):
    x = torch.randn(b, n, d, generator=g)
    y = torch.randint(0, 5, (b, n), generator=g).float()
    y[:, -2:] = -1.0
    got = float(trainer.train_step(x.cuda(), y.cuda()))
    for t in leaves:
      t.grad = None
    mask = y >= 0
    # the reference flattens with circular padding before the tower
    # (keras/layers.py:163-173), so BatchNormalization only sees copies of valid items
    _, flat_x = oracle_api.scorer.flatten_list({}, {'x': x.double()}, mask,
                                               circular_padding=True)
    flat = oracle_api.scorer.tower_forward(
        flat_x['x'], params, activation='relu',
        use_batch_norm=True, input_batch_norm=True)
    logits = oracle_api.scorer.restore_list(flat, mask)
    ol = oloss(y.double(), logits)
    ol.backward()
    with torch.no_grad():
      for t, a in zip(leaves, accum):
        a.add_(t.grad * t.grad)
        t.sub_(0.05 * t.grad / (a.sqrt() + 1e-7))
    assert got == pytest.approx(float(ol.detach()), rel=2e-4, abs=1e-6)
  want = torch.cat([torch.cat([w.reshape(-1), b_.reshape(-1)]) for w, b_ in
                    zip(params['dense_w'], params['dense_b'])] +
                   [params['in_bn_gamma'], params['in_bn_beta']] +
                   [t for pair in zip(params['bn_gamma'], params['bn_beta'])
                    for t in pair]).detach()
  assert _rel_err(tower.flat.detach(), want) <= 2e-3


def test_tower_tensor_core_rejects_unaligned_widths():
  import ranking_b200 as tfr
  tower, _ = _tower_and_params(tfr, 17, [33], 1, seed=1, precision='tf32x3')
  with pytest.raises(ValueError):
    tower(torch.randn(64, 17).cuda())


def test_tower_restore_list_mask(oracle_api):
  import ranking_b200 as tfr
  tower, params = _tower_and_params(tfr, 8, [16], 1, seed=1)
  x = torch.randn(6, 5, 8)
  mask = torch.rand(6, 5) > 0.3
  y = tower(x.cuda(), mask=mask.cuda()).reshape(6, 5)
  ref = oracle_api.scorer.restore_list(
      oracle_api.scorer.tower_forward(x.double().reshape(30, 8), params,
                                      activation='relu'), mask)
  assert _rel_err(y, ref) <= RTOL
  assert float(y[~mask.cuda()].max()) == pytest.approx(math.log(1e-10), rel=1e-6)


def test_dnn_scorer_contract(oracle_api):
  """keras/model.py:755-817: context first, sorted keys, circular padding,
  RestoreList fill."""
  import ranking_b200 as tfr
  b, n = 4, 6
  g = torch.Generator().manual_seed(0)
  ctx = {'c2': torch.randn(b, 2, generator=g), 'c1': torch.randn(b, 1, generator=g)}
  ex = {'zf': torch.randn(b, n, 3, generator=g), 'af': torch.randn(b, n, 2, generator=g)}
  mask = torch.tensor([[1, 1, 1, 1, 1, 1], [1, 1, 1, 0, 0, 0],
                       [1, 0, 0, 0, 0, 0], [1, 1, 1, 1, 1, 0]]).bool()
  scorer = tfr.keras.model.DNNScorer(hidden_layer_dims=[16, 8], output_units=1,
                                     activation='relu', use_batch_norm=False,
                                     dropout=0, seed=5)
  got = scorer({k: v.cuda() for k, v in ctx.items()},
               {k: v.cuda() for k, v in ex.items()}, mask.cuda())
  tower = scorer.tower
  nl = len(tower.dims) - 1
  params = {'dense_w': [tower.kernel(i).detach().cpu().double() for i in range(nl)],
            'dense_b': [tower.bias(i).detach().cpu().double() for i in range(nl)]}
  ref = oracle_api.scorer.dnn_scorer(
      {k: v.double() for k, v in ctx.items()},
      {k: v.double() for k, v in ex.items()}, mask, params, activation='relu')
  assert tuple(got.shape) == (b, n)
  assert _rel_err(got, ref) <= RTOL


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
@pytest.mark.parametrize('loss_key,kw', [
    ('approx_ndcg_loss', {}),
    ('pairwise_logistic_loss', {}),
    ('softmax_loss', {}),
])
def test_fused_train_step_matches_oracle(oracle_api, loss_key, kw, precision):
  """One full step: scorer fwd -> loss -> scorer bwd -> Adagrad; loss, flat
  gradient and updated parameters vs the oracle (autograd + Keras Adagrad)."""
  import ranking_b200 as tfr
  b, n, d = 16, 30, 20
  scores_unused, labels, _, _ = _batch(b, n, seed=13)
  x = torch.randn(b, n, d, generator=torch.Generator().manual_seed(1))
  mask = labels >= 0
  tower, params = _tower_and_params(tfr, d, [32, 16], 1, seed=7,
                                    precision=precision)
  p0 = tower.flat.detach().clone()
  loss_obj = tfr.keras.losses.get(loss_key, **kw)
  tr = tfr.train.RankingTrainer(tower, loss_obj, optimizer='adagrad',
                                learning_rate=0.05)
  got = tr.train_step(x.cuda(), labels.cuda(), mask=mask.cuda())
  logits = oracle_api.scorer.restore_list(
      oracle_api.scorer.tower_forward(x.double().reshape(b * n, d), params,
                                      activation='relu'), mask)
  ref = oracle_api.keras_losses.get(loss_key, **kw)(labels.double(), logits)
  ref.backward()
  g = _flat_grad(params)
  assert abs(float(got) - float(ref)) <= RTOL * max(1., abs(float(ref)))
  assert _rel_err(tr.grads, g) <= 5e-5
  accum = 0.1 + g * g
  p_ref = p0.cpu().double() - 0.05 * g / (accum.sqrt() + 1e-7)
  assert _rel_err(tower.flat, p_ref) <= 1e-5


def test_groupwise_scoring_matches_oracle(oracle_api):
  """BASELINE config 4 structure (groupwise group_size=2 + softmax), small sizes:
  logits, loss and parameter gradients vs the oracle restatement of
  model.py:164-421 (no-shuffle permutation)."""
  import ranking_b200 as tfr
  b, n, d, gs = 6, 9, 8, 2
  g = torch.Generator().manual_seed(4)
  x = torch.randn(b, n, d, generator=g)
  labels = torch.randint(0, 3, (b, n), generator=g).float()
  labels[0, 5:] = -1.
  labels[3, 1:] = -1.       # a single valid item: windows wrap onto itself
  valid = labels >= 0
  tower, params = _tower_and_params(tfr, gs * d, [16, 8], gs, seed=3)
  model = tfr.model.GroupwiseRankingModel(tfr.model.TowerGroupScoreFn(tower), gs)
  logits = model.compute_logits(x.cuda(), valid.cuda())
  loss = tfr.keras.losses.SoftmaxLoss()(labels.cuda(), logits)
  loss.backward()

  def score_fn(gf):
    bg = gf.shape[0]
    return oracle_api.scorer.tower_forward(gf.reshape(bg, gs * d), params,
                                           activation='relu')
  ref_logits = oracle_api.scorer.groupwise_logits(x.double(), valid, gs, score_fn)
  ref_loss = oracle_api.keras_losses.SoftmaxLoss()(labels.double(), ref_logits)
  ref_loss.backward()
  assert _rel_err(logits, ref_logits) <= RTOL
  assert abs(float(loss.detach()) - float(ref_loss.detach())) <= RTOL
  assert _rel_err(tower.flat.grad, _flat_grad(params)) <= 5e-5
  # reference golden (model_test.py:223-277): dummy score fn = 1 + feature + #rows
  dummy = lambda gf: (1. + gf).reshape(-1, 2) + float(gf.shape[0])
  m2 = tfr.model.GroupwiseRankingModel(dummy, 2)
  out = m2.compute_logits(torch.tensor([[[1.], [2.], [3.]]]).cuda(),
                          torch.tensor([[True, True, False]]).cuda())
  assert out.tolist() == [[5., 6., 0.]]
  out = m2.compute_logits(torch.tensor([[[1.], [2.], [0.]]]).cuda(),
                          torch.tensor([[True, True, True]]).cuda(), num_shuffles=2)
  assert out.tolist() == [[8., 9., 7.]]


def test_two_gpu_data_parallel_step_equals_single_gpu():
  """8-list batch on 1 GPU vs 2 ranks x 4 lists over NCCL: same parameters after
  one step (needs 2 GPUs; skipped on the 1-GPU test box)."""
  if torch.cuda.device_count() < 2:
    pytest.skip('needs 2 GPUs')
  import subprocess
  import sys
  import os
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  out = subprocess.run(
      [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1',
       '--nproc-per-node', '2', '--master-addr', '127.0.0.1', '--master-port',
       '29611', os.path.join(root, 'tools', 'dp_equivalence.py')],
      capture_output=True, text=True, timeout=300)
  assert out.returncode == 0, out.stdout + out.stderr
  assert 'DP_EQUIVALENCE_OK' in out.stdout, out.stdout + out.stderr


# --------------------- size-independent properties at full size --------------
def test_full_size_properties_config2():
  """BASELINE config 2 (B=1024, N=200): properties that need no oracle."""
  import ranking_b200 as tfr
  b, n = 1024, 200
  scores, labels, _, _ = _batch(b, n, seed=1234, zero_rows=False)
  s = scores.cuda().requires_grad_()
  y = labels.cuda()
  loss = tfr.keras.losses.ApproxNDCGLoss(reduction='sum')(y, s)
  loss.backward()
  # ApproxNDCG in [-1, 0] per list; loss depends on score differences only.
  assert -b <= float(loss) <= 0.0
  assert float(s.grad.sum(1).abs().max()) <= 1e-4 * float(s.grad.abs().max())
  assert float(s.grad[y < 0].abs().max()) == 0.0
  # permutation equivariance on a list
  perm = torch.randperm(n, generator=torch.Generator().manual_seed(1)).cuda()
  s2 = s.detach()[:, perm].clone().requires_grad_()
  loss2 = tfr.keras.losses.ApproxNDCGLoss(reduction='sum')(y[:, perm], s2)
  loss2.backward()
  assert abs(float(loss2) - float(loss)) <= 1e-4 * abs(float(loss))
  assert _rel_err(s2.grad, s.grad[:, perm]) <= 1e-4
  # NDCG metric: 1.0 when scores order the labels, within [0, 1] otherwise
  m = tfr.metrics_impl.rank_metrics(y, y.clone() + 0.0, None, None, (10, None))
  has_rel = (labels > 0).any(1)
  assert torch.allclose(m['ndcg'][has_rel.cuda()], torch.ones(1).cuda())
  m = tfr.metrics_impl.rank_metrics(y, s.detach(), None, None, (10, None))
  assert float(m['ndcg'].min()) >= 0.0 and float(m['ndcg'].max()) <= 1.0 + 1e-6


def test_full_size_pairwise_n1024_gradient_sums():
  import ranking_b200 as tfr
  scores, labels, _, _ = _batch(64, 1024, seed=99, zero_rows=False)
  s = scores.cuda().requires_grad_()
  loss = tfr.keras.losses.PairwiseLogisticLoss(
      lambda_weight=tfr.keras.losses.NDCGLambdaWeight())(labels.cuda(), s)
  loss.backward()
  assert float(loss) > 0
  assert float(s.grad.sum(1).abs().max()) <= 1e-4 * float(s.grad.abs().max())


def test_error_behaviour():
  import ranking_b200 as tfr
  with pytest.raises(ValueError):
    tfr.keras.losses.get('no_such_loss')
  with pytest.raises(ValueError):
    tfr.keras.metrics.get('no_such_metric')
  with pytest.raises(ValueError):
    tfr.keras.losses.DCGLambdaWeight(smooth_fraction=2.0)
  with pytest.raises(ValueError):   # rank != 2 (losses_impl.py:52-58)
    tfr.keras.losses.PairwiseLogisticLoss()(torch.zeros(3).cuda(),
                                            torch.zeros(3).cuda())
  with pytest.raises(RuntimeError):  # no CPU fallback
    tfr.keras.losses.PairwiseLogisticLoss()(torch.zeros(1, 3), torch.zeros(1, 3))
