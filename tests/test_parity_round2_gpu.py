"""GPU parity tests added in round 2 (CUDA path through the C ABI vs the CPU oracle).

Tolerances, stated where they are used:
  * losses: 1e-5 relative (north_star);
  * score gradients: PER ELEMENT |got - ref| <= 1e-5 |ref| + 1e-5 mean_list|ref|
    (the absolute floor is the list's mean gradient magnitude: single entries are sums
    of up to N signed fp32 terms and may cancel to ~0);
  * integer outputs (ranks): exact.
"""
import math

import pytest
import torch

from _tower_refs import _emulated_bf16_tower

pytestmark = pytest.mark.gpu

RTOL = 1e-5


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


def _check(cuda_loss, oracle_loss, scores, labels, weights):
  s_gpu = scores.cuda().requires_grad_()
  w_gpu = None if weights is None else weights.cuda()
  got = cuda_loss(labels.cuda(), s_gpu, w_gpu)
  got.backward()
  s_ref = scores.double().requires_grad_()
  w_ref = None if weights is None else weights.double()
  ref = oracle_loss(labels.double(), s_ref, w_ref)
  ref.backward()
  assert abs(float(got) - float(ref)) <= RTOL * max(1.0, abs(float(ref))), (
      float(got), float(ref))
  assert_grad_close(s_gpu.grad, s_ref.grad)


LAMBDAS = {
    'none': lambda K: None,
    'label_diff': lambda K: K.LabelDiffLambdaWeight(),
    'dcg_smooth': lambda K: K.DCGLambdaWeight(topn=20, smooth_fraction=0.4),
    'ndcg': lambda K: K.NDCGLambdaWeight(),
    'ndcg_top7': lambda K: K.NDCGLambdaWeight(topn=7),
    'ndcg_v2_top5': lambda K: K.NDCGLambdaWeightV2(topn=5),
    'yeti': lambda K: K.YetiDCGLambdaWeight(topn=4, normalized=True),
    'precision_top3': lambda K: K.PrecisionLambdaWeight(topn=3),
}


# N covers every tiling of the triangular K1 kernel: 1 / 2 / 4 / 8-tile chunks, several
# chunks (N > 256), partial tiles, the 8 / 4 / 2 lists-per-CTA packings and N = 1024.
@pytest.mark.parametrize('n', [1, 2, 5, 31, 32, 33, 64, 100, 128, 200, 257, 300, 513])
@pytest.mark.parametrize('lam', ['none', 'ndcg', 'dcg_smooth'])
def test_k1_triangular_sizes(cuda_api, oracle_api, n, lam):
  scores, labels, item_w = _batch(11, n, seed=100 + n)
  KC, KO = cuda_api.keras_losses, oracle_api.keras_losses
  _check(KC.PairwiseLogisticLoss(lambda_weight=LAMBDAS[lam](KC)),
         KO.PairwiseLogisticLoss(lambda_weight=LAMBDAS[lam](KO)), scores, labels, item_w)


@pytest.mark.parametrize('cls', ['PairwiseLogisticLoss', 'PairwiseHingeLoss',
                                 'PairwiseSoftZeroOneLoss'])
@pytest.mark.parametrize('lam', sorted(LAMBDAS))
def test_k1_triangular_lambdas_with_holes(cuda_api, oracle_api, cls, lam):
  """Every lambda weight x phi at N = 150 with padding scattered inside the lists."""
  scores, labels, item_w = _batch(7, 150, seed=5, holes=True)
  KC, KO = cuda_api.keras_losses, oracle_api.keras_losses
  _check(getattr(KC, cls)(lambda_weight=LAMBDAS[lam](KC), temperature=0.8),
         getattr(KO, cls)(lambda_weight=LAMBDAS[lam](KO), temperature=0.8),
         scores, labels, item_w)


def test_k1_triangular_n1024(cuda_api, oracle_api):
  scores, labels, _ = _batch(3, 1024, seed=77)
  KC, KO = cuda_api.keras_losses, oracle_api.keras_losses
  _check(KC.PairwiseLogisticLoss(lambda_weight=KC.NDCGLambdaWeight()),
         KO.PairwiseLogisticLoss(lambda_weight=KO.NDCGLambdaWeight()), scores, labels, None)


@pytest.mark.parametrize('n', [19, 150, 400])
def test_k1_triangular_row_losses(cuda_api, oracle_api, n):
  """reduction=NONE needs the [B, N] row sums of the pair-loss matrix (hi item's row)."""
  scores, labels, item_w = _batch(5, n, seed=3 + n, holes=True)
  KC, KO = cuda_api.keras_losses, oracle_api.keras_losses
  up = torch.rand(5, n)
  for lam in ['none', 'ndcg']:
    s_gpu = scores.cuda().requires_grad_()
    out = KC.PairwiseLogisticLoss(reduction=KC.Reduction.NONE,
                                  lambda_weight=LAMBDAS[lam](KC))(
                                      labels.cuda(), s_gpu, item_w.cuda())
    (out * up.cuda()).sum().backward()
    s_ref = scores.double().requires_grad_()
    ref = KO.PairwiseLogisticLoss(reduction=KO.Reduction.NONE,
                                  lambda_weight=LAMBDAS[lam](KO))(
                                      labels.double(), s_ref, item_w.double())
    (ref * up.double()).sum().backward()
    assert_grad_close(out, ref)
    assert_grad_close(s_gpu.grad, s_ref.grad)


def test_k1_estimator_reductions_large(cuda_api, oracle_api):
  """SUM_BY_NONZERO_WEIGHTS / MEAN need the per-list sum W and #(W != 0)."""
  scores, labels, item_w = _batch(6, 170, seed=4)
  LC, LO = cuda_api.losses_impl, oracle_api.losses_impl
  for red in ['SUM', 'MEAN', 'SUM_BY_NONZERO_WEIGHTS', 'SUM_OVER_BATCH_SIZE']:
    for cls in ['PairwiseLogisticLoss', 'PairwiseHingeLoss']:
      got = getattr(LC, cls)(name=None, lambda_weight=LC.DCGLambdaWeight(topn=9)).compute(
          labels.cuda(), scores.cuda(), item_w.cuda(), getattr(LC.Reduction, red))
      ref = getattr(LO, cls)(name=None, lambda_weight=LO.DCGLambdaWeight(topn=9)).compute(
          labels.double(), scores.double(), item_w.double(), getattr(LO.Reduction, red))
      assert abs(float(got) - float(ref)) <= RTOL * max(1., abs(float(ref))), (
          red, cls, float(got), float(ref))


def test_k1_sort_order_equals_counting_ranks(cuda_api, oracle_api):
  """The walk order of the triangular kernel (bitonic sort; `ranks_out` of the C entry)
  must be the counting rank, exactly, with ties broken by index and padding last."""
  from ranking_b200 import _C
  b, n = 16, 300
  scores, labels, _ = _batch(b, n, seed=8, holes=True)
  scores[:, ::7] = scores[:, 1:2]          # many exact ties -> broken by index
  s, l = scores.cuda().contiguous(), labels.cuda().contiguous()
  grad = torch.empty_like(s)
  loss = torch.empty(b, device='cuda')
  ranks = torch.zeros(b, n, dtype=torch.int32, device='cuda')
  _C.check(_C.lib.tfr_pairwise_loss_fwd_bwd(
      _C.ptr(s), _C.ptr(l), None, 0, None, b, n, 1.0, _C.PHI_LOGISTIC, None, 1.0,
      _C.ptr(grad), None, _C.ptr(loss), None, None, _C.ptr(ranks), _C.stream()))
  ref = oracle_api.losses_impl._compute_ranks(scores.double(), labels >= 0)
  assert torch.equal(ranks.cpu().long(), ref)


# ----------------------------------------------------------------------------
# bf16 scorer tower (TFR_PREC_BF16, BASELINE config 3)
# ----------------------------------------------------------------------------
@pytest.mark.parametrize('shape', [
    (300, 16, [32, 16], 1),            # small, partial tiles
    (1000, 136, [256, 128, 64], 1),    # config-2 widths
    (4096, 256, [256, 128, 64], 1),    # config-3 widths
    (2000, 64, [128], 2),              # two outputs
    (700, 40, [], 1),                  # a single Dense layer: no tensor-core GEMM at all
])
@pytest.mark.parametrize('relu', [True, False])
def test_tower_bf16_matches_emulation(shape, relu):
  """bf16 tower forward + backward vs the fp64 emulation of the same roundings.
  Tolerance: 5e-3 of the largest entry (the CUDA path accumulates in fp32: a stored
  activation that sits on a bf16 rounding boundary may round the other way, and a
  pre-activation within fp32 rounding of 0 may flip its ReLU mask bit; measured 1e-7 ..
  2e-3)."""
  import ranking_b200 as tfr
  m, d, hidden, out = shape
  g = torch.Generator().manual_seed(m + d)
  x = torch.randn(m, d, generator=g)
  tower = tfr.keras.layers.create_tower(hidden, out, activation='relu' if relu else None,
                                        use_batch_norm=False, dropout=0, input_dim=d,
                                        precision='bf16', seed=5)
  with torch.no_grad():
    for i in range(len(tower.dims) - 1):
      tower.bias(i).uniform_(-0.2, 0.2)
  mask = torch.rand(m, generator=g) > 0.1
  dscores = torch.randn(m, out, generator=g)
  ws = [tower.kernel(i).detach().cpu() for i in range(len(tower.dims) - 1)]
  bs = [tower.bias(i).detach().cpu() for i in range(len(tower.dims) - 1)]
  use_mask = out == 1
  y = tower(x.cuda(), mask=mask.cuda() if use_mask else None)
  y.backward(dscores.cuda())
  ds_eff = dscores * mask.reshape(-1, 1).float() if use_mask else dscores
  ref_scores, ref_grad = _emulated_bf16_tower(x, ws, bs, ds_eff, relu)
  got = y.detach().double().cpu()
  if use_mask:
    assert float(got[~mask].max()) == pytest.approx(math.log(1e-10), rel=1e-6)
    got, ref_scores = got[mask], ref_scores[mask]
  e_s = float((got - ref_scores).abs().max() / ref_scores.abs().max())
  e_g = float((tower.flat.grad.double().cpu() - ref_grad).abs().max() / ref_grad.abs().max())
  print('bf16 tower', shape, relu, 'scores %.2e grads %.2e' % (e_s, e_g))
  assert e_s <= 5e-3, e_s
  assert e_g <= 5e-3, e_g


def test_tower_bf16_vs_fp32_oracle(oracle_api):
  """Stated bf16 tolerance against the fp64 ORACLE (no rounding emulation): scores within
  2e-2 and parameter gradients within 6e-2 of the largest entry at config-3 widths
  (measured 5e-3 / 3e-2: three layers of bf16 products, bf16 backward signals)."""
  import ranking_b200 as tfr
  m, d, hidden = 2048, 256, [256, 128, 64]
  g = torch.Generator().manual_seed(9)
  x = torch.randn(m, d, generator=g)
  tower = tfr.keras.layers.create_tower(hidden, 1, activation='relu', use_batch_norm=False,
                                        dropout=0, input_dim=d, precision='bf16', seed=6)
  dscores = torch.randn(m, 1, generator=g)
  y = tower(x.cuda())
  y.backward(dscores.cuda())
  params = {'dense_w': [tower.kernel(i).detach().cpu().double().requires_grad_()
                        for i in range(4)],
            'dense_b': [tower.bias(i).detach().cpu().double().requires_grad_()
                        for i in range(4)]}
  ref = oracle_api.scorer.tower_forward(x.double(), params, activation='relu')
  ref.backward(dscores.double())
  ref_grad = torch.cat([torch.cat([w.grad.reshape(-1), b.grad.reshape(-1)])
                        for w, b in zip(params['dense_w'], params['dense_b'])])
  e_s = float((y.detach().double().cpu() - ref.detach()).abs().max() / ref.abs().max())
  e_g = float((tower.flat.grad.double().cpu() - ref_grad).abs().max() / ref_grad.abs().max())
  print('bf16 vs fp64 oracle: scores %.2e grads %.2e' % (e_s, e_g))
  assert e_s <= 2e-2, e_s
  assert e_g <= 6e-2, e_g


# ----------------------------------------------------------------------------
# K8: groupwise scoring folded into the tower (BASELINE config 4)
# ----------------------------------------------------------------------------
def _group_case(b, n, d, gs, hidden, seed, precision='tf32x3', activation='relu'):
  import ranking_b200 as tfr
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(b, n, d, generator=g)
  labels = torch.randint(0, 3, (b, n), generator=g).float()
  lens = torch.randint(1, n + 1, (b,), generator=g)
  labels = torch.where(torch.arange(n).unsqueeze(0) < lens.unsqueeze(1), labels,
                       torch.full_like(labels, -1.))
  labels[0, 1:] = -1.          # a single valid item: the window wraps onto itself
  tower = tfr.keras.layers.create_tower(hidden, gs, activation=activation,
                                        use_batch_norm=False, dropout=0, input_dim=gs * d,
                                        precision=precision, seed=seed)
  with torch.no_grad():
    for i in range(len(tower.dims) - 1):
      tower.bias(i).uniform_(-0.2, 0.2)
  nl = len(tower.dims) - 1
  params = {'dense_w': [tower.kernel(i).detach().cpu().double().clone().requires_grad_()
                        for i in range(nl)],
            'dense_b': [tower.bias(i).detach().cpu().double().clone().requires_grad_()
                        for i in range(nl)]}
  return tfr, x, labels, tower, params


def _flat_grad(params):
  return torch.cat([torch.cat([w.grad.reshape(-1), b.grad.reshape(-1)])
                    for w, b in zip(params['dense_w'], params['dense_b'])])


def assert_param_grads_close(got, ref, relu, tol=5e-5, relu_l2=None):
  """Parameter gradients.  Linear towers: every entry within `tol` of the largest entry.
  ReLU towers: `tol` in L2; single entries may be off by more because a hidden unit whose
  pre-activation lies within the scorer's own rounding (4e-6) of zero takes the other ReLU
  branch than the fp64 oracle — its whole contribution moves.  Those entries are bounded
  at 2e-2 of the largest entry and must be rare (< 0.5 % of the entries beyond 4 tol).
  `relu_l2`: L2 bound for full-size chunks, where the count of such gates grows with
  rows x units (3.3 M pre-activations at the config-2 chunk: ~10 of them lie within the
  forward's 4e-6 of zero, and each flips one row's contribution to a whole dW column:
  sqrt(flips / (units x active rows)) ~ 3e-3 in L2).  The linear towers of the same tests
  pin the GEMM numerics themselves at `tol` in max-norm."""
  got = got.detach().double().cpu()
  ref = ref.detach().double().cpu()
  err = (got - ref).abs()
  scale = float(ref.abs().max())
  e_max, e_l2 = float(err.max()) / scale, float(err.norm() / ref.norm())
  print('param grads: max-norm err %.2e, L2 err %.2e' % (e_max, e_l2))
  if not relu:
    assert e_max <= tol, e_max
    return
  assert e_l2 <= (relu_l2 if relu_l2 is not None else 4 * tol), e_l2
  assert e_max <= (5e-2 if relu_l2 is not None else 2e-2), e_max
  assert float((err > 4 * tol * scale).double().mean()) < (0.25 if relu_l2 is not None else 5e-3)


@pytest.mark.parametrize('shape', [(6, 9, 8, 2, [16, 8]), (5, 33, 16, 2, [32]),
                                   (4, 40, 12, 3, [32, 16]), (16, 128, 512, 2, [256, 128, 64])])
@pytest.mark.parametrize('shuffles', [1, 2])
@pytest.mark.parametrize('activation', ['relu', None])
def test_groupwise_fold_matches_oracle(oracle_api, shape, shuffles, activation):
  """Folded first layer (csrc/mlp_group.cu) vs the oracle restatement of model.py:164-421:
  logits, softmax loss, parameter gradients.  The last shape is a 16-list chunk of BASELINE
  config 4 (N=128, D=512, group_size 2, 256-128-64).  Tolerances: logits / loss 1e-5,
  gradients see assert_param_grads_close (3xTF32)."""
  b, n, d, gs, hidden = shape
  tfr, x, labels, tower, params = _group_case(b, n, d, gs, hidden, seed=b + n + d,
                                              activation=activation)
  valid = labels >= 0
  model = tfr.model.GroupwiseRankingModel(tfr.model.TowerGroupScoreFn(tower), gs)
  assert tfr.model.fold_supported(model._score_fn, gs, d)
  logits = model.compute_logits(x.cuda(), valid.cuda(), num_shuffles=shuffles)
  loss = tfr.keras.losses.SoftmaxLoss()(labels.cuda(), logits)
  loss.backward()

  def score_fn(gf):
    return oracle_api.scorer.tower_forward(gf.reshape(gf.shape[0], gs * d), params,
                                           activation=activation)
  ref_logits = oracle_api.scorer.groupwise_logits(x.double(), valid, gs, score_fn,
                                                  num_shuffles=shuffles)
  ref_loss = oracle_api.keras_losses.SoftmaxLoss()(labels.double(), ref_logits)
  ref_loss.backward()
  scale = float(ref_logits.detach().abs().max())
  assert float((logits.detach().double().cpu() - ref_logits.detach()).abs().max()) <= RTOL * scale
  assert abs(float(loss.detach()) - float(ref_loss.detach())) <= RTOL * max(
      1., abs(float(ref_loss.detach())))
  assert_param_grads_close(tower.flat.grad, _flat_grad(params), relu=activation == 'relu',
                           relu_l2=1e-2 if b * n * d > 100000 else None)
  # and the unfolded product path (gather materialised) agrees with the fold
  tower.flat.grad = None
  model.fold = False
  logits2 = model.compute_logits(x.cuda(), valid.cuda(), num_shuffles=shuffles)
  assert float((logits2 - logits).abs().max()) <= RTOL * scale


def test_groupwise_fold_with_permutation(oracle_api):
  """Caller-supplied shuffles of the valid items (the reference shuffles with TF's RNG)."""
  b, n, d, gs = 5, 21, 8, 2
  tfr, x, labels, tower, params = _group_case(b, n, d, gs, [16], seed=3)
  valid = labels >= 0
  g = torch.Generator().manual_seed(1)
  perms = []
  for _ in range(2):   # permute the valid-first order among the valid prefix only
    nv = valid.sum(1)
    perm = torch.arange(n).repeat(b, 1)
    for r in range(b):
      k = int(nv[r])
      perm[r, :k] = torch.randperm(k, generator=g)
    perms.append(perm)
  model = tfr.model.GroupwiseRankingModel(tfr.model.TowerGroupScoreFn(tower), gs)
  fold = model.compute_logits(x.cuda(), valid.cuda(), num_shuffles=2,
                              permutations=[p.cuda() for p in perms])
  model.fold = False
  plain = model.compute_logits(x.cuda(), valid.cuda(), num_shuffles=2,
                               permutations=[p.cuda() for p in perms])
  assert float((fold - plain).abs().max()) <= RTOL * float(plain.abs().max())


# ----------------------------------------------------------------------------
# BASELINE config 2 at its real shape (a 64-list chunk), fused step vs the oracle
# ----------------------------------------------------------------------------
def _c2_chunk(precision, activation='relu'):
  import ranking_b200 as tfr
  import bench
  b, n, d = 64, 200, 136
  x, y = bench.make_batch(4321, b, n, d)
  tower = tfr.keras.layers.create_tower(bench.HIDDEN, 1, activation=activation,
                                        use_batch_norm=False, dropout=0, input_dim=d,
                                        precision=precision, seed=1238)
  with torch.no_grad():
    for i in range(4):
      tower.bias(i).uniform_(-0.1, 0.1)
  return tfr, x, y, tower


@pytest.mark.parametrize('activation', ['relu', None])
def test_config2_chunk_step_matches_oracle(oracle_api, activation):
  """64 lists x 200 x 136, hidden 256-128-64, ApproxNDCG, Adagrad(0.05), scorer in 3xTF32:
  loss, d loss / d scores, flat parameter gradient and updated parameters vs the fp64 oracle.
  Tolerances: loss 1e-5; dscores per element (1e-5 |ref| + 1e-5 list mean) against the oracle
  loss on the same scores and 1e-4 against the fp64 chain;
  parameter gradients 8e-5 in L2 (assert_param_grads_close: ReLU tower); parameters 1e-5
  (an Adagrad step of 0.05 * g / sqrt(0.1 + g^2) moves a parameter by <= 0.05, so a
  gradient entry that is off by a flipped ReLU gate moves it by <= 1e-3 of that)."""
  tfr, x, y, tower = _c2_chunk('tf32x3', activation)
  p0 = tower.flat.detach().clone()
  params = {'dense_w': [tower.kernel(i).detach().cpu().double().clone().requires_grad_()
                        for i in range(4)],
            'dense_b': [tower.bias(i).detach().cpu().double().clone().requires_grad_()
                        for i in range(4)]}
  tr = tfr.train.RankingTrainer(tower, tfr.keras.losses.get('approx_ndcg_loss'),
                                optimizer='adagrad', learning_rate=0.05)
  mask = y >= 0
  got = tr.train_step(x.cuda(), y.cuda(), mask=mask.cuda())
  b, n, d = x.shape
  flat = oracle_api.scorer.tower_forward(x.double().reshape(b * n, d), params,
                                         activation=activation)
  logits = oracle_api.scorer.restore_list(flat, mask)
  logits.retain_grad()
  ref = oracle_api.keras_losses.get('approx_ndcg_loss')(y.double(), logits)
  ref.backward()
  assert abs(float(got) - float(ref.detach())) <= RTOL * max(1., abs(float(ref.detach())))
  # d loss / d scores, per element, valid slots.  (a) the loss kernel alone: the oracle loss
  # evaluated on the GPU's own scores must agree per element to 1e-5; (b) the whole chain:
  # the 3xTF32 scores are within 4e-6 of the fp64 ones and ApproxNDCG divides them by its
  # temperature 0.1, so the chain's d loss / d scores can only agree to ~1e-4 per element.
  ds = tr.dscores.detach().double().cpu()
  s_gpu = tr.scores.detach().double().cpu().requires_grad_()
  oracle_api.keras_losses.get('approx_ndcg_loss')(y.double(), s_gpu).backward()
  assert_grad_close(ds * mask, s_gpu.grad * mask, outliers=1e-3)
  assert_grad_close(ds * mask, logits.grad * mask, rtol=1e-4, outliers=1e-3)
  g = _flat_grad(params)
  assert_param_grads_close(tr.grads, g, relu=activation == 'relu', tol=2e-5, relu_l2=1e-2)
  accum = 0.1 + g * g
  p_ref = p0.cpu().double() - 0.05 * g / (accum.sqrt() + 1e-7)
  e_p = float((tower.flat.detach().double().cpu() - p_ref).abs().max() / p_ref.abs().max())
  # (ReLU: a parameter whose gradient entry moved by a flipped gate moves by up to 1e-3 of
  #  the 0.05 step, see the docstring; the linear tower pins the update itself at 1e-5)
  assert e_p <= (1e-3 if activation == 'relu' else 1e-5), e_p


def test_config2_chunk_scores_and_ndcg10(oracle_api):
  """Scores within 1e-5 of the fp64 oracle, identical rank arrays, NDCG@10 per list equal
  to the oracle metric on the same scores within 2 fp32 ulps."""
  tfr, x, y, tower = _c2_chunk('tf32x3')
  params = {'dense_w': [tower.kernel(i).detach().cpu().double() for i in range(4)],
            'dense_b': [tower.bias(i).detach().cpu().double() for i in range(4)]}
  b, n, d = x.shape
  scores = tower(x.cuda()).reshape(b, n).detach()
  ref = oracle_api.scorer.tower_forward(x.double().reshape(b * n, d), params,
                                        activation='relu').reshape(b, n)
  assert float((scores.double().cpu() - ref).abs().max() / ref.abs().max()) <= RTOL
  yd = y.cuda()
  ranks = tfr.utils.sorted_ranks(scores, yd).cpu().long()
  assert torch.equal(ranks, oracle_api.losses_impl._compute_ranks(scores.double().cpu(), y >= 0))
  got, _ = tfr.metrics_impl.NDCGMetric(name=None, topn=10).compute(yd, scores, None)
  want, _ = oracle_api.metrics_impl.NDCGMetric(name=None, topn=10).compute(
      y.double(), scores.double().cpu(), None)
  assert float((got.double().cpu() - want).abs().max()) <= 2 * 1.1920929e-07


# ----------------------------------------------------------------------------
# K9: circular padding in front of a BatchNormalization tower on the fused trainer
# ----------------------------------------------------------------------------
@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
def test_fused_trainer_batch_norm_sees_circular_padding(precision):
  """With BN the fused step must equal the DNNScorer path (FlattenList circular padding ->
  tower -> RestoreList): batch statistics over copies of valid rows only
  (keras/layers.py:163-173).  Same loss, same parameter gradients, same moving statistics."""
  import ranking_b200 as tfr
  b, n, d = 12, 20, 16
  g = torch.Generator().manual_seed(2)
  x = torch.randn(b, n, d, generator=g) * 3 + 1
  y = torch.randint(0, 4, (b, n), generator=g).float()
  lens = torch.randint(3, n + 1, (b,), generator=g)
  y = torch.where(torch.arange(n).unsqueeze(0) < lens.unsqueeze(1), y, torch.full_like(y, -1.))
  x = torch.where((y >= 0).unsqueeze(2), x, torch.full_like(x, 50.))   # loud padding rows
  mask = y >= 0

  def make():
    return tfr.keras.layers.create_tower([32, 16], 1, activation='relu', use_batch_norm=True,
                                         input_batch_norm=True, dropout=0, input_dim=d,
                                         precision=precision, seed=11)
  t1, t2 = make(), make()
  loss_obj = tfr.keras.losses.get('approx_ndcg_loss')
  tr = tfr.train.RankingTrainer(t1, loss_obj, optimizer='sgd', learning_rate=0.0)
  got = tr.train_step(x.cuda(), y.cuda(), mask=mask.cuda())
  scorer = tfr.keras.model.DNNScorer(hidden_layer_dims=[32, 16], output_units=1)
  scorer.tower = t2
  logits = scorer({}, {'f': x.cuda()}, mask.cuda())
  ref = loss_obj(y.cuda(), logits)
  ref.backward()
  tol = 2e-5 if precision == 'fp32' else 1e-4
  assert abs(float(got) - float(ref.detach())) <= tol * max(1., abs(float(ref.detach())))
  err = float((tr.grads - t2.flat.grad).abs().max() / t2.flat.grad.abs().max())
  assert err <= tol, err
  assert float((t1.bn_state - t2.bn_state).abs().max()) <= tol
