"""Bilinear (keras/layers.py:807-890) without a GPU: the reference's BilinearTest
(keras/layers_test.py:345-358) on the CPU oracle, a closed-form value, the argument checks of
the K14 C ABI, and the two-tower click recovery experiment of tests/_click_refs.py through the
oracle, which fixes the margin the GPU trainer is held to (tests/test_bilinear_gpu.py)."""
import ctypes

import torch

import _click_refs as CR

# Recovery margin, set from the oracle run below (measured NDCG@5 on held-out lists scored at
# position 0: bilinear two-tower 0.9998 vs naive 0.9045, a gap of 0.095) with a margin of
# about 2x.
DELTA = 0.05
# The relevance embedding width of that experiment.
E_CLICK = 8


def test_call_shape():
  """BilinearTest.test_call."""
  from oracle import bilinear
  v1 = torch.tensor([[1., 1.], [1., 0.]])
  v2 = torch.tensor([[0., 1.], [0., 0.]])
  out = bilinear.bilinear(v1, v2, *bilinear.init_bilinear(2, 1, seed=0))
  assert list(out.shape) == [2, 1]


def test_config_round_trip():
  """BilinearTest.test_serialization, on the layer's config (no GPU needed to build it)."""
  import __graft_entry__ as g
  g.build()
  import ranking_b200 as tfr
  layer = tfr.keras.layers.Bilinear(10, 2, seed=1, device='cpu')
  cfg = layer.get_config()
  assert cfg == {'embedding_dim': 10, 'output_dim': 2}
  loaded = tfr.keras.layers.Bilinear(**cfg, seed=1, device='cpu')
  assert loaded.get_config() == cfg
  assert torch.equal(loaded.flat, layer.flat)
  assert tuple(layer.bilinear_term().shape) == (10, 10, 2)
  assert tuple(layer.linear_term_1().shape) == (10, 2)
  assert tuple(layer.linear_term_2().shape) == (10, 2)
  assert tuple(layer.const_term().shape) == (2,)


def test_init_matches_oracle_and_keras_weights_round_trip():
  import __graft_entry__ as g
  g.build()
  import ranking_b200 as tfr
  from oracle import bilinear
  layer = tfr.keras.layers.Bilinear(6, 3, seed=7, device='cpu')
  ref = bilinear.init_bilinear(6, 3, seed=7)
  for got, want in zip([layer.bilinear_term(), layer.linear_term_1(), layer.linear_term_2(),
                        layer.const_term()], ref):
    assert torch.equal(got.detach(), want)
  # standard deviations of the reference's initialisers
  big = bilinear.init_bilinear(64, 32, seed=1)
  assert abs(float(big[0].std()) - 1 / 64) < 0.02 / 64
  assert abs(float(big[1].std()) - 1 / 8) < 0.1 / 8
  assert float(big[3].abs().max()) == 0.
  new = [torch.randn(6, 6, 3), torch.randn(6, 3), torch.randn(6, 3), torch.randn(3)]
  layer.load_keras_weights(new)
  assert torch.equal(layer.bilinear_term().detach(), new[0])
  assert torch.equal(layer.const_term().detach(), new[3])
  for bad in (new[:3], [new[0], new[1], new[2], torch.zeros(4)]):
    try:
      layer.load_keras_weights(bad)
    except ValueError:
      continue
    raise AssertionError('load_keras_weights accepted %d arrays' % len(bad))


def test_closed_form():
  """E = 2, K = 2 with injected weights, evaluated by hand."""
  from oracle import bilinear
  W = torch.tensor([[[1., 0.], [2., 1.]], [[0., 3.], [-1., 2.]]], dtype=torch.float64)
  W1 = torch.tensor([[1., -1.], [0.5, 2.]], dtype=torch.float64)
  W2 = torch.tensor([[2., 0.], [1., 1.]], dtype=torch.float64)
  b = torch.tensor([0.25, -0.5], dtype=torch.float64)
  v1 = torch.tensor([[1., 2.]], dtype=torch.float64)
  v2 = torch.tensor([[3., -1.]], dtype=torch.float64)
  # k = 0: v1 W[:, :, 0] v2 = [1, 2] [[1, 2], [0, -1]] [3, -1] = [1, 0] . [3, -1] = 3
  #        v1 W1[:, 0] = 1 + 1 = 2;  v2 W2[:, 0] = 6 - 1 = 5;  + 0.25  -> 10.25
  # k = 1: [1, 2] [[0, 1], [3, 2]] [3, -1] = [6, 5] . [3, -1] = 13
  #        v1 W1[:, 1] = -1 + 4 = 3;  v2 W2[:, 1] = 0 - 1 = -1;  - 0.5  -> 14.5
  y = bilinear.bilinear(v1, v2, W, W1, W2, b)
  assert torch.equal(y, torch.tensor([[10.25, 14.5]], dtype=torch.float64))


def test_c_abi_argument_checks():
  """NULL pointers and sizes past the limits return TFR_INVALID_ARGUMENT (1) before any CUDA
  call, so this runs without a GPU."""
  import __graft_entry__ as g
  g.build()
  from ranking_b200 import _C
  lib = _C.lib
  assert lib.tfr_bilinear_param_count(16, 1) == 16 * 16 + 2 * 16 + 1
  assert lib.tfr_bilinear_param_count(128, 1) == 128 * 128 + 2 * 128 + 1
  assert lib.tfr_bilinear_param_count(16, 32) == 16 * 16 * 32 + 2 * 16 * 32 + 32
  for e, k in ((0, 1), (129, 1), (16, 0), (16, 33), (64, 5), (23, 32), (-1, 1)):
    assert lib.tfr_bilinear_param_count(e, k) == 0, (e, k)
    assert lib.tfr_bilinear_workspace_bytes(10, e, k) == 0, (e, k)
  assert lib.tfr_bilinear_workspace_bytes(0, 16, 1) == 0
  assert lib.tfr_bilinear_workspace_bytes(204800, 16, 1) > 0
  p = ctypes.c_void_p(16)   # never dereferenced: every call below fails its checks first
  args = lambda m, e, k: (p, p, m, e, k, p, None, p, None)   # noqa: E731
  assert lib.tfr_bilinear_fwd(None, p, 4, 16, 1, p, None, p, None) == 1
  assert 'NULL' in _C.last_error()
  assert lib.tfr_bilinear_fwd(p, p, 4, 16, 1, None, None, p, None) == 1
  assert lib.tfr_bilinear_fwd(p, p, 4, 16, 1, p, None, None, None) == 1
  for m, e, k in ((0, 16, 1), (-3, 16, 1), (4, 0, 1), (4, 129, 1), (4, 16, 0), (4, 16, 33),
                  (4, 64, 5)):
    assert lib.tfr_bilinear_fwd(*args(m, e, k)) == 1, (m, e, k)
    assert lib.tfr_bilinear_bwd(p, p, m, e, k, p, None, p, p, p, p, p, None) == 1, (m, e, k)
  full = [p, p, 4, 16, 1, p, None, p, p, p, p, p, None]
  for i in (0, 1, 5, 7, 8, 9, 10, 11):
    bad = list(full)
    bad[i] = None
    assert lib.tfr_bilinear_bwd(*bad) == 1, i
    assert 'NULL' in _C.last_error()


def _naive_step(params, leaves, accum, xb, cb):
  from oracle import keras_losses, scorer
  for p in leaves:
    p.grad = None
  logits = scorer.tower_forward(xb.reshape(-1, CR.D), params)
  keras_losses.SigmoidCrossEntropyLoss()(cb, logits.reshape(cb.shape)).backward()
  with torch.no_grad():
    for p, a in zip(leaves, accum):
      a.add_(p.grad * p.grad)
      p.sub_(CR.LR * p.grad / (a.sqrt() + 1e-7))


def test_bilinear_click_recovery_oracle():
  """A linear relevance tower x -> R^8, a 64-row position table of width 8 and Bilinear(8, 1),
  trained with sigmoid cross entropy on position-biased clicks (tests/_click_refs.py), ranks
  held-out lists scored at position 0 better than a model trained naively on the clicks,
  through the CPU oracle.  This run sets DELTA."""
  from oracle import bilinear, scorer
  x, c, _ = CR.click_logs(CR.TRAIN_LISTS, seed=1)
  xt, _, p_rel = CR.click_logs(CR.TEST_LISTS, seed=2)
  gen = torch.Generator().manual_seed(5)
  table = (torch.rand(64, E_CLICK, generator=gen, dtype=torch.float64) * 0.1 - 0.05).float()
  tt = bilinear.BilinearClickTrainer(scorer.init_tower_params(CR.D, [], E_CLICK, seed=3), table,
                                     bilinear.init_bilinear(E_CLICK, 1, seed=4),
                                     learning_rate=CR.LR)
  naive = scorer.init_tower_params(CR.D, [], 1, seed=3)
  leaves = naive['dense_w'] + naive['dense_b']
  for p in leaves:
    p.requires_grad_()
  accum = [torch.full_like(p, 0.1) for p in leaves]
  for xb, cb in CR.batches(x, c):
    tt.train_step(xb, cb)
    _naive_step(naive, leaves, accum, xb, cb)
  s_two = tt.predict(xt, serving_position=0)
  with torch.no_grad():
    s_naive = scorer.tower_forward(xt.reshape(-1, CR.D), naive).reshape(xt.shape[:2])
  got, base = CR.ndcg_at(s_two, p_rel, 5), CR.ndcg_at(s_naive, p_rel, 5)
  assert got >= base + DELTA, (got, base)
