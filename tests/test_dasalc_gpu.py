"""DASALC (K13, csrc/dasalc.cu) against the fp64 restatement in _dasalc_refs.py, with the
noise and dropout draws replayed in Python.

Inputs are drawn so that no BatchNormalization column has a near-zero variance: features and
embeddings are standard normal and biases small, so every hidden ReLU column keeps a sizeable
share of positive rows.  Tolerances: 3xTF32 is fp32-faithful, so scores agree to 1e-5 of the
largest |score| (as the tower and DIN tests); plain TF32 rounds every GEMM operand to a
10-bit mantissa, and those errors pass through four BatchNormalizations, so it is held to
2e-2 of the largest |score|."""
import ctypes
import itertools
import math
import os
import subprocess
import sys

import pytest
import torch

import ranking_b200 as tfr
from ranking_b200 import _C
from ranking_b200.research import dasalc
from oracle import din as odin
from oracle import keras_losses as oracle_losses
from oracle import scorer as oracle_scorer
from oracle import utils as oracle_utils
import _dasalc_refs as ref

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NUMERICAL = os.path.join(ROOT, 'tests', 'golden', 'numerical')


def _list_mask(b, n, gen):
  """Full, all-padded, single-item and ragged lists."""
  m = torch.rand(b, n, generator=gen) < 0.6
  m[0] = True
  m[1] = False
  m[2] = False
  m[2, n // 3] = True
  return m.reshape(-1)


def _make(d, w, h, seed, dropout=0.3, noise=0.5, precision='tf32x3'):
  gen = torch.Generator().manual_seed(seed)
  sc = dasalc.DASALCScorer(d, w, h, dropout=dropout, input_noise_stddev=noise,
                           batch_norm_moment=0.9, precision=precision, seed=seed)
  with torch.no_grad():
    for name in sc.KERNELS:
      b = sc.bias(name)
      b.copy_(torch.randn(b.shape, generator=gen) * 0.1)
    for name in sc.NORMS:
      gm, be = sc.batch_norm(name)
      gm.copy_(1.0 + torch.randn(gm.shape, generator=gen) * 0.2)
      be.copy_(torch.randn(be.shape, generator=gen) * 0.2)
      mean, var = sc.moving_stats(name)
      mean.copy_(torch.randn(mean.shape, generator=gen) * 0.3)
      var.copy_(0.5 + torch.rand(var.shape, generator=gen))
  return sc, gen


def _next_seed(sc, training):
  draws = training and (sc.dropout > 0 or sc.input_noise_stddev > 0)
  return (sc._base << 32) | ((sc._calls + (1 if draws else 0)) & 0xFFFFFFFF)


def _oracle(sc, x, e, mask, training, seed, flat=None, state=None):
  flat = sc.flat.detach().cpu().double() if flat is None else flat
  state = sc.bn_state.detach().cpu().double() if state is None else state
  return ref.forward(x.double(), e.double(), flat, sc.input_dim, sc.hidden_dim, sc.context_dim,
                     state=state, training=training, rate=sc.dropout,
                     sigma=sc.input_noise_stddev, seed=seed, mask=mask)


SHAPES = [  # (B, N, D, W, h): M = B N is never a multiple of 128
    (4, 75, 136, 512, 100),
    (3, 111, 4, 64, 4),
    (5, 26, 136, 3072, 100),
    (6, 43, 4, 512, 100),
    (4, 50, 136, 64, 4),
]


@pytest.mark.parametrize('shape', SHAPES)
@pytest.mark.parametrize('training', [True, False])
def test_forward_scores_and_moving_stats(shape, training):
  b, n, d, w, h = shape
  sc, gen = _make(d, w, h, 11 + d + w)
  sc.train(training)
  x = ref.transform(torch.randn(b * n, d, generator=gen) * 3).float()
  e = torch.randn(b * n, h, generator=gen)
  mask = _list_mask(b, n, gen)
  state0 = sc.bn_state.detach().cpu().double().clone()
  seed = _next_seed(sc, training)
  got = sc((x.cuda(), e.cuda()), mask.cuda()).detach()
  torch.cuda.synchronize()
  want, stats = _oracle(sc, x, e, mask, training, seed, state=state0)
  err = (got.cpu().double() - want).abs().max().item()
  assert err <= 1e-5 * want.abs().max().item(), (err, want.abs().max().item())
  assert bool((got.cpu()[~mask] == math.log(1e-10)).all())
  if training:
    assert len(stats) == 4
    new = ref.updated_state(state0, stats, 0.9)
    assert (sc.bn_state.cpu().double() - new).abs().max().item() < 1e-5
  else:
    assert torch.equal(sc.bn_state.cpu().double(), state0)


def _rel_l2(a, b):
  return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


@pytest.mark.parametrize('shape', [SHAPES[0], SHAPES[1], SHAPES[3], SHAPES[2]])
@pytest.mark.parametrize('training', [True, False])
def test_gradients_every_block_and_embedding(shape, training, monkeypatch):
  """Relative L2 error of every parameter block and of dE against fp64 autograd, with the
  three ReLUs gated as the kernel gated them (_dasalc_refs.kernel_gates) and every gate
  checked against its layer recomputed from the kernel's stored input
  (_dasalc_refs.local_checks).  At W = 3072 the ReLUs hold ~10^6 gates and a few pre-activations lie
  within fp32 rounding of zero; an ungated fp64 reference may take the other branch there,
  which moves whole dW columns.  With the gates shared every shape is held to 1e-4."""
  b, n, d, w, h = shape
  sc, gen = _make(d, w, h, 5 + w)
  sc.train(training)
  x = ref.transform(torch.randn(b * n, d, generator=gen) * 3).float()
  e = torch.randn(b * n, h, generator=gen)
  mask = _list_mask(b, n, gen)
  r = torch.randn(b * n, generator=gen)
  state0 = sc.bn_state.detach().cpu().double().clone()
  seed = _next_seed(sc, training)
  workspaces = []
  new_workspace = sc._new_workspace
  monkeypatch.setattr(sc, '_new_workspace', lambda m: workspaces.append(new_workspace(m)) or
                      workspaces[-1])
  ec = e.cuda().requires_grad_()
  s = sc((x.cuda(), ec), mask.cuda())
  s.backward(r.cuda())
  torch.cuda.synchronize()
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  kg = ref.kernel_gates(workspaces[0], d, w, h, b * n, sms)
  kg = {k: [g.cpu() for g in v] if k == 'hidden' else v.cpu() for k, v in kg.items()}
  # every sign word, t and c explained by the input the kernel stored for its layer
  local = ref.local_checks(kg, sc.flat.detach().cpu().double(), d, w, h)
  assert max(local[k] for k in ('relu1', 'relu2', 't', 'c')) <= 1, local
  assert min(local['judged1'], local['judged2']) > 0.8, local
  gates = {'hidden': kg['hidden'], 'cross': kg['cross']}
  flat = sc.flat.detach().cpu().double().requires_grad_()
  ed = e.double().requires_grad_()
  kw = dict(state=state0, training=training, rate=sc.dropout, sigma=sc.input_noise_stddev,
            seed=seed)
  want, _ = ref.forward(x.double(), ed, flat, d, w, h, mask=mask, gates=gates, **kw)
  (want * r.double()).sum().backward()
  errs = ref.block_errors(sc.flat.grad.cpu(), flat.grad, d, w, h)
  assert max(errs.values()) < 1e-4, errs
  assert _rel_l2(ec.grad.cpu().double(), ed.grad) < 1e-4


def test_tf32_forward_within_stated_tolerance():
  b, n, d, w, h = SHAPES[0]
  sc, gen = _make(d, w, h, 3, precision='tf32')
  x = ref.transform(torch.randn(b * n, d, generator=gen) * 3).float()
  e = torch.randn(b * n, h, generator=gen)
  mask = _list_mask(b, n, gen)
  for training in (True, False):
    sc.train(training)
    state0 = sc.bn_state.detach().cpu().double().clone()
    seed = _next_seed(sc, training)
    got = sc((x.cuda(), e.cuda()), mask.cuda()).detach().cpu().double()
    want, _ = _oracle(sc, x, e, mask, training, seed, state=state0)
    assert (got - want).abs().max().item() <= 2e-2 * want.abs().max().item()


def test_two_identical_calls_give_identical_bits():
  b, n, d, w, h = SHAPES[0]
  sc, gen = _make(d, w, h, 8)
  m = b * n
  x = ref.transform(torch.randn(m, d, generator=gen) * 3).cuda()
  x = x.float()
  e = torch.randn(m, h, generator=gen).cuda()
  mask = _list_mask(b, n, gen).to(torch.uint8).cuda()
  ds = torch.randn(m, generator=gen).cuda()
  cfg = sc._run_cfg(training=True)
  state0 = sc.bn_state.clone()
  outs = []
  for _ in range(2):
    sc.bn_state.copy_(state0)
    ws = sc._new_workspace(m)
    scores = torch.empty(m, device='cuda')
    grads = torch.empty_like(sc.flat.data)
    de = torch.empty(m, h + 4, device='cuda')
    st = _C.stream()
    _C.check(_C.lib.tfr_dasalc_fwd(_C.ptr(x), _C.ptr(e), h, m, ctypes.byref(cfg),
                                   _C.ptr(sc.flat.data), _C.ptr(mask), _C.ptr(ws),
                                   _C.ptr(scores), _C.PREC_TF32X3, st))
    _C.check(_C.lib.tfr_dasalc_bwd(_C.ptr(x), m, ctypes.byref(cfg), _C.ptr(sc.flat.data),
                                   _C.ptr(ds), _C.ptr(mask), _C.ptr(ws), _C.ptr(grads),
                                   _C.ptr(de), h + 4, _C.PREC_TF32X3, st))
    torch.cuda.synchronize()
    outs.append((scores.clone(), grads.clone(), de[:, :h].clone(), sc.bn_state.clone()))
  for a, b_ in zip(*outs):
    assert torch.equal(a, b_)


def test_log1p_cutoff_kernel():
  x = torch.tensor([0.0, 1.0, -1.0, -3.0, 1e20, -1e20])
  got = dasalc.log1p_cutoff(x.cuda()).cpu().double()
  want = torch.tensor([0.0, math.log(2), -math.log(2), -math.log(4), 30.0, -30.0],
                      dtype=torch.float64)
  assert (got - want).abs().max().item() < 1e-6
  r = torch.randn(1000, 37) * torch.logspace(-3, 15, 37)
  got = dasalc.log1p_cutoff(r.cuda(), cutoff=12.0).cpu().double()
  assert (got - ref.transform(r, 12.0)).abs().max().item() < 2e-6


# -- the trainer ------------------------------------------------------------------
def _trainer(seed, d, w, h, lr=0.05, rate=0.2, noise=0.5):
  din = tfr.keras.layers.DocumentInteractionAttention(2, h, 1, dropout=rate,
                                                      input_noise_stddev=noise, seed=seed)
  sc, _ = _make(d, w, h, seed + 1, dropout=rate, noise=noise)
  tr = tfr.train.DASALCRankingTrainer(din, sc, tfr.keras.losses.get('softmax_loss'),
                                      optimizer='adagrad', learning_rate=lr)
  return tr, din, sc


def _din_seed(din, training):
  draws = training and (din.dropout > 0 or din.input_noise_stddev)
  return (din._base << 32) | ((din._calls + (1 if draws else 0)) & 0xFFFFFFFF)


def _oracle_step(tr, din, sc, x, y, flat, state, training=True):
  """Scores (and, in training, loss and flat gradient) of transform -> circular pad -> DIN ->
  DASALC -> RestoreList -> SoftmaxLoss, in fp64 with the trainer's next draws replayed."""
  b, n, d = x.shape
  mask = y >= 0
  flat = flat.clone().requires_grad_(training)
  nd = din.flat.numel()
  xd = ref.transform(x)
  idx, _ = oracle_utils.padded_nd_indices(mask)
  xd = torch.gather(xd, 1, idx.unsqueeze(-1).expand(-1, -1, d))
  ds = _din_seed(din, training)
  keeps = noise = None
  if training:
    keeps = odin.keep_masks(ds, b, n, din.num_heads, din.head_size, din.num_layers, din.dropout)
    noise = odin.noise(ds, b, n, din.head_size, din.input_noise_stddev)
  emb = odin.forward(xd, mask, flat[:nd], din.num_heads, din.head_size, din.num_layers,
                     rate=din.dropout, keeps=keeps, noise_add=noise)
  s, stats = ref.forward(xd.reshape(b * n, d), emb.reshape(b * n, -1), flat[nd:], d,
                         sc.hidden_dim, sc.context_dim, state=state, training=training,
                         rate=sc.dropout, sigma=sc.input_noise_stddev,
                         seed=_next_seed(sc, training))
  logits = oracle_scorer.restore_list(s.reshape(b, n), mask)
  if not training:
    return logits.detach(), None, None, None
  loss = oracle_losses.SoftmaxLoss()(y.double(), logits)
  loss.backward()
  return logits.detach(), loss.item(), flat.grad, ref.updated_state(state, stats, 0.9)


def _batch(gen, b, n, d):
  x = torch.randn(b, n, d, generator=gen) * 4
  y = torch.randint(0, 5, (b, n), generator=gen).float()
  y[torch.rand(b, n, generator=gen) < 0.3] = -1.0
  y[0, :] = torch.randint(0, 5, (n,), generator=gen).float()
  y[1, 1:] = -1.0   # a single-item list
  return x, y


def test_trainer_three_adagrad_steps_and_predict():
  b, n, d, w, h = 6, 30, 16, 64, 16
  tr, din, sc = _trainer(21, d, w, h)
  gen = torch.Generator().manual_seed(4)
  flat = tr.tower.flat.detach().cpu().double()
  state = sc.bn_state.detach().cpu().double()
  accum = torch.full_like(flat, 0.1)
  for _ in range(3):
    x, y = _batch(gen, b, n, d)
    _, want_loss, g, state = _oracle_step(tr, din, sc, x, y, flat, state)
    got = float(tr.train_step(x.cuda(), y.cuda()))
    torch.cuda.synchronize()
    assert abs(got - want_loss) <= 1e-5 * max(1.0, abs(want_loss)), (got, want_loss)
    assert _rel_l2(tr.grads.cpu().double(), g) < 1e-4
    accum += g ** 2
    flat = flat - 0.05 * g / (accum.sqrt() + 1e-7)
  assert (tr.tower.flat.detach().cpu().double() - flat).abs().max().item() < 1e-4
  assert (sc.bn_state.cpu().double() - state).abs().max().item() < 1e-4
  assert din.flat.data_ptr() == tr.tower.flat.data_ptr()
  assert sc.flat.data_ptr() == tr.tower.flat.data_ptr() + 4 * din.flat.numel()
  # predict: the same chain in inference mode (moving statistics, no draws)
  x, y = _batch(gen, b, n, d)
  calls = (din._calls, sc._calls)
  got = tr.predict(x.cuda(), y_true=y.cuda()).cpu().double()
  assert (din._calls, sc._calls) == calls
  want, _, _, _ = _oracle_step(tr, din, sc, x, y, tr.tower.flat.detach().cpu().double(),
                               sc.bn_state.detach().cpu().double(), training=False)
  valid = y >= 0
  err = (got[valid] - want[valid]).abs().max().item()
  assert err <= 1e-5 * want[valid].abs().max().item(), err


def _fixture_batches(path, b=4):
  spec = {'custom_features_%d' % (i + 1): (1, 0.0) for i in range(136)}
  spec['utility'] = (1, -1.0)
  return tfr.data.elwc_batches(path, b, 200, None, spec, 'utility')


def test_pipeline_fit_checkpoint_resumes(tmp_path):
  path = os.path.join(NUMERICAL, 'train_numerical_elwc.tfrecord')

  def run(steps, ckdir, skip=0):
    # no noise / dropout: the draws' per-call counters are not part of a checkpoint
    tr, _, _ = _trainer(3, 136, 64, 16, rate=0.0, noise=0.0)
    it = itertools.islice((bt for _ in range(50) for bt in _fixture_batches(path)), skip, None)
    tfr.pipeline.fit(tr, it, steps, checkpoint_dir=ckdir, log_fn=lambda m: None)
    return tr
  a = str(tmp_path / 'a')
  run(2, a)
  resumed = run(4, a, skip=2)   # resumes at step 2 and trains on batches 3 and 4
  fresh = run(4, str(tmp_path / 'b'))
  assert torch.equal(resumed.tower.flat.detach(), fresh.tower.flat.detach())
  assert torch.equal(resumed.tower.bn_state, fresh.tower.bn_state)
  res = tfr.pipeline.evaluate(fresh, list(_fixture_batches(path)))
  assert res and all(float(v) == float(v) for v in res.values())


def test_example_script_runs():
  out = subprocess.run(
      [sys.executable, os.path.join(ROOT, 'examples', 'dasalc_train.py'),
       '--train_path', os.path.join(NUMERICAL, 'train_numerical_elwc.tfrecord'),
       '--eval_path', os.path.join(NUMERICAL, 'vali_numerical_elwc.tfrecord'),
       '--num_train_steps', '300', '--batch_size', '8'],
      capture_output=True, text=True, timeout=900, cwd=ROOT)
  assert out.returncode == 0, out.stdout + out.stderr
  assert 'step 300 loss' in out.stdout and 'ndcg' in out.stdout.lower(), out.stdout
  print(out.stdout[-2000:])
