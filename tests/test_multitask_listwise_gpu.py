"""Multi-task listwise ranking: DASALC with a [W, T] output layer (tfr_dasalc_fwd_tasks /
_bwd_tasks) against _multitask_listwise_refs.py's fp64 restatement, and the multi-task DIN and
DASALC trainers against the fp64 composition (oracle DIN, fp64 tower / DASALC, per-task oracle
losses, Adagrad).  Tolerances are test_dasalc_gpu.py's: 3xTF32 scores to 1e-5 of the largest
|score|, every gradient block to 1e-4 relative L2, with the ReLU gates taken from the kernel."""
import ctypes
import math
import os
import subprocess
import sys

import pytest
import torch

import ranking_b200 as tfr
from ranking_b200 import _C
from oracle import din as odin
from oracle import keras_losses as OL
from oracle import scorer as oracle_scorer
from oracle import utils as oracle_utils
import _dasalc_refs as ref
import _multitask_listwise_refs as mref
from test_dasalc_gpu import _din_seed, _list_mask, _make, _next_seed, _rel_l2

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG_EPS = float(torch.tensor(math.log(1e-10), dtype=torch.float32))   # the kernels' fill


def _make_tasks(d, w, h, t, seed, **kw):
  """A single-task scorer (made as test_dasalc_gpu does) and a T-task scorer with the same
  parameters and moving statistics, whose task u has output column u = small random values."""
  sc1, gen = _make(d, w, h, seed, **kw)
  sct = tfr.research.dasalc.DASALCScorer(d, w, h, dropout=sc1.dropout,
                                         input_noise_stddev=sc1.input_noise_stddev,
                                         batch_norm_moment=0.9, precision=sc1.precision,
                                         seed=seed, output_units=t)
  flat1 = sc1.flat.detach().cpu().double()
  flats = [flat1.clone() for _ in range(t)]
  o, _ = mref._head(d, w, h)
  for u in range(1, t):
    flats[u][o:o + w + 1] = torch.randn(w + 1, generator=gen, dtype=torch.float64) * 0.2
  with torch.no_grad():
    sct.flat.copy_(mref.single_to_tasks(flats, d, w, h).float())
    sct.bn_state.copy_(sc1.bn_state)
  sct._base = sc1._base
  return sc1, sct, gen


def _call(sc, x, e, mask, ds, weights, t, precision, training, single=False):
  """One forward + backward through the C API; (scores, grads, dE, bn_state after)."""
  m, h = x.shape[0], sc.context_dim
  cfg = sc._run_cfg(training=training)
  ws = sc._new_workspace(m)
  scores = torch.empty(t, m, device='cuda')
  grads = torch.empty_like(sc.flat.data)
  de = torch.empty(m, h + 4, device='cuda')
  st = _C.stream()
  if single:
    _C.check(_C.lib.tfr_dasalc_fwd(_C.ptr(x), _C.ptr(e), h, m, ctypes.byref(cfg),
                                   _C.ptr(sc.flat.data), _C.ptr(mask), _C.ptr(ws),
                                   _C.ptr(scores), precision, st))
    _C.check(_C.lib.tfr_dasalc_bwd(_C.ptr(x), m, ctypes.byref(cfg), _C.ptr(sc.flat.data),
                                   _C.ptr(ds), _C.ptr(mask), _C.ptr(ws), _C.ptr(grads),
                                   _C.ptr(de), h + 4, precision, st))
  else:
    w = None if weights is None else (ctypes.c_float * t)(*weights)
    _C.check(_C.lib.tfr_dasalc_fwd_tasks(_C.ptr(x), _C.ptr(e), h, m, ctypes.byref(cfg),
                                         _C.ptr(sc.flat.data), _C.ptr(mask), _C.ptr(ws),
                                         _C.ptr(scores), t, precision, st))
    _C.check(_C.lib.tfr_dasalc_bwd_tasks(_C.ptr(x), m, ctypes.byref(cfg), _C.ptr(sc.flat.data),
                                         _C.ptr(ds), w, _C.ptr(mask), _C.ptr(ws), _C.ptr(grads),
                                         _C.ptr(de), h + 4, t, precision, st))
  torch.cuda.synchronize()
  return scores, grads, de[:, :h].clone(), sc.bn_state.clone()


def _inputs(gen, b, n, d, h, t):
  m = b * n
  x = ref.transform(torch.randn(m, d, generator=gen) * 3).float()
  e = torch.randn(m, h, generator=gen)
  mask = _list_mask(b, n, gen)
  ds = torch.randn(t, m, generator=gen)
  return x, e, mask, ds


@pytest.mark.parametrize('precision', ['tf32x3', 'tf32'])
@pytest.mark.parametrize('training', [True, False])
@pytest.mark.parametrize('weights', [None, [1.0]])
def test_one_task_is_the_single_task_bits(precision, training, weights):
  b, n, d, w, h = 4, 75, 136, 512, 100
  sc, gen = _make(d, w, h, 17, precision=precision)
  x, e, mask, ds = _inputs(gen, b, n, d, h, 1)
  x, e, m8, ds = x.cuda(), e.cuda(), mask.to(torch.uint8).cuda(), ds.cuda()
  prec = sc._precision
  state0 = sc.bn_state.clone()
  seed_calls = sc._calls
  a = _call(sc, x, e, m8, ds, weights, 1, prec, training, single=True)
  sc.bn_state.copy_(state0)
  sc._calls = seed_calls
  bt = _call(sc, x, e, m8, ds, weights, 1, prec, training)
  for u, v in zip(a, bt):
    assert torch.equal(u, v)


@pytest.mark.parametrize('t,weights', [(2, [1.0, 0.0]), (3, [0.5, -1.25, 2.0]),
                                       (8, [1.0, 0.0, -0.5, 3.0, 0.25, 1.0, -2.0, 0.75])])
@pytest.mark.parametrize('training', [True, False])
def test_planes_and_gradients_against_fp64(t, weights, training):
  """Planes, every gradient block and dE against fp64 autograd of sum_u w_u <plane_u, r_u>,
  with the ReLU gates of a single-task call on the same inputs (the layers before the output
  layer do not depend on T).  Masked rows: ln(1e-10) on every plane, no gradient."""
  b, n, d, w, h = 4, 75, 136, 512, 100
  sc1, sct, gen = _make_tasks(d, w, h, t, 5 + t)
  x, e, mask, ds = _inputs(gen, b, n, d, h, t)
  sc1.train(training)
  sct.train(training)
  state0 = sct.bn_state.detach().cpu().double().clone()
  seed = _next_seed(sct, training)
  workspaces = []
  new_ws = sc1._new_workspace
  sc1._new_workspace = lambda m: workspaces.append(new_ws(m)) or workspaces[-1]
  sc1((x.cuda(), e.cuda()), mask.cuda())   # the gates
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  kg = ref.kernel_gates(workspaces[0], d, w, h, b * n, sms)
  gates = {'hidden': [g.cpu() for g in kg['hidden']], 'cross': kg['cross'].cpu()}
  scores, grads, de, state = _call(sct, x.cuda(), e.cuda(), mask.to(torch.uint8).cuda(),
                                   ds.cuda(), weights, t, sct._precision, training)
  flat = sct.flat.detach().cpu().double().requires_grad_()
  ed = e.double().requires_grad_()
  want, stats = mref.forward_tasks(x.double(), ed, flat, d, w, h, t, state=state0,
                                   training=training, rate=sct.dropout,
                                   sigma=sct.input_noise_stddev, seed=seed, mask=mask,
                                   gates=gates)
  got = scores.cpu().double()
  valid = mask.reshape(-1)
  assert (got[:, valid] - want[:, valid]).abs().max() <= 1e-5 * want[:, valid].abs().max()
  assert bool((got[:, ~valid] == LOG_EPS).all())
  wt = torch.tensor(weights, dtype=torch.float64)[:, None]
  (want * ds.double() * wt).sum().backward()
  errs = mref.block_errors(grads.cpu(), flat.grad, d, w, h, t)
  assert max(errs.values()) < 1e-4, errs
  assert _rel_l2(de.cpu().double(), ed.grad) < 1e-4
  o, _ = mref._head(d, w, h)
  g = grads.cpu().reshape(-1)
  for u, wu in enumerate(weights):   # a task of weight 0 leaves its column untouched
    if wu == 0:
      assert bool((g[o:o + w * t].reshape(w, t)[:, u] == 0).all()) and g[o + w * t + u] == 0
  if training:
    new = ref.updated_state(state0, stats, 0.9)
    assert (state.cpu().double() - new).abs().max().item() < 1e-5


def test_two_identical_calls_give_identical_bits():
  b, n, d, w, h, t = 4, 75, 136, 512, 100, 3
  _, sct, gen = _make_tasks(d, w, h, t, 8)
  x, e, mask, ds = [v.cuda() for v in _inputs(gen, b, n, d, h, t)]
  m8 = mask.to(torch.uint8)
  state0 = sct.bn_state.clone()
  outs = []
  for _ in range(2):
    sct.bn_state.copy_(state0)
    sct._calls = 0
    outs.append(_call(sct, x, e, m8, ds, [0.5, -1.0, 2.0], t, sct._precision, True))
  for a, b_ in zip(*outs):
    assert torch.equal(a, b_)


# -- the trainers --------------------------------------------------------------------
ORACLE = {'softmax_loss': OL.SoftmaxLoss, 'sigmoid_cross_entropy_loss': OL.SigmoidCrossEntropyLoss,
          'mean_squared_loss': OL.MeanSquaredLoss, 'approx_ndcg_loss': OL.ApproxNDCGLoss}
LOSS_SETS = [{'rel': 'softmax_loss', 'click': 'sigmoid_cross_entropy_loss'},
             {'rel': 'approx_ndcg_loss', 'click': 'mean_squared_loss'}]


def _labels(gen, b, n, tasks):
  """Partial labels: every task misses some items the other task labels; list 1 has one
  item, list 2 none."""
  valid = torch.rand(b, n, generator=gen) < 0.8
  valid[1, 1:] = False
  valid[2] = False
  ys = {}
  for i, task in enumerate(tasks):
    y = (torch.randint(0, 5, (b, n), generator=gen).float() if i == 0 else
         (torch.rand(b, n, generator=gen) < 0.4).float())
    y[~valid] = -1.0
    y[torch.rand(b, n, generator=gen) < 0.2] = -1.0
    ys[task] = y
  return ys


def _union(ys):
  m = None
  for y in ys.values():
    m = (y >= 0) if m is None else m | (y >= 0)
  return m


def _dasalc_trainer(losses, weights, seed, d=16, w=64, h=16, rate=0.2, noise=0.5):
  din = tfr.keras.layers.DocumentInteractionAttention(2, h, 1, dropout=rate,
                                                      input_noise_stddev=noise, seed=seed)
  _, sct, _ = _make_tasks(d, w, h, len(losses), seed + 1, dropout=rate, noise=noise)
  tr = tfr.train.MultiTaskDASALCRankingTrainer(
      din, sct, {k: tfr.keras.losses.get(v) for k, v in losses.items()}, loss_weights=weights,
      optimizer='adagrad', learning_rate=0.05)
  return tr, din, sct


def _dasalc_oracle(tr, din, sc, x, ys, losses, weights, flat, state, training=True):
  b, n, d = x.shape
  t = len(losses)
  mask = _union(ys)
  flat = flat.clone().requires_grad_(training)
  nd = din.flat.numel()
  xd = ref.transform(x)
  idx, _ = oracle_utils.padded_nd_indices(mask)
  xd = torch.gather(xd, 1, idx.unsqueeze(-1).expand(-1, -1, d))
  dseed = _din_seed(din, training)
  keeps = noise = None
  if training:
    keeps = odin.keep_masks(dseed, b, n, din.num_heads, din.head_size, din.num_layers,
                            din.dropout)
    noise = odin.noise(dseed, b, n, din.head_size, din.input_noise_stddev)
  emb = odin.forward(xd, mask, flat[:nd], din.num_heads, din.head_size, din.num_layers,
                     rate=din.dropout, keeps=keeps, noise_add=noise)
  planes, stats = mref.forward_tasks(xd.reshape(b * n, d), emb.reshape(b * n, -1), flat[nd:],
                                     d, sc.hidden_dim, sc.context_dim, t, state=state,
                                     training=training, rate=sc.dropout,
                                     sigma=sc.input_noise_stddev, seed=_next_seed(sc, training))
  return _finish(planes, mask, ys, losses, weights, flat, training, stats, state, b, n)


def _finish(planes, mask, ys, losses, weights, flat, training, stats, state, b, n):
  logits = {k: oracle_scorer.restore_list(planes[i].reshape(b, n), mask)
            for i, k in enumerate(losses)}
  if not training:
    return logits, None, None, None
  total = sum((weights or {}).get(k, 1.0) * ORACLE[v]()(ys[k].double(), logits[k])
              for k, v in losses.items())
  total.backward()
  new_state = None if stats is None else ref.updated_state(state, stats, 0.9)
  return logits, total.item(), flat.grad, new_state


@pytest.mark.parametrize('losses', LOSS_SETS)
@pytest.mark.parametrize('weights', [None, {'click': -0.5}, {'rel': 2.0, 'click': 0.25}])
def test_dasalc_trainer_step_against_fp64(losses, weights):
  b, n, d = 6, 30, 16
  tr, din, sc = _dasalc_trainer(losses, weights, 21)
  gen = torch.Generator().manual_seed(4)
  flat = tr.tower.flat.detach().cpu().double()
  state = sc.bn_state.detach().cpu().double()
  x = torch.randn(b, n, d, generator=gen) * 4
  ys = _labels(gen, b, n, list(losses))
  _, want, g, state = _dasalc_oracle(tr, din, sc, x, ys, losses, weights, flat, state)
  got = float(tr.train_step(x.cuda(), {k: y.cuda() for k, y in ys.items()}))
  torch.cuda.synchronize()
  assert abs(got - want) <= 1e-5 * max(1.0, abs(want)), (got, want)
  assert _rel_l2(tr.grads.cpu().double(), g) < 1e-4
  assert (sc.bn_state.cpu().double() - state).abs().max().item() < 1e-4
  flat = flat - 0.05 * g / ((0.1 + g ** 2).sqrt() + 1e-7)
  assert (tr.tower.flat.detach().cpu().double() - flat).abs().max().item() < 1e-4
  # predict: one plane per task, the fill on the items without any label
  x2 = torch.randn(b, n, d, generator=gen) * 4
  ys2 = _labels(gen, b, n, list(losses))
  pred = tr.predict(x2.cuda(), labels={k: y.cuda() for k, y in ys2.items()})
  want2, _, _, _ = _dasalc_oracle(tr, din, sc, x2, ys2, losses, weights,
                                  tr.tower.flat.detach().cpu().double(),
                                  sc.bn_state.detach().cpu().double(), training=False)
  valid = _union(ys2)
  assert list(pred) == list(losses)
  for k in losses:
    p = pred[k].cpu().double()
    assert p.shape == (b, n) and bool((p[~valid] == LOG_EPS).all())
    assert (p[valid] - want2[k][valid]).abs().max() <= 1e-5 * want2[k][valid].abs().max()


def _din_trainer(losses, weights, seed, d=16, h=8, hidden=(32, 16), multi=True):
  torch.manual_seed(seed)
  din = tfr.keras.layers.DocumentInteractionAttention(2, h, 1, dropout=0.0, seed=seed).build(d)
  units = len(losses) if multi else 1
  tower = tfr.keras.layers.create_tower(list(hidden), units, activation='relu', input_dim=d + h,
                                        use_batch_norm=False, dropout=0.0, seed=seed + 1,
                                        precision='tf32x3')
  kw = dict(optimizer='adagrad', learning_rate=0.05)
  if multi:
    return tfr.train.MultiTaskDINRankingTrainer(
        din, tower, {k: tfr.keras.losses.get(v) for k, v in losses.items()},
        loss_weights=weights, **kw), din, tower
  return tfr.train.DINRankingTrainer(din, tower, tfr.keras.losses.get(
      list(losses.values())[0]), **kw), din, tower


def _din_oracle(din, tower, x, ys, losses, weights, flat, training=True):
  b, n, d = x.shape
  mask = _union(ys)
  flat = flat.clone().requires_grad_(training)
  nd = din.flat.numel()
  xd = x.double()
  emb = odin.forward(xd, mask, flat[:nd], din.num_heads, din.head_size, din.num_layers)
  a = torch.cat([xd, emb], -1).reshape(b * n, -1)
  off, dims = nd, tower.dims
  for i in range(len(dims) - 1):
    wgt = flat[off:off + dims[i] * dims[i + 1]].reshape(dims[i], dims[i + 1])
    off += dims[i] * dims[i + 1]
    a = a @ wgt + flat[off:off + dims[i + 1]]
    off += dims[i + 1]
    if i < len(dims) - 2:
      a = torch.relu(a)
  return _finish(a.t(), mask, ys, losses, weights, flat, training, None, None, b, n)


@pytest.mark.parametrize('losses', LOSS_SETS)
@pytest.mark.parametrize('weights', [None, {'rel': 2.0, 'click': -0.5}])
def test_din_trainer_step_against_fp64(losses, weights):
  b, n, d = 6, 30, 16
  tr, din, tower = _din_trainer(losses, weights, 9)
  gen = torch.Generator().manual_seed(2)
  flat = tr.tower.flat.detach().cpu().double()
  x = torch.randn(b, n, d, generator=gen)
  ys = _labels(gen, b, n, list(losses))
  _, want, g, _ = _din_oracle(din, tower, x, ys, losses, weights, flat)
  got = float(tr.train_step(x.cuda(), {k: y.cuda() for k, y in ys.items()}))
  torch.cuda.synchronize()
  assert abs(got - want) <= 1e-5 * max(1.0, abs(want)), (got, want)
  assert _rel_l2(tr.grads.cpu().double(), g) < 1e-4
  pred = tr.predict(x.cuda(), mask=_union(ys).cuda())
  want2, _, _, _ = _din_oracle(din, tower, x, ys, losses, weights,
                               tr.tower.flat.detach().cpu().double(), training=False)
  valid = _union(ys)
  for k in losses:
    p = pred[k].cpu().double()
    assert bool((p[~valid] == LOG_EPS).all())
    assert (p[valid] - want2[k][valid]).abs().max() <= 1e-5 * want2[k][valid].abs().max()


@pytest.mark.parametrize('kind', ['din', 'dasalc'])
def test_one_task_trainer_is_the_single_task_trainer_bits(kind):
  b, n, d = 6, 30, 16
  losses = {'rel': 'softmax_loss'}
  if kind == 'din':
    multi, _, _ = _din_trainer(losses, None, 5)
    single, _, _ = _din_trainer(losses, None, 5, multi=False)
  else:
    multi, _, _ = _dasalc_trainer(losses, None, 5)
    din = tfr.keras.layers.DocumentInteractionAttention(2, 16, 1, dropout=0.2,
                                                        input_noise_stddev=0.5, seed=5)
    sc, _ = _make(d, 64, 16, 6, dropout=0.2, noise=0.5)
    single = tfr.train.DASALCRankingTrainer(din, sc, tfr.keras.losses.get('softmax_loss'),
                                            optimizer='adagrad', learning_rate=0.05)
  assert torch.equal(multi.tower.flat.data, single.tower.flat.data)
  gen = torch.Generator().manual_seed(7)
  for _ in range(3):
    x = (torch.randn(b, n, d, generator=gen) * 4).cuda()
    y = _labels(gen, b, n, ['rel'])['rel'].cuda()
    lm = float(multi.train_step(x, {'rel': y}))
    ls = float(single.train_step(x, y, mask=(y >= 0)))
    assert lm == ls
    assert torch.equal(multi.tower.flat.data, single.tower.flat.data)
    assert torch.equal(multi.tower.bn_state, single.tower.bn_state)


@pytest.mark.parametrize('kind', ['din', 'dasalc'])
def test_checkpoint_resume_continues_bit_exactly(kind, tmp_path):
  losses = {'rel': 'softmax_loss', 'click': 'sigmoid_cross_entropy_loss'}
  b, n, d = 6, 30, 16

  def make():
    if kind == 'din':
      return _din_trainer(losses, {'click': 0.5}, 3)[0]
    # no draws: their per-call counters are not part of a checkpoint
    return _dasalc_trainer(losses, {'click': 0.5}, 3, rate=0.0, noise=0.0)[0]

  gen = torch.Generator().manual_seed(1)
  batches = []
  for _ in range(4):
    x = torch.randn(b, n, d, generator=gen).cuda()
    batches.append((x, {k: y.cuda() for k, y in _labels(gen, b, n, list(losses)).items()}))
  a = make()
  for x, ys in batches[:2]:
    a.train_step(x, ys)
  path = str(tmp_path / 'ckpt.pt')
  tfr.pipeline.save_checkpoint(a, path, 2)
  resumed = make()
  assert tfr.pipeline.load_checkpoint(resumed, path) == 2
  for x, ys in batches[2:]:
    a.train_step(x, ys)
    resumed.train_step(x, ys)
  assert torch.equal(a.tower.flat.data, resumed.tower.flat.data)
  assert torch.equal(a.accum, resumed.accum)
  assert torch.equal(a.tower.bn_state, resumed.tower.bn_state)


@pytest.mark.parametrize('kind', ['din', 'dasalc'])
def test_pipeline_epoch_logs_every_task(kind, tmp_path):
  losses = {'rel': 'softmax_loss', 'click': 'sigmoid_cross_entropy_loss'}
  b, n, d = 8, 20, 16
  gen = torch.Generator().manual_seed(0)

  def batches():
    g = torch.Generator().manual_seed(3)
    for _ in range(4):
      x = torch.randn(b, n, d, generator=g)
      ys = _labels(g, b, n, list(losses))
      yield x, ys, _union(ys), None

  def model():
    if kind == 'din':
      _, din, tower = _din_trainer(losses, None, 4)
      return din, tower
    _, din, sc = _dasalc_trainer(losses, None, 4)
    return din, sc

  cls = {'din': tfr.train.MultiTaskDINRankingTrainer,
         'dasalc': tfr.train.MultiTaskDASALCRankingTrainer}[kind]
  hp = tfr.pipeline.PipelineHparams(model_dir=str(tmp_path), num_epochs=1, steps_per_epoch=3,
                                    validation_steps=2, learning_rate=0.05, loss=losses,
                                    loss_weights={'click': 0.5})
  p = tfr.pipeline.MultiTaskPipeline(model, batches, batches, hp, log_fn=lambda m: None,
                                     trainer_cls=cls)
  hist = p.train_and_validate()
  assert len(hist) == 1
  logs = hist[0]
  for task in losses:
    assert math.isfinite(logs[task + '_loss'])
    for k in ('ndcg_1', 'ndcg_5', 'ndcg_10', 'ndcg'):
      assert 0.0 <= logs[task + '_metric/' + k] <= 1.0
  assert abs(logs['loss'] - (logs['rel_loss'] + 0.5 * logs['click_loss'])) < 1e-5
  assert os.path.exists(os.path.join(str(tmp_path), 'ckpt.pt'))


@pytest.mark.parametrize('scorer', ['din', 'dasalc'])
def test_example_runs_synthetic(scorer, tmp_path):
  out = subprocess.run([sys.executable, os.path.join(ROOT, 'examples', 'multitask_train.py'),
                        '--synthetic', '--scorer', scorer, '--epochs', '2',
                        '--steps_per_epoch', '8', '--work_dir', str(tmp_path)],
                       capture_output=True, text=True, timeout=900, cwd=ROOT)
  assert out.returncode == 0, out.stdout + out.stderr
  lines = {l.split()[0]: l for l in out.stdout.splitlines() if 'NDCG@5' in l}
  assert set(lines) == {'relevance', 'click'}, out.stdout
  assert ('scorer %s' % scorer) in out.stdout
