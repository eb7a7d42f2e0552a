"""GAMLayer / GAMScorer / GAMRankingTrainer (csrc/gam.cu) against the fp64 oracle
(oracle/gam.py)."""
import numpy as np
import pytest
import torch

from oracle import gam as OG
from oracle import keras_losses as OL
from oracle import scorer as OS

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _need_cuda():
  if not torch.cuda.is_available():
    pytest.skip('no CUDA device')


def _rel(a, b):
  a = torch.as_tensor(a).detach().cpu().double()
  b = torch.as_tensor(b).detach().cpu().double()
  return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def _l2(a, b):
  a = torch.as_tensor(a).detach().cpu().double()
  b = torch.as_tensor(b).detach().cpu().double()
  return float((a - b).norm() / (b.norm() + 1e-30))


def _leaves(p):
  out = []
  for w, b in zip(p['dense_w'], p['dense_b']):
    out += [w, b]
  for g, b in zip(p['bn_gamma'], p['bn_beta']):
    out += [g, b]
  return out


def _pack(p):
  return torch.cat([t.detach().reshape(-1) for t in _leaves(p)])


def _grad(p):
  return torch.cat([t.grad.reshape(-1) if t.grad is not None else torch.zeros(t.numel(),
                                                                           dtype=t.dtype)
                    for t in _leaves(p)])


def _make(tfr, ex_dims, hidden, ctx_dims=(), ctx_hidden=None, act=None, bn=False,
          dropout=0.0, seed=5):
  """A built GAMLayer and oracle parameters (fp64, requires_grad) with identical values;
  biases / BN affine parameters are randomised so that every term is exercised."""
  gam = tfr.keras.layers.GAMLayer(len(ex_dims), hidden, len(ctx_dims), ctx_hidden,
                                  activation=act, use_batch_norm=bn, dropout=dropout,
                                  seed=seed)
  gam.build(ex_dims, list(ctx_dims) or None)
  params = OG.init_gam_params(ex_dims, hidden, ctx_dims, ctx_hidden, use_batch_norm=bn,
                              seed=seed)
  g = torch.Generator().manual_seed(seed)
  towers = params['example'] + params['context']
  for i, p in enumerate(towers):
    for b in p['dense_b']:
      b.uniform_(-0.3, 0.3, generator=g)
    for t in p['bn_gamma']:
      t.uniform_(0.5, 1.5, generator=g)
    for t in p['bn_beta']:
      t.uniform_(-0.3, 0.3, generator=g)
    with torch.no_grad():
      gam.tower_slice(i)[0].copy_(_pack(p).float())
    for t in _leaves(p):
      t.requires_grad_()
  return gam, params


def _moving(gam, params):
  out = {'example': [], 'context': []}
  for i, _ in enumerate(params['example'] + params['context']):
    _, st, dims = gam.tower_slice(i)
    kind = 'example' if i < len(params['example']) else 'context'
    mv, o = {}, 0
    for d, h in enumerate(dims[1:-1] if st.numel() else []):
      mv[d] = [st[o:o + h].detach().cpu().double().clone(),
               st[o + h:o + 2 * h].detach().cpu().double().clone()]
      o += 2 * h
    out[kind].append(mv)
  return out


def _inputs(m, dims, seed):
  g = torch.Generator().manual_seed(seed)
  return [torch.randn(m, d, generator=g) for d in dims]


def _flat_grad(gam, params):
  return torch.cat([_grad(p) for p in params['example'] + params['context']])


@pytest.mark.parametrize('hidden,df,f,act,bn', [
    ([16], 1, 136, None, False),
    ([16, 8], 3, 7, None, False),
    ([8, 12, 4], 1, 5, None, False),
    ([16, 8], 1, 136, 'relu', True),
    ([32, 16], 3, 9, 'relu', True),
    ([], 2, 6, None, False),
])
def test_forward_and_gradient_parity(hidden, df, f, act, bn):
  import ranking_b200 as tfr
  m = 1237
  ex_dims = [df] * f
  if df == 3:
    ex_dims[1] = 1     # one narrower feature
  gam, params = _make(tfr, ex_dims, hidden, act=act, bn=bn)
  xs = _inputs(m, ex_dims, 1)
  up = torch.randn(m, 1, generator=torch.Generator().manual_seed(2))
  gam.train()
  logits, sub, _ = gam(([x.cuda() for x in xs], None))
  (logits * up.cuda()).sum().backward()
  ref, rsub, _ = OG.gam_layer([x.double() for x in xs], None, params, activation=act,
                              use_batch_norm=bn, training=True)
  (ref * up.double()).sum().backward()
  assert _rel(logits, ref) <= 2e-5
  assert _rel(torch.cat(sub, 1), torch.cat(rsub, 1)) <= 2e-5
  got, want = gam.flat.grad, _flat_grad(gam, params)
  if act is None and not bn:
    assert _rel(got, want) <= 2e-4
  else:
    # a pre-activation within rounding of 0 may flip its ReLU branch between fp32 and
    # fp64 (as in test_tower_batch_norm_training): compare in L2
    assert _l2(got, want) <= 1e-2


def test_batch_norm_statistics_and_eval():
  import ranking_b200 as tfr
  m, hidden, ex_dims = 900, [16, 8], [1] * 12 + [2] * 3
  gam, params = _make(tfr, ex_dims, hidden, act='relu', bn=True)
  moving = _moving(gam, params)
  xs = _inputs(m, ex_dims, 3)
  gam.train()
  gam(([x.cuda() for x in xs], None))
  # the kernels update with the fp32 momentum (as tfr_mlp does): 1 - float32(0.999)
  OG.gam_layer([x.double() for x in xs], None, params, activation='relu',
               use_batch_norm=True, training=True, bn_moving=moving,
               momentum=float(np.float32(0.999)))
  got = _moving(gam, params)
  for kind in ('example',):
    for a, b in zip(got[kind], moving[kind]):
      for d in a:
        assert _rel(a[d][0], b[d][0]) <= 1e-5 and _rel(a[d][1], b[d][1]) <= 1e-5
  state = gam.bn_state.clone()
  gam.eval()
  ye, _, _ = gam(([x.cuda() for x in xs], None))
  assert torch.equal(gam.bn_state, state)
  ref, _, _ = OG.gam_layer([x.double() for x in xs], None, params, activation='relu',
                           use_batch_norm=True, training=False, bn_moving=got)
  assert _rel(ye, ref) <= 2e-5


def _keep(seed, layer, m, width, rate):
  with np.errstate(over='ignore'):
    s = np.uint64(seed) * np.uint64(0x100000001B3) + np.uint64(layer + 1)
    idx = np.arange(m * width, dtype=np.uint64)
    z = s + np.uint64(0x9E3779B97F4A7C15) * (idx + np.uint64(1))
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z = z ^ (z >> np.uint64(31))
  u = (z >> np.uint64(40)).astype(np.float32) * np.float32(1.0 / 16777216.0)
  return torch.from_numpy(~(u < np.float32(rate))).reshape(m, width)


@pytest.mark.parametrize('act,bn', [(None, False), ('relu', True)])
def test_dropout_replay(act, bn):
  """Example tower f, layer d draws element m*(F*h) + f*h + u of the block-diagonal
  layer's tfr_mlp mask; replayed through the oracle."""
  import ranking_b200 as tfr
  m, hidden, f, p = 1500, [16, 8], 10, 0.5
  gam, params = _make(tfr, [1] * f, hidden, act=act, bn=bn, dropout=p)
  xs = _inputs(m, [1] * f, 4)
  up = torch.randn(m, 1, generator=torch.Generator().manual_seed(5))
  gam.train()
  gam._dropout_calls = 0
  y, _, _ = gam(([x.cuda() for x in xs], None))
  (y * up.cuda()).sum().backward()
  seed = (gam._dropout_base << 32) | 1
  full = [_keep(seed, d, m, f * h, p).reshape(m, f, h) for d, h in enumerate(hidden)]
  for k in full:
    assert abs(1.0 - float(k.double().mean()) - p) < 0.02
  keeps = {'example': [[k[:, i, :].double() / (1 - p) for k in full] for i in range(f)],
           'context': []}
  ref, _, _ = OG.gam_layer([x.double() for x in xs], None, params, activation=act,
                           use_batch_norm=bn, keep_masks=keeps)
  (ref * up.double()).sum().backward()
  assert _rel(y, ref) <= 2e-5
  assert _l2(gam.flat.grad, _flat_grad(gam, params)) <= (1e-2 if bn else 2e-4)
  gam._dropout_calls = 0
  y2, _, _ = gam(([x.cuda() for x in xs], None))
  assert torch.equal(y2, y)
  y3, _, _ = gam(([x.cuda() for x in xs], None))
  assert not torch.equal(y3, y)


@pytest.mark.parametrize('n_ctx', [1, 2])
def test_context_weighting(n_ctx):
  import ranking_b200 as tfr
  m, ex_dims, ctx_dims = 777, [1, 2, 1], [2, 3][:n_ctx]
  gam, params = _make(tfr, ex_dims, [8, 4], ctx_dims, [6, 5], act='relu', bn=False)
  xs = _inputs(m, ex_dims, 6)
  cs = _inputs(m, ctx_dims, 7)
  up = torch.randn(m, 1, generator=torch.Generator().manual_seed(8))
  gam.train()
  y, sub, w = gam(([x.cuda() for x in xs], [c.cuda() for c in cs]))
  (y * up.cuda()).sum().backward()
  ref, rsub, rw = OG.gam_layer([x.double() for x in xs], [c.double() for c in cs], params,
                               activation='relu')
  (ref * up.double()).sum().backward()
  assert len(w) == n_ctx and all(list(t.shape) == [m, 3] for t in w)
  assert _rel(y, ref) <= 2e-5
  for a, b in zip(w, rw):
    assert _rel(a, b) <= 2e-5
  assert _l2(gam.flat.grad, _flat_grad(gam, params)) <= 1e-4
  # a call without context inputs ignores the context towers (layers.py:758-787)
  gam.flat.grad = None
  for t in [t for p in params['example'] + params['context'] for t in _leaves(p)]:
    t.grad = None
  y0, _, w0 = gam(([x.cuda() for x in xs], None))
  y0.sum().backward()
  r0, _, _ = OG.gam_layer([x.double() for x in xs], None, params, activation='relu')
  r0.sum().backward()
  assert w0 == [] and _rel(y0, r0) <= 2e-5
  assert _l2(gam.flat.grad, _flat_grad(gam, params)) <= 1e-4


def test_one_feature_equals_create_tower():
  """A one-feature GAM without context is create_tower on the same parameters and seed:
  same layout, same BN, same dropout mask (fp32 against fp32)."""
  import ranking_b200 as tfr
  m, d, hidden = 1031, 12, [16, 8]
  gam = tfr.keras.layers.GAMLayer(1, hidden, activation='relu', use_batch_norm=True,
                                  dropout=0.5, seed=3)
  gam.build([d])
  tower = tfr.keras.layers.create_tower(hidden, 1, activation='relu', use_batch_norm=True,
                                        dropout=0.5, input_dim=d, seed=3, precision='fp32')
  with torch.no_grad():
    gam.flat.uniform_(-0.5, 0.5)
    tower.flat.copy_(gam.flat)
  x = torch.randn(m, d).cuda()
  up = torch.randn(m, 1).cuda()
  gam.train()
  tower.train()
  gam._dropout_calls = tower._dropout_calls = 0
  yg, _, _ = gam(([x], None))
  yt = tower(x)
  (yg * up).sum().backward()
  (yt * up).sum().backward()
  assert _rel(yg, yt) <= 1e-5
  assert _l2(gam.flat.grad, tower.flat.grad) <= 1e-4
  assert _rel(gam.bn_state, tower.bn_state) <= 1e-5


def test_determinism():
  import ranking_b200 as tfr
  m, ex_dims = 3000, [1] * 40
  gam, _ = _make(tfr, ex_dims, [16, 8], act='relu', bn=True, dropout=0.5)
  xs = [x.cuda() for x in _inputs(m, ex_dims, 9)]
  outs = []
  for _ in range(2):
    gam._dropout_calls = 0
    gam.flat.grad = None
    y, _, _ = gam((xs, None))
    y.sum().backward()
    outs.append((y.detach().clone(), gam.flat.grad.clone()))
  assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1])


def test_gam_scorer_contract():
  """Sorted keys, circular padding, RestoreList fill (like test_dnn_scorer_contract)."""
  import ranking_b200 as tfr
  b, n = 3, 5
  g = torch.Generator().manual_seed(10)
  ex = {'zeta': torch.randn(b, n, 1, generator=g), 'alpha': torch.randn(b, n, 2, generator=g)}
  cx = {'ctx': torch.randn(b, 2, generator=g)}
  mask = torch.ones(b, n, dtype=torch.bool)
  mask[1, 3:] = False
  mask[2, 1:] = False
  scorer = tfr.keras.model.GAMScorer(example_hidden_layer_dims=[4], context_hidden_layer_dims=[3],
                                     activation='relu', use_batch_norm=False, dropout=0.0,
                                     seed=2)
  out = scorer({k: v.cuda() for k, v in cx.items()}, {k: v.cuda() for k, v in ex.items()},
               mask.cuda())
  gam = scorer.gam
  assert gam.example_dims == [2, 1] and gam.context_dims == [2]   # sorted: alpha, zeta
  params = {'example': [], 'context': []}
  for i in range(3):
    flat, _, dims = gam.tower_slice(i)
    flat = flat.detach().cpu().double()
    p = {'dense_w': [], 'dense_b': [], 'bn_gamma': [], 'bn_beta': []}
    o = 0
    for a, c in zip(dims[:-1], dims[1:]):
      p['dense_w'].append(flat[o:o + a * c].reshape(a, c))
      o += a * c
      p['dense_b'].append(flat[o:o + c])
      o += c
    params['example' if i < 2 else 'context'].append(p)
  ref = OG.gam_scorer({k: v.double() for k, v in cx.items()},
                      {k: v.double() for k, v in ex.items()}, mask, params, activation='relu')
  assert list(out.shape) == [b, n]
  assert _rel(out, ref) <= 2e-5    # includes the ln(1e-10) fill of the padded slots


def _oracle_logits(params, x, y, dims):
  mask = y >= 0
  _, flat = OS.flatten_list({}, {'x': x.double()}, mask, circular_padding=True)
  cols = torch.split(flat['x'], dims, 1)
  logits, _, _ = OG.gam_layer(list(cols), None, params, activation='relu',
                              use_batch_norm=True)
  return OS.restore_list(logits, mask)


def test_trainer_trajectory_and_checkpoint(tmp_path):
  import ranking_b200 as tfr
  b, n, dims = 16, 12, [1] * 10 + [2, 4]
  gam, params = _make(tfr, dims, [16, 8], act='relu', bn=True)
  loss = tfr.keras.losses.get('approx_ndcg_loss')
  trainer = tfr.train.GAMRankingTrainer(gam, loss, dims, optimizer='adagrad',
                                        learning_rate=0.05)
  oloss = OL.get('approx_ndcg_loss')
  leaves = [t for p in params['example'] for t in _leaves(p)]
  accum = [torch.full_like(t, 0.1) for t in leaves]
  g = torch.Generator().manual_seed(2)
  batches = []
  for step in range(3):
    x = torch.randn(b, n, sum(dims), generator=g)
    y = torch.randint(0, 5, (b, n), generator=g).float()
    y[:, -3:] = -1.0
    batches.append((x, y))
    got = float(trainer.train_step(x.cuda(), y.cuda()))
    for t in leaves:
      t.grad = None
    ol = oloss(y.double(), _oracle_logits(params, x, y, dims))
    ol.backward()
    with torch.no_grad():
      for t, a in zip(leaves, accum):
        a.add_(t.grad * t.grad)
        t.sub_(0.05 * t.grad / (a.sqrt() + 1e-7))
    assert got == pytest.approx(float(ol.detach()), rel=2e-4, abs=1e-6)
  want = torch.cat([_pack(p) for p in params['example']])
  assert _rel(gam.flat.detach(), want) <= 2e-3
  # pipeline.fit: 4 steps straight == 2 steps, checkpoint, resume for 2 more
  def fresh():
    gm, _ = _make(tfr, dims, [16, 8], act='relu', bn=True, seed=11)
    return tfr.train.GAMRankingTrainer(gm, loss, dims, optimizer='adagrad', learning_rate=0.05)
  data = batches + batches[:1]
  t1 = fresh()
  tfr.pipeline.fit(t1, iter(data), 4, log_fn=lambda *_: None)
  t2 = fresh()
  tfr.pipeline.fit(t2, iter(data), 2, checkpoint_dir=str(tmp_path), log_fn=lambda *_: None)
  t3 = fresh()
  tfr.pipeline.fit(t3, iter(data[2:]), 4, checkpoint_dir=str(tmp_path), log_fn=lambda *_: None)
  assert torch.equal(t3.tower.flat.detach(), t1.tower.flat.detach())
  assert torch.equal(t3.tower.bn_state, t1.tower.bn_state)
