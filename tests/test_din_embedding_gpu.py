"""The DIN's input gradient (tfr_din_input_grad, csrc/din.cu, K11) and
DINEmbeddingRankingTrainer: pooled token features -> DocumentInteractionAttention -> tower, the
model of the reference's ANTIQUE example with its document interaction network.

The C entry is checked against fp64 autograd of oracle/din.forward with respect to x; the
trainer against the fp64 composition oracle/embedding.pool -> ConcatFeatures ->
oracle/din.forward -> tower -> RestoreList -> ApproxNDCG, with every dropout / noise draw
replayed.  The argument checks at the top need no GPU.
"""
import ctypes
import os
import subprocess
import sys

import pytest
import torch

from oracle import din as odin
from oracle import embedding as oemb
from oracle import keras_losses as oracle_losses
from oracle import scorer as oracle_scorer
from oracle import utils as oracle_utils

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ANTIQUE = os.path.join(ROOT, 'tests', 'golden', 'antique')
gpu = pytest.mark.gpu


# ---- argument checks (no GPU) -------------------------------------------------------------
def _lib():
  import __graft_entry__ as g
  g.build()
  from ranking_b200 import _C
  return _C


def _cfg(_C, d=8, h=4, heads=1, layers=1):
  cfg = _C.DinCfg()
  cfg.input_dim, cfg.head_size, cfg.num_heads, cfg.num_layers = d, h, heads, layers
  cfg.dropout, cfg.input_noise_stddev, cfg.training, cfg.seed = 0.0, 0.0, 1, 0
  return cfg


def test_input_grad_argument_errors_without_gpu():
  """Every bad argument gives status 1 and a message before any CUDA call (the pointers are
  never dereferenced)."""
  _C = _lib()
  fake = ctypes.c_void_p(1 << 20)
  good = _cfg(_C)
  bad_cfgs = [_cfg(_C, d=6), _cfg(_C, h=6), _cfg(_C, h=132), _cfg(_C, heads=0),
              _cfg(_C, h=128, heads=5), _cfg(_C, layers=0), _cfg(_C, layers=9)]
  cases = [(ctypes.byref(c), 2, 3, fake, fake, 0, 4, fake, 4, 0) for c in bad_cfgs]
  cases += [
      (None, 2, 3, fake, fake, 0, 8, fake, 8, 0),                # NULL cfg
      (ctypes.byref(good), 2, 3, None, fake, 0, 8, fake, 8, 0),  # NULL params
      (ctypes.byref(good), 2, 3, fake, None, 0, 8, fake, 8, 0),  # NULL workspace
      (ctypes.byref(good), 2, 3, fake, fake, 0, 8, None, 8, 0),  # NULL dX
      (ctypes.byref(good), 2, 3, fake, fake, -1, 4, fake, 8, 0),  # window starts before 0
      (ctypes.byref(good), 2, 3, fake, fake, 5, 4, fake, 8, 0),  # window ends past D
      (ctypes.byref(good), 2, 3, fake, fake, 0, 0, fake, 8, 0),  # empty window
      (ctypes.byref(good), 2, 3, fake, fake, 2, 5, fake, 4, 0),  # ldx < ncols
      (ctypes.byref(good), 2, 3, fake, fake, 0, 8, fake, 8, 2),  # accumulate not 0 / 1
      (ctypes.byref(good), 2, 3, fake, fake, 0, 8, fake, 8, -1),
      (ctypes.byref(good), 2, 1025, fake, fake, 0, 8, fake, 8, 0),  # list too long
      (ctypes.byref(good), -1, 3, fake, fake, 0, 8, fake, 8, 0),    # negative batch
  ]
  for i, args in enumerate(cases):
    rc = _C.lib.tfr_din_input_grad(*args, None)
    assert rc == 1, (i, rc)
    assert _C.last_error(), i


def test_binding_lists_input_grad():
  _C = _lib()
  assert 'tfr_din_input_grad' in _C.EXPORTED_SYMBOLS
  assert hasattr(_C.lib, 'tfr_din_input_grad')


# ---- tfr_din_input_grad through the C ABI -------------------------------------------------
def _mask(b, n, gen):
  """Ragged validity: a full list, an all-padded list, a single-valid-item list, random."""
  m = torch.rand(b, n, generator=gen) < 0.6
  m[0] = True
  if b > 1:
    m[1] = False
  if b > 2:
    m[2] = False
    m[2, n // 2] = True
  return m


def _make_din(b, n, d, h, heads, nl, seed, dropout=0.0, noise=None):
  """Inputs and a DIN whose biases / LayerNorm parameters are non-trivial, so that no
  LayerNorm row has a near-zero variance (see tests/test_din_gpu.py)."""
  import ranking_b200 as tfr
  gen = torch.Generator().manual_seed(seed)
  x = torch.randn(b, n, d, generator=gen)
  din = tfr.keras.layers.DocumentInteractionAttention(heads, h, nl, dropout=dropout,
                                                      input_noise_stddev=noise, seed=seed)
  din.build(d)
  with torch.no_grad():
    p = odin.unflatten(din.flat.data, d, h, heads, nl)
    for name, t in p.items():
      if name.startswith('b'):
        t.copy_(torch.randn(t.shape, generator=gen) * 0.2)
      if name.startswith('gamma'):
        t.copy_(1.0 + torch.randn(t.shape, generator=gen) * 0.2)
  return x, _mask(b, n, gen), din


class _Abi(object):
  """tfr_din_fwd + tfr_din_bwd on one workspace, then windows of tfr_din_input_grad."""

  def __init__(self, din, x, mask, training):
    from ranking_b200 import _C
    self._C = _C
    self.din = din
    self.b, self.n, self.d = x.shape
    self.x = x.cuda().contiguous()
    self.m8 = mask.to(torch.uint8).cuda().contiguous()
    self.cfg = din._run_cfg(training=training)
    self.ws = din._new_workspace(self.b, self.n)

  def fwd_bwd(self, dout):
    _C, din = self._C, self.din
    m = self.b * self.n
    out = torch.empty(m, din.head_size, device='cuda')
    grads = torch.empty_like(din.flat.data)
    _C.check(_C.lib.tfr_din_fwd(_C.ptr(self.x), _C.ptr(self.m8), self.b, self.n,
                                ctypes.byref(self.cfg), _C.ptr(din.flat.data), _C.ptr(self.ws),
                                _C.ptr(out), din.head_size, _C.stream()))
    _C.check(_C.lib.tfr_din_bwd(_C.ptr(self.x), _C.ptr(self.m8), self.b, self.n,
                                ctypes.byref(self.cfg), _C.ptr(din.flat.data),
                                _C.ptr(dout.cuda().contiguous()), din.head_size, _C.ptr(self.ws),
                                _C.ptr(grads), _C.stream()))
    return out, grads

  def input_grad(self, col0, ncols, dx, ldx, accumulate=0, offset=0):
    _C = self._C
    _C.check(_C.lib.tfr_din_input_grad(ctypes.byref(self.cfg), self.b, self.n,
                                       _C.ptr(self.din.flat.data), _C.ptr(self.ws), col0, ncols,
                                       ctypes.c_void_p(dx.data_ptr() + 4 * offset), ldx,
                                       accumulate, _C.stream()))
    return dx


def _oracle_dx(din, x, mask, dout, cfg):
  """fp64 d (sum dout * din(x)) / d x with the call's dropout / noise draws replayed."""
  b, n, _ = x.shape
  keeps = noise = None
  if cfg.training and din.dropout > 0:
    keeps = odin.keep_masks(cfg.seed, b, n, din.num_heads, din.head_size, din.num_layers,
                            din.dropout)
  if cfg.training and din.input_noise_stddev:
    noise = odin.noise(cfg.seed, b, n, din.head_size, din.input_noise_stddev)
  xd = x.double().requires_grad_()
  out = odin.forward(xd, mask, din.flat.detach().cpu().double(), din.num_heads, din.head_size,
                     din.num_layers, rate=din.dropout, keeps=keeps, noise_add=noise)
  (out * dout.double().reshape(out.shape)).sum().backward()
  return out.detach(), xd.grad.reshape(b * n, -1)


def _rel_l2(a, b):
  return float((a - b).norm() / max(float(b.norm()), 1e-30))


@gpu
@pytest.mark.parametrize('d,h,heads,nl,training', [
    (4, 4, 1, 1, False), (40, 64, 2, 2, True), (136, 100, 3, 1, False),
    (260, 128, 4, 2, True), (40, 128, 1, 1, True), (136, 64, 2, 2, False),
    (260, 4, 1, 2, True), (4, 100, 2, 1, True), (40, 16, 4, 1, False)])
def test_input_gradient_against_autograd(d, h, heads, nl, training):
  b, n = 4, 29
  x, mask, din = _make_din(b, n, d, h, heads, nl, seed=d + h + heads,
                           dropout=0.2 if training else 0.0, noise=0.1 if training else None)
  abi = _Abi(din, x, mask, training)
  dout = torch.randn(b * n, h, generator=torch.Generator().manual_seed(7))
  out, _ = abi.fwd_bwd(dout)
  want_out, want = _oracle_dx(din, x, mask, dout, abi.cfg)
  assert _rel_l2(out.cpu().double(), want_out.reshape(b * n, h)) < 1e-5
  got = abi.input_grad(0, d, torch.full((b * n, d), 5.0, device='cuda'), d)
  torch.cuda.synchronize()
  assert _rel_l2(got.cpu().double(), want) < 5e-5


@gpu
@pytest.mark.parametrize('training', [False, True])
def test_windows_accumulate_and_determinism(training):
  b, n, d, h, e = 5, 33, 40, 32, 20
  x, mask, din = _make_din(b, n, d, h, 2, 2, seed=3, dropout=0.3 if training else 0.0,
                           noise=0.1 if training else None)
  abi = _Abi(din, x, mask, training)
  m = b * n
  dout = torch.randn(m, h, generator=torch.Generator().manual_seed(1))
  _, g_before = abi.fwd_bwd(dout)
  _, want = _oracle_dx(din, x, mask, dout, abi.cfg)
  # full window, twice: identical bits
  full = abi.input_grad(0, d, torch.empty(m, d, device='cuda'), d)
  again = abi.input_grad(0, d, torch.empty(m, d, device='cuda'), d)
  assert torch.equal(full, again)
  assert _rel_l2(full.cpu().double(), want) < 5e-5
  # [0, E)
  first = abi.input_grad(0, e, torch.empty(m, e, device='cuda'), e)
  assert _rel_l2(first.cpu().double(), want[:, :e]) < 5e-5
  # an interior window, col0 not a multiple of 4, into a wider buffer: columns past ncols and
  # before the offset stay as they were
  col0, nc, ldx, off = 6, 21, 29, 3
  buf = torch.full((m, ldx), 7.0, device='cuda')
  abi.input_grad(col0, nc, buf, ldx, offset=off)
  assert bool((buf[:, :off] == 7.0).all()) and bool((buf[:, off + nc:] == 7.0).all())
  assert _rel_l2(buf[:, off:off + nc].cpu().double(), want[:, col0:col0 + nc]) < 5e-5
  # accumulate = 1 is exactly prefill + (accumulate = 0 result)
  gen = torch.Generator().manual_seed(4)
  prefill = torch.randn(m, ldx, generator=gen).cuda()
  g0 = abi.input_grad(col0, nc, torch.zeros(m, ldx, device='cuda'), ldx, offset=off)
  acc = abi.input_grad(col0, nc, prefill.clone(), ldx, accumulate=1, offset=off)
  want_acc = prefill.clone()
  want_acc[:, off:off + nc] = prefill[:, off:off + nc] + g0[:, off:off + nc]
  assert torch.equal(acc, want_acc)
  # both sides of a split, accumulated in either order, equal one full accumulate
  p2 = torch.randn(m, d, generator=gen).cuda()
  a = abi.input_grad(0, d, p2.clone(), d, accumulate=1)
  b1 = abi.input_grad(17, d - 17, p2.clone(), d, accumulate=1, offset=17)
  b1 = abi.input_grad(0, 17, b1, d, accumulate=1)
  assert torch.equal(a, b1)
  # the input gradient neither reads nor disturbs the parameter gradients
  _, g_after = abi.fwd_bwd(dout)
  assert torch.equal(g_before, g_after)
  torch.cuda.synchronize()


@gpu
def test_padded_rows_get_zero_gradient():
  """A padded row of a list that has a valid item attends to the valid items but no row
  attends to it, so with a zero dout its input gradient is exactly zero."""
  b, n, d, h = 6, 40, 24, 16
  x, mask, din = _make_din(b, n, d, h, 2, 2, seed=9, dropout=0.2, noise=0.1)
  abi = _Abi(din, x, mask, True)
  dout = torch.randn(b, n, h, generator=torch.Generator().manual_seed(2))
  dout[~mask] = 0.0
  abi.fwd_bwd(dout.reshape(b * n, h))
  dx = abi.input_grad(0, d, torch.full((b * n, d), 3.0, device='cuda'), d).cpu().view(b, n, d)
  pad = (~mask) & mask.any(1, keepdim=True)
  assert int(pad.sum()) > 0
  assert bool((dx[pad] == 0).all())
  assert float(dx[mask].abs().max()) > 0


# ---- DINEmbeddingRankingTrainer -------------------------------------------------------------
V, E, E2, D, T, T2 = 60, 8, 4, 8, 12, 8


def _ids(r, t, v, gen, fill=0.3):
  ids = torch.randint(0, v, (r, t), generator=gen, dtype=torch.int32)
  ids[torch.rand(r, t, generator=gen) < fill] = -1
  ids[::5] = -1
  return ids


def _trainer(bn=False, dropout=0.0, din_feature='document_interaction_embedding', h=16,
             heads=2, nl=1, seed=3, lr=0.05):
  """Context features query (shared, E) and qlen (extra, E2); example features anchor (extra)
  and document_tokens (shared).  With the default din_feature the DIN block lands between
  anchor and document_tokens."""
  import ranking_b200 as tfr
  layers = tfr.keras.layers
  shared = layers.TokenEmbedding(V, E, combiner='mean', seed=seed)
  extra = layers.TokenEmbedding(V // 2, E2, combiner='sqrtn', seed=seed + 1)
  din = layers.DocumentInteractionAttention(heads, h, nl, dropout=dropout, seed=seed + 2)
  d_din = D + 2 * E + 2 * E2
  tower = layers.create_tower([32, 16], 1, activation='relu', use_batch_norm=bn,
                              dropout=dropout, input_dim=d_din + h, seed=seed + 3,
                              precision='tf32x3')
  feats = {'context': {'query': 'shared', 'qlen': 'extra'},
           'example': {'document_tokens': 'shared', 'anchor': 'extra'}}
  tr = tfr.train.DINEmbeddingRankingTrainer(
      {'shared': shared, 'extra': extra}, feats, din, tower,
      tfr.keras.losses.get('approx_ndcg_loss'), din_feature=din_feature, optimizer='adagrad',
      learning_rate=lr)
  with torch.no_grad():   # non-trivial DIN biases / LayerNorm parameters (see _make_din)
    gen = torch.Generator().manual_seed(seed)
    p = odin.unflatten(din.flat.data, d_din, h, heads, nl)
    for name, t in p.items():
      if name.startswith('b'):
        t.copy_(torch.randn(t.shape, generator=gen) * 0.2)
      if name.startswith('gamma'):
        t.copy_(1.0 + torch.randn(t.shape, generator=gen) * 0.2)
  return tr, shared, extra, din, tower


def _batch(gen, b, n):
  x = torch.randn(b, n, D, generator=gen)
  y = torch.randint(0, 5, (b, n), generator=gen).float()
  y[torch.rand(b, n, generator=gen) < 0.3] = -1.0
  y[:, 0] = torch.randint(1, 5, (b,), generator=gen).float()   # a valid item per list
  y[1, 1:] = -1.0
  tokens = {'context': {'query': _ids(b, 5, V, gen), 'qlen': _ids(b, 3, V // 2, gen)},
            'example': {'document_tokens': _ids(b * n, T, V, gen).reshape(b, n, T),
                        'anchor': _ids(b * n, T2, V // 2, gen).reshape(b, n, T2)}}
  for f in tokens['example'].values():
    f[y < 0] = -1                              # padded items have empty bags
  return x, y, tokens


def _seeds(din, tower):
  """The DIN's and the tower's seeds of the trainer's next training step."""
  draws = din.dropout > 0 or din.input_noise_stddev
  dseed = (din._base << 32) | ((din._calls + (1 if draws else 0)) & 0xFFFFFFFF)
  tseed = (tower._dropout_base << 32) | ((tower._dropout_calls + 1) & 0xFFFFFFFF)
  return dseed, tseed


def _oracle_step(tr, x, y, tokens, flat, din_input_grad=True):
  """fp64 loss and flat gradient of the composition, with the next step's draws replayed.
  With BN the dense rows and the example id rows are circularly padded before the DIN.
  din_input_grad=False drops the DIN's input gradient (its input is detached)."""
  b, n, d = x.shape
  mask = y >= 0
  flat = flat.clone().requires_grad_()
  sc, tower, din = tr.tower, tr.mlp, tr.din
  h = din.head_size
  dseed, tseed = _seeds(din, tower)
  xd = x.double()
  ids = {k: v.long() for kind in tokens.values() for k, v in kind.items()}
  if tower.use_batch_norm:
    idx, _ = oracle_utils.padded_nd_indices(mask)
    xd = torch.gather(xd, 1, idx.unsqueeze(-1).expand(-1, -1, d))
    for name in tokens['example']:
      t = ids[name].shape[-1]
      ids[name] = torch.gather(ids[name], 1, idx.unsqueeze(-1).expand(-1, -1, t))
  cols = [xd.reshape(b * n, d)]
  for kind, name, ti in tr.features:
    emb = tr.embeddings[ti]
    off = sc.table_offsets[ti]
    table = flat[off:off + emb.flat.numel()].view(emb.vocab_size, emb.embedding_dim)
    pooled = oemb.pool(ids[name], table, emb.combiner)
    if kind == 'context':
      pooled = pooled.unsqueeze(1).expand(-1, n, -1)
    cols.append(pooled.reshape(b * n, -1))
  din_in = torch.cat(cols, 1)                                    # ConcatFeatures
  keeps = None
  if din.dropout > 0:
    keeps = odin.keep_masks(dseed, b, n, din.num_heads, h, din.num_layers, din.dropout)
  src = din_in if din_input_grad else din_in.detach()
  emb_out = odin.forward(src.reshape(b, n, -1), mask, flat[sc.n_tables:sc.tower_offset],
                         din.num_heads, h, din.num_layers, rate=din.dropout, keeps=keeps)
  s = tr.split
  hcur = torch.cat([din_in[:, :s], emb_out.reshape(b * n, h), din_in[:, s:]], 1)
  off, dims = sc.tower_offset, tower.dims
  for i in range(len(dims) - 1):
    w = flat[off:off + dims[i] * dims[i + 1]].reshape(dims[i], dims[i + 1])
    off += dims[i] * dims[i + 1]
    hcur = hcur @ w + flat[off:off + dims[i + 1]]
    off += dims[i + 1]
    if i + 2 < len(dims):
      if tower.use_batch_norm:
        g0, b0, _ = tower.bn_offsets[i]
        g0, b0 = sc.tower_offset + g0, sc.tower_offset + b0
        mean = hcur.mean(0)
        var = ((hcur - mean) ** 2).mean(0)
        hcur = (hcur - mean) / torch.sqrt(var + 1e-3) * flat[g0:g0 + dims[i + 1]] + \
            flat[b0:b0 + dims[i + 1]]
      hcur = torch.relu(hcur)
      if tower.dropout > 0:
        keep = ~(odin.uniform(tseed, i + 1, b * n * dims[i + 1]) < tower.dropout)
        hcur = hcur * torch.from_numpy(keep).reshape(b * n, -1) / (1.0 - tower.dropout)
  logits = oracle_scorer.restore_list(hcur, mask)
  loss = oracle_losses.ApproxNDCGLoss()(y.double(), logits)
  loss.backward()
  return loss.item(), flat.grad


@gpu
def test_trainer_layout_and_flat_views():
  tr, shared, extra, din, tower = _trainer()
  assert tr.features == [('context', 'qlen', 0), ('context', 'query', 1),
                         ('example', 'anchor', 0), ('example', 'document_tokens', 1)]
  assert din.input_dim == D + 2 * E + 2 * E2 and tr.dense_dim == D
  # [x | qlen | query | anchor | DIN | document_tokens]
  assert tr.split == D + E2 + E + E2
  base = tr.tower.flat.data_ptr()
  assert extra.flat.data_ptr() == base
  assert shared.flat.data_ptr() == base + 4 * extra.flat.numel()
  assert din.flat.data_ptr() == base + 4 * tr.tower.n_tables
  assert tower.flat.data_ptr() == base + 4 * (tr.tower.n_tables + din.flat.numel())
  assert tr.tower.flat.numel() == (shared.flat.numel() + extra.flat.numel() +
                                   din.flat.numel() + tower.flat.numel())


@gpu
@pytest.mark.parametrize('bn', [False, True])
def test_trainer_one_step_against_composition(bn):
  """Without BN / dropout to 5e-5 in L2; with hidden BN, tower dropout, DIN dropout and
  circular padding to 1e-3 (the tower's BN / dropout bar).  The tables alone meet the same
  bar, which the composition without the DIN's input gradient misses by more than 1e-2."""
  b, n = 6, 16
  tr, shared, extra, din, tower = _trainer(bn=bn, dropout=0.2 if bn else 0.0)
  x, y, tokens = _batch(torch.Generator().manual_seed(5), b, n)
  flat = tr.tower.flat.detach().cpu().double()
  want_loss, g = _oracle_step(tr, x, y, tokens, flat)
  _, g_nodin = _oracle_step(tr, x, y, tokens, flat, din_input_grad=False)
  got = float(tr.train_step(x.cuda(), y.cuda(), tokens=tokens))
  torch.cuda.synchronize()
  bar = 1e-3 if bn else 5e-5
  assert abs(got - want_loss) <= 1e-5 * max(1.0, abs(want_loss)), (got, want_loss)
  assert _rel_l2(tr.grads.cpu().double(), g) < bar
  nt = tr.tower.n_tables
  assert _rel_l2(tr.grads[:nt].cpu().double(), g[:nt]) < bar
  assert _rel_l2(g_nodin[:nt], g[:nt]) > 1e-2
  tr.check_ids()


@gpu
@pytest.mark.parametrize('din_feature', ['document_interaction_embedding', 'zz_interaction'])
def test_trainer_three_adagrad_steps(din_feature):
  """Three steps replayed in fp64.  'zz_interaction' sorts after every example feature: the
  DIN block ends the tower input and only one input-gradient window is taken."""
  b, n = 5, 12
  tr, shared, extra, din, tower = _trainer(din_feature=din_feature, h=8, heads=1, nl=2,
                                           seed=8)
  if din_feature.startswith('zz'):
    assert tr.split == din.input_dim
  gen = torch.Generator().manual_seed(13)
  flat = tr.tower.flat.detach().cpu().double()
  accum = torch.full_like(flat, 0.1)
  for step in range(3):
    x, y, tokens = _batch(gen, b, n)
    want_loss, g = _oracle_step(tr, x, y, tokens, flat)
    got = float(tr.train_step(x.cuda(), y.cuda(), tokens=tokens))
    torch.cuda.synchronize()
    assert abs(got - want_loss) <= 1e-5 * max(1.0, abs(want_loss)), (step, got, want_loss)
    assert _rel_l2(tr.grads.cpu().double(), g) < 5e-5, step
    nt = tr.tower.n_tables
    assert _rel_l2(tr.grads[:nt].cpu().double(), g[:nt]) < 5e-5, step
    accum += g ** 2
    flat = flat - 0.05 * g / (accum.sqrt() + 1e-7)
    assert float((tr.tower.flat.detach().cpu().double() - flat).abs().max()) < 1e-5, step


@gpu
def test_trainer_rejects_bad_configurations():
  import ranking_b200 as tfr
  layers = tfr.keras.layers
  loss = tfr.keras.losses.get('approx_ndcg_loss')
  feats = {'context': {'query': 't'}, 'example': {'doc': 't'}}

  def make(input_dim, din_built=None, din_feature='document_interaction_embedding', **kw):
    emb = layers.TokenEmbedding(10, 4, seed=0)
    din = layers.DocumentInteractionAttention(1, 8, 1, dropout=0.0, seed=1)
    if din_built is not None:
      din.build(din_built)
    kw.setdefault('precision', 'tf32x3')
    tower = layers.create_tower([8], 1, use_batch_norm=False, dropout=0, input_dim=input_dim,
                                seed=1, **kw)
    return tfr.train.DINEmbeddingRankingTrainer({'t': emb}, feats, din, tower, loss,
                                                din_feature=din_feature)

  make(16)      # D_din = 8 = the two features: accepted
  with pytest.raises(ValueError):
    make(20, din_built=8)                  # tower input_dim != D_din + h
  with pytest.raises(ValueError):
    make(18)                               # D_din = 10, not a multiple of 4
  with pytest.raises(ValueError):
    make(12)                               # D_din = 4 < the features' 8 columns
  for name in ('query', 'doc'):
    with pytest.raises(ValueError):
      make(16, din_feature=name)           # collides with a token feature
  for kw in [dict(precision='fp32'), dict(input_batch_norm=True), dict(precision='bf16')]:
    with pytest.raises(ValueError):
      make(16, **kw)


# ---- the ANTIQUE fixture ------------------------------------------------------------------
@gpu
def test_fixture_trains_through_pipeline_fit(tmp_path):
  import ranking_b200 as tfr
  data, layers = tfr.data, tfr.keras.layers
  vocab = data.Vocabulary.from_file(os.path.join(ANTIQUE, 'vocab.txt'))
  spec = {'context': {'query_tokens': (8, vocab)}, 'example': {'document_tokens': (8, vocab)}}
  path = os.path.join(ANTIQUE, 'train_elwc.tfrecord')

  def batches():
    return data.elwc_batches(path, 5, 50, None, {'relevance': (1, -1)}, 'relevance',
                             token_feature_spec=spec)

  emb = layers.TokenEmbedding(vocab.num_ids, 20, seed=1)
  din = layers.DocumentInteractionAttention(1, 16, 1, dropout=0.5, seed=3)
  tower = layers.create_tower([16, 8], 1, activation='relu', use_batch_norm=True, dropout=0.5,
                              input_dim=56, seed=2, precision='tf32x3')
  tr = tfr.train.DINEmbeddingRankingTrainer(
      {'shared': emb}, {'context': {'query_tokens': 'shared'},
                        'example': {'document_tokens': 'shared'}}, din, tower,
      tfr.keras.losses.get('approx_ndcg_loss'), optimizer='adagrad', learning_rate=0.05)
  # [query_tokens | document_interaction_embedding | document_tokens]: 'document_i' < 'document_t'
  assert tr.split == 20
  table0, din0 = emb.flat.detach().clone(), din.flat.detach().clone()
  it = (bt for _ in range(10) for bt in batches())
  step, last = tfr.pipeline.fit(tr, it, 12, checkpoint_dir=str(tmp_path), log_fn=lambda m: None)
  assert step == 12 and last == last and -1.0 <= last <= 0.0
  assert not torch.equal(table0, emb.flat.detach())
  assert not torch.equal(din0, din.flat.detach())
  tr.check_ids()
  tower.eval()
  din.eval()
  res = tfr.pipeline.evaluate(tr, list(batches()))
  assert res and all(float(v) == float(v) for v in res.values())
  assert os.path.exists(os.path.join(str(tmp_path), 'ckpt.pt'))


@gpu
def test_antique_example_with_document_interaction():
  data = os.path.join(ANTIQUE, 'train_elwc.tfrecord')
  out = subprocess.run(
      [sys.executable, os.path.join(ROOT, 'examples', 'antique_train.py'),
       '--train_path', data, '--eval_path', data,
       '--vocab_file', os.path.join(ANTIQUE, 'vocab.txt'),
       '--use_document_interaction', '1', '--num_train_steps', '5'],
      capture_output=True, text=True, timeout=600, cwd=ROOT)
  assert out.returncode == 0, out.stdout + out.stderr
  assert 'step 5 loss' in out.stdout and 'ndcg' in out.stdout.lower(), out.stdout
