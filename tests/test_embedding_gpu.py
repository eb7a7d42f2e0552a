"""Pooled embedding bags (csrc/embedding.cu, K12), TokenEmbedding and EmbeddingRankingTrainer
against the fp64 oracle (oracle/embedding.py + oracle/scorer.py + the oracle loss)."""
import os
import subprocess
import sys

import pytest
import torch

import ranking_b200 as tfr
from oracle import embedding as oemb
from oracle import keras_losses as oracle_losses
from oracle import scorer as oracle_scorer
from oracle import utils as oracle_utils
from ranking_b200 import _C

pytestmark = pytest.mark.gpu
layers = tfr.keras.layers
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ANTIQUE = os.path.join(ROOT, 'tests', 'golden', 'antique')
COMBINERS = {'sum': 0, 'mean': 1, 'sqrtn': 2}


def _ids(r, t, v, gen, fill=0.3):
  """Bags with duplicates, -1 slots (not only at the tail) and empty bags."""
  ids = torch.randint(0, v, (r, t), generator=gen, dtype=torch.int32)
  ids[torch.rand(r, t, generator=gen) < fill] = -1
  ids[::5] = -1                      # empty bags
  if t > 2:
    ids[1::7, 1] = ids[1::7, 0]      # duplicates
  return ids


def _fwd(ids, table, combiner, rpb=1, ldo=None, bad=None):
  r, t = ids.shape
  v, e = table.shape
  ldo = ldo or e
  out = torch.full((r * rpb, ldo), 7.0, dtype=torch.float32, device='cuda')
  _C.check(_C.lib.tfr_embedding_fwd(_C.ptr(ids), r, t, _C.ptr(table), v, e,
                                    COMBINERS[combiner], rpb, _C.ptr(out), ldo, _C.ptr(bad),
                                    _C.stream()))
  return out


def _bwd(ids, dout, v, e, combiner, rpb=1, dtable=None, accumulate=0, bad=None):
  r, t = ids.shape
  ws = torch.empty(_C.lib.tfr_embedding_workspace_bytes(r, t, v, e), dtype=torch.uint8,
                   device='cuda')
  if dtable is None:
    dtable = torch.full((v, e), 3.0, dtype=torch.float32, device='cuda')
  _C.check(_C.lib.tfr_embedding_bwd(_C.ptr(ids), r, t, _C.ptr(dout), dout.shape[1], rpb, v, e,
                                    COMBINERS[combiner], accumulate, _C.ptr(ws), _C.ptr(dtable),
                                    _C.ptr(bad), _C.stream()))
  return dtable


def _oracle_grad(ids, table, dout, combiner, rpb=1):
  tb = table.detach().cpu().double().requires_grad_()
  pooled = oemb.pool(ids.cpu().long(), tb, combiner)
  rep = pooled.repeat_interleave(rpb, 0)
  (rep * dout.cpu().double()).sum().backward()
  return pooled.detach(), tb.grad


@pytest.mark.parametrize('combiner', ['mean', 'sum', 'sqrtn'])
@pytest.mark.parametrize('r,t,v,e,rpb', [(1, 1, 1, 1, 1), (300, 16, 50, 20, 1),
                                         (64, 128, 30522, 20, 1), (37, 7, 9, 33, 3),
                                         (16, 40, 70000, 64, 50)])
def test_forward_backward_against_oracle(combiner, r, t, v, e, rpb):
  gen = torch.Generator().manual_seed(r * 31 + t)
  ids = _ids(r, t, v, gen)
  table = torch.randn(v, e, generator=gen).cuda()
  ldo = e + 5
  out = _fwd(ids.cuda(), table, combiner, rpb, ldo)
  dout = torch.randn(r * rpb, e, generator=gen)
  want, want_g = _oracle_grad(ids, table, dout, combiner, rpb)
  got = out[:, :e].cpu().double().reshape(r, rpb, e)
  scale = max(float(want.abs().max()), 1e-30)
  assert float((got - want.unsqueeze(1)).abs().max()) <= 1e-6 * scale
  assert bool((out[:, e:] == 7.0).all())          # columns past E untouched
  dt = _bwd(ids.cuda(), dout.cuda(), v, e, combiner, rpb)
  gscale = max(float(want_g.abs().max()), 1e-30)
  assert float((dt.cpu().double() - want_g).abs().max()) <= 1e-5 * gscale
  # rows no id hit are written 0
  hit = torch.zeros(v, dtype=torch.bool)
  hit[ids[ids >= 0].long()] = True
  assert bool((dt.cpu()[~hit] == 0).all())


def test_skewed_batch_and_determinism():
  """One id in every slot of every bag (R * T = 256 K occurrences of id 7): the segment is
  split into chunks, and two identical calls give identical bits."""
  gen = torch.Generator().manual_seed(3)
  r, t, v, e = 2048, 128, 30522, 20
  ids = _ids(r, t, v, gen, fill=0.1)
  ids[:, ::2] = 7
  table = torch.randn(v, e, generator=gen).cuda()
  dout = torch.randn(r, e, generator=gen)
  _, want_g = _oracle_grad(ids, table, dout, 'mean')
  a = _bwd(ids.cuda(), dout.cuda(), v, e, 'mean')
  b = _bwd(ids.cuda(), dout.cuda(), v, e, 'mean')
  assert torch.equal(a, b)
  assert float((a.cpu().double() - want_g).abs().max()) <= 1e-5 * float(want_g.abs().max())
  ids[:] = 7
  a = _bwd(ids.cuda(), dout.cuda(), v, e, 'sum')
  b = _bwd(ids.cuda(), dout.cuda(), v, e, 'sum')
  assert torch.equal(a, b)
  want = dout.double().sum(0) * t
  assert float((a[7].cpu().double() - want).abs().max()) <= 1e-5 * float(want.abs().max())


def test_shared_table_accumulates():
  gen = torch.Generator().manual_seed(5)
  v, e = 40, 12
  q = _ids(8, 4, v, gen)
  d = _ids(8 * 6, 9, v, gen)
  table = torch.randn(v, e, generator=gen).cuda()
  gq = torch.randn(8 * 6, e, generator=gen)   # the query bag is repeated over 6 rows
  gd = torch.randn(8 * 6, e, generator=gen)
  _, wq = _oracle_grad(q, table, gq, 'mean', rpb=6)
  _, wd = _oracle_grad(d, table, gd, 'sqrtn')
  dt = _bwd(q.cuda(), gq.cuda(), v, e, 'mean', rpb=6)
  dt = _bwd(d.cuda(), gd.cuda(), v, e, 'sqrtn', dtable=dt, accumulate=1)
  want = wq + wd
  assert float((dt.cpu().double() - want).abs().max()) <= 1e-5 * float(want.abs().max())


def test_out_of_range_ids_are_skipped_and_counted():
  v, e = 10, 4
  ids = torch.tensor([[1, v, -2, 3], [-1, -1, -1, -1], [v + 100, -7, 2, 2]], dtype=torch.int32)
  table = torch.randn(v, e).cuda()
  bad = torch.zeros(1, dtype=torch.int32, device='cuda')
  out = _fwd(ids.cuda(), table, 'mean', bad=bad)
  assert int(bad) == 4
  clean = torch.where((ids >= -1) & (ids < v), ids, torch.full_like(ids, -1))
  want = oemb.pool(clean.long(), table.cpu().double(), 'mean')
  assert float((out.cpu().double() - want).abs().max()) <= 1e-6 * float(want.abs().max())
  bad.zero_()
  dout = torch.randn(3, e)
  dt = _bwd(ids.cuda(), dout.cuda(), v, e, 'mean', bad=bad)
  assert int(bad) == 4
  _, wg = _oracle_grad(clean, table, dout, 'mean')
  assert float((dt.cpu().double() - wg).abs().max()) <= 1e-5 * float(wg.abs().max())
  emb = layers.TokenEmbedding(v, e, seed=1)
  with pytest.raises(ValueError, match='outside'):
    emb(ids.cuda())
  with pytest.raises(ValueError):
    _C.check(_C.lib.tfr_embedding_fwd(None, 1, 1, None, v, e, 1, 1, None, e, None, None))


def test_token_embedding_layer_composes_with_tower():
  """TokenEmbedding -> Tower through torch autograd: the table gradient equals the fp64
  composition's."""
  gen = torch.Generator().manual_seed(8)
  v, e, b, t = 30, 8, 24, 6
  emb = layers.TokenEmbedding(v, e, combiner='mean', seed=4)
  assert float(emb.flat.detach().abs().max()) <= 0.05
  tower = layers.create_tower([16], 1, activation='relu', use_batch_norm=False, dropout=0,
                              input_dim=e, seed=2, precision='tf32x3')
  ids = _ids(b, t, v, gen)
  out = tower(emb(ids.cuda()))
  g = torch.randn(b, 1, generator=gen)
  (out * g.cuda()).sum().backward()
  table = emb.flat.detach().cpu().double().view(v, e).requires_grad_()
  p = {'dense_w': [tower.kernel(i).detach().cpu().double() for i in range(2)],
       'dense_b': [tower.bias(i).detach().cpu().double() for i in range(2)]}
  want = oracle_scorer.tower_forward(oemb.pool(ids.long(), table), p, activation='relu')
  (want * g.double()).sum().backward()
  assert float((out.detach().cpu().double() - want.detach()).abs().max()) <= 1e-5
  got = emb.flat.grad.cpu().double().view(v, e)
  err = (got - table.grad).norm() / table.grad.norm()
  assert float(err) < 5e-5


# ---- EmbeddingRankingTrainer ------------------------------------------------------------
def _trainer(bn, d, v=60, e=8, lr=0.05, seed=3, hidden=(32, 16)):
  shared = layers.TokenEmbedding(v, e, combiner='mean', seed=seed)
  extra = layers.TokenEmbedding(v // 2, 4, combiner='sqrtn', seed=seed + 1)
  tower = layers.create_tower(list(hidden), 1, activation='relu', use_batch_norm=bn, dropout=0,
                              input_dim=d + 2 * e + 4, seed=seed + 2, precision='tf32x3')
  feats = {'context': {'query': 'shared', 'qlen': 'extra'}, 'example': {'doc': 'shared'}}
  tr = tfr.train.EmbeddingRankingTrainer({'shared': shared, 'extra': extra}, feats, tower,
                                         tfr.keras.losses.get('approx_ndcg_loss'),
                                         optimizer='adagrad', learning_rate=lr)
  # query and doc share a table: the second one's backward accumulates
  return tr, shared, extra, tower


def _batch(gen, b, n, d, v=60):
  x = torch.randn(b, n, d, generator=gen)
  y = torch.randint(0, 5, (b, n), generator=gen).float()
  y[torch.rand(b, n, generator=gen) < 0.3] = -1.0
  y[:, 0] = torch.randint(1, 5, (b,), generator=gen).float()   # a valid item per list
  y[1, 1:] = -1.0
  tokens = {'context': {'query': _ids(b, 5, v, gen), 'qlen': _ids(b, 3, v // 2, gen)},
            'example': {'doc': _ids(b * n, 12, v, gen).reshape(b, n, 12)}}
  tokens['example']['doc'][y < 0] = -1       # padded items have empty bags
  return x, y, tokens


def _oracle_step(tr, x, y, tokens, flat):
  """fp64 loss and flat gradient of tower([x | query | qlen | doc]) -> RestoreList ->
  ApproxNDCG; with BN the dense rows and the doc id rows are circularly padded first."""
  b, n, d = x.shape
  mask = y >= 0
  flat = flat.clone().requires_grad_()
  sc, tower = tr.tower, tr.mlp
  xd = x.double()
  ids = {k: v.long() for kind in tokens.values() for k, v in kind.items()}
  if tower.use_batch_norm:
    idx, _ = oracle_utils.padded_nd_indices(mask)
    xd = torch.gather(xd, 1, idx.unsqueeze(-1).expand(-1, -1, d))
    ids['doc'] = torch.gather(ids['doc'], 1, idx.unsqueeze(-1).expand(-1, -1, 12))
  cols = [xd.reshape(b * n, d)]
  for kind, name, ti in tr.features:
    emb = tr.embeddings[ti]
    off = sc.table_offsets[ti]
    table = flat[off:off + emb.flat.numel()].view(emb.vocab_size, emb.embedding_dim)
    pooled = oemb.pool(ids[name], table, emb.combiner)
    if kind == 'context':
      pooled = pooled.unsqueeze(1).expand(-1, n, -1)
    cols.append(pooled.reshape(b * n, -1))
  h = torch.cat(cols, 1)
  off, dims = sc.n_tables, tower.dims
  for i in range(len(dims) - 1):
    w = flat[off:off + dims[i] * dims[i + 1]].reshape(dims[i], dims[i + 1])
    off += dims[i] * dims[i + 1]
    h = h @ w + flat[off:off + dims[i + 1]]
    off += dims[i + 1]
    if i + 2 < len(dims):
      if tower.use_batch_norm:
        g0, b0, _ = tower.bn_offsets[i]
        mean = h.mean(0)
        var = ((h - mean) ** 2).mean(0)
        h = (h - mean) / torch.sqrt(var + 1e-3) * flat[sc.n_tables + g0:sc.n_tables + g0 +
                                                      dims[i + 1]] + \
            flat[sc.n_tables + b0:sc.n_tables + b0 + dims[i + 1]]
      h = torch.relu(h)
  logits = oracle_scorer.restore_list(h, mask)
  loss = oracle_losses.ApproxNDCGLoss()(y.double(), logits)
  loss.backward()
  return loss.item(), flat.grad


def _rel_l2(a, b):
  return float((a - b).norm() / max(float(b.norm()), 1e-30))


@pytest.mark.parametrize('bn', [False, True])
def test_trainer_three_adagrad_steps(bn):
  b, n, d = 6, 16, 8
  tr, shared, extra, tower = _trainer(bn, d)
  assert tr.features == [('context', 'qlen', 0), ('context', 'query', 1),
                         ('example', 'doc', 1)]
  assert shared.flat.data_ptr() == tr.tower.flat.data_ptr() + 4 * extra.flat.numel()
  gen = torch.Generator().manual_seed(11)
  flat = tr.tower.flat.detach().cpu().double()
  accum = torch.full_like(flat, 0.1)
  for step in range(3):
    x, y, tokens = _batch(gen, b, n, d)
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
  tr.check_ids()


def test_trainer_rejects_unsupported_towers():
  emb = layers.TokenEmbedding(10, 4, seed=0)
  for kw in [dict(precision='fp32'), dict(input_batch_norm=True, precision='tf32x3'),
             dict(precision='bf16')]:
    tower = layers.create_tower([8], 1, use_batch_norm=False, dropout=0, input_dim=4, seed=1,
                                **kw)
    with pytest.raises(ValueError):
      tfr.train.EmbeddingRankingTrainer({'t': emb}, {'example': {'doc': 't'}}, tower,
                                        tfr.keras.losses.get('approx_ndcg_loss'))
  tower = layers.create_tower([8], 1, use_batch_norm=False, dropout=0, input_dim=4, seed=1,
                              precision='tf32x3')
  with pytest.raises(ValueError):
    tfr.train.EmbeddingRankingTrainer({'t': emb}, {'example': {'doc': 'missing'}}, tower,
                                      tfr.keras.losses.get('approx_ndcg_loss'))


def test_fixture_trains_through_pipeline_fit(tmp_path):
  """The ANTIQUE fixture: (x, y, tokens) batches of elwc_batches through pipeline.fit with a
  checkpoint, then evaluate."""
  data = tfr.data
  vocab = data.Vocabulary.from_file(os.path.join(ANTIQUE, 'vocab.txt'))
  spec = {'context': {'query_tokens': (8, vocab)}, 'example': {'document_tokens': (8, vocab)}}
  path = os.path.join(ANTIQUE, 'train_elwc.tfrecord')

  def batches():
    return data.elwc_batches(path, 5, 50, None, {'relevance': (1, -1)}, 'relevance',
                             token_feature_spec=spec)

  emb = layers.TokenEmbedding(vocab.num_ids, 20, seed=1)
  tower = layers.create_tower([16, 8], 1, activation='relu', use_batch_norm=True, dropout=0.5,
                              input_dim=40, seed=2, precision='tf32x3')
  tr = tfr.train.EmbeddingRankingTrainer(
      {'shared': emb}, {'context': {'query_tokens': 'shared'},
                        'example': {'document_tokens': 'shared'}}, tower,
      tfr.keras.losses.get('approx_ndcg_loss'), optimizer='adagrad', learning_rate=0.05)
  before = emb.flat.detach().clone()
  it = (bt for _ in range(10) for bt in batches())
  step, last = tfr.pipeline.fit(tr, it, 12, checkpoint_dir=str(tmp_path), log_fn=lambda m: None)
  assert step == 12 and last == last and -1.0 <= last <= 0.0
  assert not torch.equal(before, emb.flat.detach())
  tr.check_ids()
  tower.eval()
  res = tfr.pipeline.evaluate(tr, list(batches()))
  assert res and all(float(v) == float(v) for v in res.values())
  assert os.path.exists(os.path.join(str(tmp_path), 'ckpt.pt'))


def test_two_gpu_data_parallel_equals_single_gpu():
  if torch.cuda.device_count() < 2:
    pytest.skip('needs 2 GPUs')
  out = subprocess.run(
      [sys.executable, '-m', 'torch.distributed.run', '--nnodes=1', '--nproc-per-node', '2',
       '--master-addr', '127.0.0.1', '--master-port', '29613',
       os.path.join(ROOT, 'tools', 'embedding_dp_equivalence.py')],
      capture_output=True, text=True, timeout=300)
  assert out.returncode == 0, out.stdout + out.stderr
  assert 'DP_EQUIVALENCE_OK' in out.stdout, out.stdout + out.stderr
