"""Training-step throughput of EmbeddingRankingTrainer (csrc/embedding.cu + the scorer tower)
at the ANTIQUE example's shape scaled to a full batch: B = 1024 lists of N = 50 items, a
query bag of T = 16 tokens (context) and a document bag of T = 128 tokens per item, one shared
table of V = 30522 rows x E = 20 (mean combiner), a [256, 128, 64] ReLU tower on the 40 pooled
columns, ApproxNDCG, Adagrad 0.05.  Bag lengths are uniform in [1, T], ids uniform in [0, V),
20 % of the items padded (empty bags).

Prints one JSON line: lists/s and ms/step of EmbeddingRankingTrainer.train_step (CUDA events
after warm-up); a per-phase split (embedding forward, tower forward + loss + backward with the
input gradient, embedding backward, optimizer); algorithmic bytes from the shapes (ids,
gathered rows R*T*E*4, pooled writes, sort traffic); and lists/s of a batched PyTorch
formulation of the same model (nn.EmbeddingBag with padding_idx, Linear tower, TF32 off, the
same ApproxNDCG, autograd, torch.optim.Adagrad) in the same run.  Needs a CUDA device.
  python tools/embedding_step.py [--steps 30] [--warmup 5]
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

B, N, TQ, TD, V, E, HIDDEN, LR = 1024, 50, 16, 128, 30522, 20, [256, 128, 64], 0.05
HBM_BW = 3.35e12         # H100 SXM data sheet


def card():
  try:
    out = subprocess.check_output(
        ['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
         '--format=csv,noheader', '-i', str(torch.cuda.current_device())], text=True)
    name, power, clock = [s.strip() for s in out.strip().split('\n')[0].split(',')]
    return {'gpu': name, 'power_limit': power, 'max_sm_clock': clock}
  except (OSError, subprocess.CalledProcessError, ValueError):
    return {'gpu': torch.cuda.get_device_name(), 'power_limit': 'unknown'}


def bags(g, rows, t):
  ids = torch.randint(0, V, (rows, t), generator=g, dtype=torch.int32)
  lens = torch.randint(1, t + 1, (rows, 1), generator=g)
  ids[torch.arange(t).unsqueeze(0) >= lens] = -1
  return ids


def batch(seed):
  g = torch.Generator().manual_seed(seed)
  y = torch.randint(0, 5, (B, N), generator=g).float()
  y[torch.rand(B, N, generator=g) < 0.2] = -1.0
  y[:, 0] = 1.0
  q = bags(g, B, TQ)
  d = bags(g, B * N, TD).reshape(B, N, TD)
  d[y < 0] = -1
  x = torch.zeros(B, N, 0)
  return x.cuda(), y.cuda(), {'context': {'query_tokens': q.cuda()},
                              'example': {'document_tokens': d.cuda()}}


def timed(step, steps, warmup):
  for _ in range(warmup):
    step()
  torch.cuda.synchronize()
  t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  t0.record()
  for _ in range(steps):
    step()
  t1.record()
  torch.cuda.synchronize()
  return t0.elapsed_time(t1) / 1e3 / steps


def cuda_trainer():
  import ranking_b200 as tfr
  emb = tfr.keras.layers.TokenEmbedding(V, E, combiner='mean', seed=1)
  tower = tfr.keras.layers.create_tower(HIDDEN, 1, activation='relu', use_batch_norm=False,
                                        dropout=0, input_dim=2 * E, seed=2, precision='tf32x3')
  return tfr.train.EmbeddingRankingTrainer(
      {'shared': emb}, {'context': {'query_tokens': 'shared'},
                        'example': {'document_tokens': 'shared'}}, tower,
      tfr.keras.losses.get('approx_ndcg_loss'), optimizer='adagrad', learning_rate=LR)


def phases(tr, x, y, tokens, steps):
  """ms per phase of the fused step: the trainer's own calls, CUDA events between them."""
  names = ['embedding_fwd', 'tower', 'embedding_bwd', 'optimizer']
  acc = dict.fromkeys(names, 0.0)
  m8 = None
  for it in range(steps + 1):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(names) + 1)]
    cfg = ctypes.byref(tr.tower._run_cfg(training=True))
    tr._set_tokens(tokens, B, N)
    tr._circular_pad(x, y >= 0)
    # embedding forward alone: the trainer's _forward without the tower
    from ranking_b200 import _C
    ev[0].record()
    col = 0
    for k, (_, _, ti) in enumerate(tr.features):
      emb = tr.embeddings[ti]
      ids, r, t, rpb = tr._bags(k, B, N)
      _C.check(_C.lib.tfr_embedding_fwd(_C.ptr(ids), r, t, _C.ptr(emb.flat.data), V, E,
                                        emb._combiner, rpb,
                                        ctypes.c_void_p(tr.xe.data_ptr() + 4 * col),
                                        tr.mlp.input_dim, _C.ptr(tr.bad_ids), _C.stream()))
      col += E
    ev[1].record()
    st = _C.stream()
    mlp, g = tr.mlp, tr.grads
    _C.check(_C.lib.tfr_mlp_fwd(_C.ptr(tr.xe), B * N, cfg, _C.ptr(mlp.flat.data), None,
                                _C.ptr(tr.ws), _C.ptr(tr.scores), mlp._precision, st))
    tr.loss.fused_fwd_bwd(y, tr.scores, None, tr.dscores, tr.per_list, tr.total2)
    _C.check(_C.lib.tfr_mlp_bwd(_C.ptr(tr.xe), B * N, cfg, _C.ptr(mlp.flat.data),
                                _C.ptr(tr.dscores), None, _C.ptr(tr.ws),
                                ctypes.c_void_p(g.data_ptr() + 4 * tr.tower.n_tables),
                                mlp._precision, st))
    _C.check(_C.lib.tfr_mlp_input_grad(cfg, B * N, _C.ptr(mlp.flat.data), _C.ptr(tr.ws), 0,
                                       tr.emb_width, _C.ptr(tr.d_emb), tr.emb_width,
                                       mlp._precision, st))
    ev[2].record()
    col = 0
    for k, (_, _, ti) in enumerate(tr.features):
      emb = tr.embeddings[ti]
      ids, r, t, rpb = tr._bags(k, B, N)
      _C.check(_C.lib.tfr_embedding_bwd(
          _C.ptr(ids), r, t, ctypes.c_void_p(tr.d_emb.data_ptr() + 4 * col), tr.emb_width, rpb,
          V, E, emb._combiner, int(k > 0), _C.ptr(tr._emb_ws),
          ctypes.c_void_p(g.data_ptr() + 4 * tr.tower.table_offsets[ti]), None, st))
      col += E
    ev[3].record()
    tr._apply(g)
    ev[4].record()
    torch.cuda.synchronize()
    if it == 0:
      continue
    for i, n in enumerate(names):
      acc[n] += ev[i].elapsed_time(ev[i + 1]) / steps
  return {k: round(v, 3) for k, v in acc.items()}


def torch_step_fn(y, tokens):
  """What a PyTorch user would write: nn.EmbeddingBag (mean, -1 mapped to a padding row that
  the mean skips) for both features, a Linear tower, the same ApproxNDCG, autograd, Adagrad."""
  import ranking_b200 as tfr
  dev = y.device
  bag = torch.nn.EmbeddingBag(V + 1, E, mode='mean', padding_idx=V).to(dev)
  with torch.no_grad():
    bag.weight[:V].uniform_(-0.05, 0.05)
  dims = [2 * E] + HIDDEN + [1]
  lin = [torch.nn.Linear(dims[i], dims[i + 1]).to(dev) for i in range(len(dims) - 1)]
  params = list(bag.parameters()) + [p for l in lin for p in l.parameters()]
  opt = torch.optim.Adagrad(params, lr=LR, initial_accumulator_value=0.1, eps=1e-7)
  loss_obj = tfr.keras.losses.get('approx_ndcg_loss')
  mask = y >= 0
  q = tokens['context']['query_tokens'].long()
  d = tokens['example']['document_tokens'].long().reshape(B * N, TD)
  q = torch.where(q < 0, torch.full_like(q, V), q)
  d = torch.where(d < 0, torch.full_like(d, V), d)

  def step():
    qe = bag(q).unsqueeze(1).expand(B, N, E)
    de = bag(d).reshape(B, N, E)
    h = torch.cat([qe, de], -1).reshape(B * N, 2 * E)
    for i, l in enumerate(lin):
      h = l(h)
      if i + 1 < len(lin):
        h = torch.relu(h)
    logits = torch.where(mask, h.reshape(B, N), torch.full_like(y, -23.025850929940457))
    loss = loss_obj(y, logits)
    opt.zero_grad(set_to_none=True)
    loss.backward()
    opt.step()
  return step


def work():
  """Algorithmic bytes of the embedding side of one step (fwd + bwd), from the shapes."""
  rq, rd = B, B * N
  ids = 4 * (rq * TQ + rd * TD)
  gathered = 4 * E * (rq * TQ + rd * TD)                 # R * T * E * 4, both features
  pooled = 4 * E * 2 * B * N                             # pooled writes into the tower input
  # backward: ids read, per-bag gradient rows, two radix passes over (key, bag) pairs, the
  # segment sums re-read one gradient row per occurrence, table gradient written
  sort = 2 * (2 * 4 * 2) * (rq * TQ + rd * TD)
  seg = 4 * E * (rq * TQ + rd * TD) + 4 * V * E
  return {'ids_mb': round(ids / 1e6, 1), 'gathered_rows_mb': round(gathered / 1e6, 1),
          'pooled_writes_mb': round(pooled / 1e6, 1), 'sort_mb': round(sort / 1e6, 1),
          'segment_sum_mb': round(seg / 1e6, 1),
          'hbm_bound_ms': round((ids * 2 + gathered + pooled + sort + seg) / HBM_BW * 1e3, 3)}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=30)
  ap.add_argument('--warmup', type=int, default=5)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('embedding_step.py needs a CUDA device')
  torch.backends.cuda.matmul.allow_tf32 = False
  torch.backends.cudnn.allow_tf32 = False
  res = {'shape': {'B': B, 'N': N, 'T_query': TQ, 'T_document': TD, 'V': V, 'E': E,
                   'tower': HIDDEN}}
  res.update(card())
  x, y, tokens = batch(0)
  tr = cuda_trainer()
  sec = timed(lambda: tr.train_step(x, y, tokens=tokens), args.steps, args.warmup)
  res['cuda'] = {'lists_per_s': round(B / sec, 1), 'step_ms': round(sec * 1e3, 3),
                 'timed_steps': args.steps,
                 'phases_ms': phases(tr, x, y, tokens, max(20, args.steps))}
  res['algorithmic'] = work()
  del tr
  torch.cuda.empty_cache()
  step = torch_step_fn(y, tokens)
  ps = timed(step, max(20, args.steps), args.warmup)
  res['pytorch'] = {'lists_per_s': round(B / ps, 1), 'step_ms': round(ps * 1e3, 3)}
  print(json.dumps(res))


if __name__ == '__main__':
  main()
