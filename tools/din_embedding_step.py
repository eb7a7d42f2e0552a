"""Training-step throughput of DINEmbeddingRankingTrainer: the ANTIQUE example with its document
interaction network (examples/keras/antique_kpl_din.py, use_document_interaction=True) at the
shape of tools/embedding_step.py: B = 1024 lists of N = 50 items, a query bag of T = 16 tokens
(context) and a document bag of T = 128 tokens per item, one shared table of V = 30522 rows x
E = 20 (mean), a DocumentInteractionAttention over the 40 pooled columns (L = 1, H = 1,
h = 128, dropout 0), a [256, 128, 64] ReLU tower on [query | DIN | document], ApproxNDCG,
Adagrad 0.05.  Bag lengths are uniform in [1, T], 20 % of the items padded (empty bags).

Prints one JSON line: lists/s and ms/step of DINEmbeddingRankingTrainer.train_step (CUDA events
after warm-up); a per-phase split (embedding forward, DIN forward, tower forward + loss +
backward with the input gradient, DIN backward, DIN input gradient, embedding backward,
optimizer); the card; and lists/s of a batched PyTorch formulation of the same model
(nn.EmbeddingBag, tools/din_step.py's attention, Linear tower, TF32 off, the same ApproxNDCG,
autograd, torch.optim.Adagrad) in the same run.  Needs a CUDA device.
  python tools/din_embedding_step.py [--steps 30] [--warmup 5]
"""
import argparse
import ctypes
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import torch  # noqa: E402

from embedding_step import B, N, TQ, TD, V, E, HIDDEN, LR, batch, card, timed  # noqa: E402

L, H, HS = 1, 1, 128


def cuda_trainer():
  import ranking_b200 as tfr
  layers = tfr.keras.layers
  emb = layers.TokenEmbedding(V, E, combiner='mean', seed=1)
  din = layers.DocumentInteractionAttention(H, HS, L, dropout=0.0, seed=3)
  tower = layers.create_tower(HIDDEN, 1, activation='relu', use_batch_norm=False, dropout=0,
                              input_dim=2 * E + HS, seed=2, precision='tf32x3')
  return tfr.train.DINEmbeddingRankingTrainer(
      {'shared': emb}, {'context': {'query_tokens': 'shared'},
                        'example': {'document_tokens': 'shared'}}, din, tower,
      tfr.keras.losses.get('approx_ndcg_loss'), optimizer='adagrad', learning_rate=LR)


def phases(tr, x, y, tokens, steps):
  """ms per phase of the fused step: the trainer's own calls, CUDA events between them."""
  from ranking_b200 import _C
  names = ['embedding_fwd', 'din_fwd', 'tower', 'din_bwd', 'din_input_grad', 'embedding_bwd',
           'optimizer']
  acc = dict.fromkeys(names, 0.0)
  din, mlp, sc = tr.din, tr.mlp, tr.tower
  s, d_din, width = tr.split, din.input_dim, mlp.input_dim
  m = B * N
  for it in range(steps + 1):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(names) + 1)]
    cfg = ctypes.byref(sc._run_cfg(training=True))
    tr._set_tokens(tokens, B, N)
    tr._circular_pad(x, y >= 0)
    lm = (y >= 0).reshape(-1).to(torch.uint8).contiguous()
    dcfg = din._run_cfg(training=True)
    st = _C.stream()
    g = tr.grads
    ev[0].record()
    tr._pool(x, tr.xd, d_din)
    tr.xe[:, :s].copy_(tr.xd[:, :s])
    tr.xe[:, s + HS:].copy_(tr.xd[:, s:])
    ev[1].record()
    _C.check(_C.lib.tfr_din_fwd(_C.ptr(tr.xd), _C.ptr(lm), B, N, ctypes.byref(dcfg),
                                _C.ptr(din.flat.data), _C.ptr(tr.din_ws),
                                ctypes.c_void_p(tr.xe.data_ptr() + 4 * s), width, st))
    ev[2].record()
    _C.check(_C.lib.tfr_mlp_fwd(_C.ptr(tr.xe), m, cfg, _C.ptr(mlp.flat.data), None,
                                _C.ptr(tr.ws), _C.ptr(tr.scores), mlp._precision, st))
    tr.loss.fused_fwd_bwd(y, tr.scores, None, tr.dscores, tr.per_list, tr.total2)
    _C.check(_C.lib.tfr_mlp_bwd(_C.ptr(tr.xe), m, cfg, _C.ptr(mlp.flat.data),
                                _C.ptr(tr.dscores), None, _C.ptr(tr.ws),
                                ctypes.c_void_p(g.data_ptr() + 4 * sc.tower_offset),
                                mlp._precision, st))
    _C.check(_C.lib.tfr_mlp_input_grad(cfg, m, _C.ptr(mlp.flat.data), _C.ptr(tr.ws), 0, width,
                                       _C.ptr(tr.d_xe), width, mlp._precision, st))
    ev[3].record()
    _C.check(_C.lib.tfr_din_bwd(_C.ptr(tr.xd), _C.ptr(lm), B, N, ctypes.byref(dcfg),
                                _C.ptr(din.flat.data), ctypes.c_void_p(tr.d_xe.data_ptr() + 4 * s),
                                width, _C.ptr(tr.din_ws),
                                ctypes.c_void_p(g.data_ptr() + 4 * sc.n_tables), st))
    ev[4].record()
    for c0, c1, dst in ((0, s, 0), (s, d_din, s + HS)):
      if c1 > c0:
        _C.check(_C.lib.tfr_din_input_grad(ctypes.byref(dcfg), B, N, _C.ptr(din.flat.data),
                                           _C.ptr(tr.din_ws), c0, c1 - c0,
                                           ctypes.c_void_p(tr.d_xe.data_ptr() + 4 * dst), width,
                                           1, st))
    ev[5].record()
    tr._tables_bwd(B, N, g, tr.d_xe, width, [0, s + HS])
    ev[6].record()
    tr._apply(g)
    ev[7].record()
    torch.cuda.synchronize()
    if it == 0:
      continue   # warm-up pass
    for i, n in enumerate(names):
      acc[n] += ev[i].elapsed_time(ev[i + 1]) / steps
  return {k: round(v, 3) for k, v in acc.items()}


def torch_step_fn(y, tokens):
  """What a PyTorch user would write: nn.EmbeddingBag (mean, -1 mapped to a padding row that
  the mean skips), tools/din_step.py's attention (einsum projections, SDPA with an additive
  -1e9 mask, layer_norm), a Linear tower, the same ApproxNDCG, autograd, Adagrad."""
  import ranking_b200 as tfr
  dev = y.device

  def glorot(*shape, fan_in, fan_out):
    lim = (6.0 / (fan_in + fan_out)) ** 0.5
    return ((torch.rand(*shape, device=dev) * 2 - 1) * lim).requires_grad_()

  def zeros(*shape):
    return torch.zeros(*shape, device=dev, requires_grad=True)

  bag = torch.nn.EmbeddingBag(V + 1, E, mode='mean', padding_idx=V).to(dev)
  with torch.no_grad():
    bag.weight[:V].uniform_(-0.05, 0.05)
  w_in, b_in = glorot(2 * E, HS, fan_in=2 * E, fan_out=HS), zeros(HS)
  lay = []
  for _ in range(L):
    lay.append([glorot(HS, H, HS, fan_in=H * HS, fan_out=HS * HS), zeros(H, HS),
                glorot(HS, H, HS, fan_in=H * HS, fan_out=HS * HS), zeros(H, HS),
                glorot(HS, H, HS, fan_in=H * HS, fan_out=HS * HS), zeros(H, HS),
                glorot(H, HS, HS, fan_in=H * HS, fan_out=H * HS), zeros(HS),
                torch.ones(HS, device=dev, requires_grad=True), zeros(HS)])
  dims = [2 * E + HS] + HIDDEN + [1]
  lin = [torch.nn.Linear(dims[i], dims[i + 1]).to(dev) for i in range(len(dims) - 1)]
  params = (list(bag.parameters()) + [w_in, b_in] + [p for ps in lay for p in ps] +
            [p for l in lin for p in l.parameters()])
  opt = torch.optim.Adagrad(params, lr=LR, initial_accumulator_value=0.1, eps=1e-7)
  loss_obj = tfr.keras.losses.get('approx_ndcg_loss')
  mask = y >= 0
  add = torch.where(mask, 0.0, -1e9).reshape(B, 1, 1, N)
  q_ids = tokens['context']['query_tokens'].long()
  d_ids = tokens['example']['document_tokens'].long().reshape(B * N, TD)
  q_ids = torch.where(q_ids < 0, torch.full_like(q_ids, V), q_ids)
  d_ids = torch.where(d_ids < 0, torch.full_like(d_ids, V), d_ids)

  def step():
    qe = bag(q_ids).unsqueeze(1).expand(B, N, E)
    de = bag(d_ids).reshape(B, N, E)
    z = torch.relu(torch.cat([qe, de], -1) @ w_in + b_in)
    for wq, bq, wk, bk, wv, bv, wo, bo, gm, bt in lay:
      q = (torch.einsum('bnc,chd->bnhd', z, wq) + bq).transpose(1, 2)
      k = (torch.einsum('bnc,chd->bnhd', z, wk) + bk).transpose(1, 2)
      v = (torch.einsum('bnc,chd->bnhd', z, wv) + bv).transpose(1, 2)
      o = torch.nn.functional.scaled_dot_product_attention(q, k, v, attn_mask=add)
      yv = torch.einsum('bhnd,hde->bne', o, wo) + bo
      z = torch.nn.functional.layer_norm(yv + z, (HS,), gm, bt, eps=1e-12)
    h = torch.cat([qe, z, de], -1).reshape(B * N, -1)
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


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=30)
  ap.add_argument('--warmup', type=int, default=5)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('din_embedding_step.py needs a CUDA device')
  torch.backends.cuda.matmul.allow_tf32 = False
  torch.backends.cudnn.allow_tf32 = False
  res = {'shape': {'B': B, 'N': N, 'T_query': TQ, 'T_document': TD, 'V': V, 'E': E,
                   'din': {'layers': L, 'heads': H, 'head_size': HS}, 'tower': HIDDEN}}
  res.update(card())
  x, y, tokens = batch(0)
  tr = cuda_trainer()
  sec = timed(lambda: tr.train_step(x, y, tokens=tokens), args.steps, args.warmup)
  res['cuda'] = {'lists_per_s': round(B / sec, 1), 'step_ms': round(sec * 1e3, 3),
                 'timed_steps': args.steps,
                 'phases_ms': phases(tr, x, y, tokens, max(20, args.steps))}
  del tr
  torch.cuda.empty_cache()
  step = torch_step_fn(y, tokens)
  ps = timed(step, max(20, args.steps), args.warmup)
  res['pytorch'] = {'lists_per_s': round(B / ps, 1), 'step_ms': round(ps * 1e3, 3)}
  print(json.dumps(res))


if __name__ == '__main__':
  main()
