"""Training-step throughput of DASALCRankingTrainer (csrc/din.cu + csrc/dasalc.cu) at the
reference's Web30K shape: B = 128 lists of N = 200 items, D = 136 features; a 4-layer, 2-head,
head_size 100 DocumentInteractionAttention and the latent-cross scorer with W = 512, dropout 0.4,
input noise 1.5, BN momentum 0.9; softmax loss; Adagrad.

Prints one JSON line: lists/s and ms/step of train_step (CUDA events); the DIN's and the
scorer's share of the step (CUDA events between the phases of the same chain); the two
latent-cross kernels' times (torch.profiler, in a run of their own) against their HBM byte
bounds; and lists/s of a batched PyTorch autograd formulation of the same model (fp32, TF32
off, torch.optim.Adagrad) on the same card, with the card's name and power limit.  Needs a
CUDA device.

--din_precision fp32,tf32 times the trainer with each DocumentInteractionAttention precision
('cuda', 'cuda_tf32'), and the PyTorch model runs with TF32 off ('pytorch') and on
('pytorch_tf32'), the arms alternated as in tools/din_step.py; each trainer's attention kernels
are timed with torch.profiler in a run of their own, against the TF32 data-sheet bound.
  python tools/dasalc_step.py [--steps 30] [--warmup 5] [--din_precision fp32[,tf32]]
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

from din_step import (alternated, attention_flop, attention_kernels, card,  # noqa: E402
                      set_torch_tf32)

B, N, D, W, HS, H, L = 128, 200, 136, 512, 100, 2, 4
RATE, NOISE, MOM, LR = 0.4, 1.5, 0.9, 0.05
HBM_BW = 3.35e12         # H100 SXM data sheet


def batch(seed):
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(B, N, D, generator=g) * 5
  y = torch.randint(0, 5, (B, N), generator=g).float()
  y[:, N - 20:] = -1.0
  return x.cuda(), y.cuda()


def cuda_trainer(precision='fp32'):
  import ranking_b200 as tfr
  from ranking_b200.research import dasalc
  din = tfr.keras.layers.DocumentInteractionAttention(H, HS, L, dropout=RATE,
                                                      input_noise_stddev=NOISE, seed=1,
                                                      precision=precision)
  sc = dasalc.DASALCScorer(D, W, HS, dropout=RATE, input_noise_stddev=NOISE,
                           batch_norm_moment=MOM, seed=2)
  return tfr.train.DASALCRankingTrainer(din, sc, tfr.keras.losses.get('softmax_loss'),
                                        optimizer='adagrad', learning_rate=LR)


def phases(tr, x, y, steps):
  """ms per phase of the fused step (the chain of DASALCRankingTrainer.train_step)."""
  from ranking_b200 import _C
  names = ['transform_pad', 'din_fwd', 'scorer_fwd', 'loss', 'scorer_bwd', 'din_bwd',
           'optimizer']
  acc = dict.fromkeys(names, 0.0)
  m = B * N
  mask = y >= 0
  m8 = mask.reshape(-1).to(torch.uint8).contiguous()
  din, sc = tr.din, tr.scorer
  for it in range(steps + 1):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(names) + 1)]
    cfg = ctypes.byref(sc._run_cfg(training=True))
    dcfg = ctypes.byref(din._run_cfg(training=True))
    st = _C.stream()
    ev[0].record()
    xp = tr._circular_pad(tr._prep_x(x), mask)
    ev[1].record()
    _C.check(_C.lib.tfr_din_fwd(_C.ptr(xp), _C.ptr(m8), B, N, dcfg, _C.ptr(din.flat.data),
                                _C.ptr(tr.din_ws), _C.ptr(tr.emb), HS, st))
    ev[2].record()
    _C.check(_C.lib.tfr_dasalc_fwd(_C.ptr(xp), _C.ptr(tr.emb), HS, m, cfg, _C.ptr(sc.flat.data),
                                   _C.ptr(m8), _C.ptr(tr.ws), _C.ptr(tr.scores), sc._precision,
                                   st))
    ev[3].record()
    tr.loss.fused_fwd_bwd(y, tr.scores, None, tr.dscores, tr.per_list, tr.total2)
    ev[4].record()
    g = tr.grads
    _C.check(_C.lib.tfr_dasalc_bwd(_C.ptr(xp), m, cfg, _C.ptr(sc.flat.data), _C.ptr(tr.dscores),
                                   _C.ptr(m8), _C.ptr(tr.ws),
                                   ctypes.c_void_p(g.data_ptr() + 4 * din.flat.numel()),
                                   _C.ptr(tr.d_emb), HS, sc._precision, st))
    ev[5].record()
    _C.check(_C.lib.tfr_din_bwd(_C.ptr(xp), _C.ptr(m8), B, N, dcfg, _C.ptr(din.flat.data),
                                _C.ptr(tr.d_emb), HS, _C.ptr(tr.din_ws), _C.ptr(g), st))
    ev[6].record()
    tr._apply(g)
    ev[7].record()
    torch.cuda.synchronize()
    if it == 0:
      continue   # warm-up pass
    for i, n in enumerate(names):
      acc[n] += ev[i].elapsed_time(ev[i + 1]) / steps
  return {k: round(v, 3) for k, v in acc.items()}


def cross_kernels(tr, x, y, steps):
  """Mean µs of the latent-cross forward and backward kernels over `steps` training steps
  (torch.profiler, CUDA activities)."""
  from torch.profiler import ProfilerActivity, profile
  for _ in range(3):
    tr.train_step(x, y)
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(steps):
      tr.train_step(x, y)
    torch.cuda.synchronize()
  tot = {'cross_fwd_kernel': [0.0, 0], 'cross_bwd_kernel': [0.0, 0]}
  for evt in prof.events():
    for k in tot:
      if k in evt.name and evt.device_time > 0:
        tot[k][0] += evt.device_time
        tot[k][1] += 1
  m = B * N
  fwd_bytes = 2.0 * 4 * m * W + 4 * m            # read t, c; write s
  bwd_bytes = 4.0 * 4 * m * W + 4 * m            # read t, c; write dt, dc; read ds
  out = {}
  for k, byts in (('cross_fwd_kernel', fwd_bytes), ('cross_bwd_kernel', bwd_bytes)):
    us = tot[k][0] / max(tot[k][1], 1)
    bound = byts / HBM_BW * 1e6
    out[k] = {'us': round(us, 2), 'calls': tot[k][1], 'bytes_mb': round(byts / 1e6, 1),
              'hbm_bound_us': round(bound, 2),
              'share_of_bound': round(bound / us, 3) if us > 0 else None}
  return out


def torch_step_fn(x, y):
  """What a PyTorch user would write: the same transform, circular padding by gather, einsum
  attention projections with SDPA and layer_norm, batch_norm / dropout / the latent cross as
  torch ops, the same softmax loss, autograd, Adagrad."""
  import ranking_b200 as tfr
  from ranking_b200 import utils
  dev = x.device
  F = torch.nn.functional

  def glorot(*shape, fan_in, fan_out):
    lim = (6.0 / (fan_in + fan_out)) ** 0.5
    return ((torch.rand(*shape, device=dev) * 2 - 1) * lim).requires_grad_()

  def zeros(*shape):
    return torch.zeros(*shape, device=dev, requires_grad=True)

  def ones(*shape):
    return torch.ones(*shape, device=dev, requires_grad=True)

  w_in, b_in = glorot(D, HS, fan_in=D, fan_out=HS), zeros(HS)
  lay = []
  for _ in range(L):
    lay.append([glorot(HS, H, HS, fan_in=H * HS, fan_out=HS * HS), zeros(H, HS),
                glorot(HS, H, HS, fan_in=H * HS, fan_out=HS * HS), zeros(H, HS),
                glorot(HS, H, HS, fan_in=H * HS, fan_out=HS * HS), zeros(H, HS),
                glorot(H, HS, HS, fan_in=H * HS, fan_out=H * HS), zeros(HS), ones(HS),
                zeros(HS)])
  dense = {'1': (D, W), '2': (W, W), 't': (W, W), 'c': (HS, W), 'o': (W, 1)}
  kw = {k: glorot(a, b, fan_in=a, fan_out=b) for k, (a, b) in dense.items()}
  kb = {k: zeros(b) for k, (a, b) in dense.items()}
  bn = {k: (ones(w), zeros(w)) for k, w in (('in', D), ('1', W), ('2', W), ('c', HS))}
  run = {k: (torch.zeros(w, device=dev), torch.ones(w, device=dev))
         for k, w in (('in', D), ('1', W), ('2', W), ('c', HS))}
  params = [w_in, b_in] + [p for ps in lay for p in ps] + list(kw.values()) + \
      list(kb.values()) + [p for pr in bn.values() for p in pr]
  opt = torch.optim.Adagrad(params, lr=LR, initial_accumulator_value=0.1, eps=1e-7)
  loss_obj = tfr.keras.losses.get('softmax_loss')
  mask = y >= 0
  add = torch.where(mask, 0.0, -1e9).reshape(B, 1, 1, N)
  idx = utils.padded_nd_indices(mask)[0].long()

  def norm(k, t):
    return F.batch_norm(t, run[k][0], run[k][1], bn[k][0], bn[k][1], training=True,
                        momentum=1 - MOM, eps=1e-3)

  def step():
    xt = torch.clamp(torch.sign(x) * torch.log1p(x.abs()), -30.0, 30.0)
    xt = torch.gather(xt, 1, idx.unsqueeze(-1).expand(-1, -1, D))
    z = torch.relu(xt @ w_in + b_in)
    z = z + NOISE * torch.randn_like(z)
    for wq, bq, wk, bk, wv, bv, wo, bo, gm, bt in lay:
      q = (torch.einsum('bnc,chd->bnhd', z, wq) + bq).transpose(1, 2)
      k = (torch.einsum('bnc,chd->bnhd', z, wk) + bk).transpose(1, 2)
      v = (torch.einsum('bnc,chd->bnhd', z, wv) + bv).transpose(1, 2)
      o = F.scaled_dot_product_attention(q, k, v, attn_mask=add, dropout_p=RATE)
      yv = F.dropout(torch.einsum('bhnd,hde->bne', o, wo) + bo, RATE)
      z = F.layer_norm(yv + z, (HS,), gm, bt, eps=1e-12)
    a = norm('in', xt.reshape(-1, D))
    a = a + NOISE * torch.randn_like(a)
    for i in ('1', '2'):
      a = F.dropout(norm(i, torch.relu(a @ kw[i] + kb[i])), RATE)
    t = a @ kw['t'] + kb['t']
    c = norm('c', z.reshape(-1, HS)) @ kw['c'] + kb['c']
    o = F.dropout(torch.relu(t * c + t), RATE)
    s = (o @ kw['o'] + kb['o']).reshape(B, N)
    logits = torch.where(mask, s, torch.full_like(y, -23.025850929940457))
    loss = loss_obj(y, logits)
    opt.zero_grad(set_to_none=True)
    loss.backward()
    opt.step()
  return step


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=30)
  ap.add_argument('--warmup', type=int, default=5)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--din_precision', default='fp32',
                  help='comma-separated DocumentInteractionAttention precisions: fp32, tf32')
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('dasalc_step.py needs a CUDA device')
  set_torch_tf32(False)
  res = {'shape': {'B': B, 'N': N, 'D': D, 'hidden': W, 'heads': H, 'head_size': HS,
                   'layers': L}}
  res.update(card())
  x, y = batch(0)
  precs = args.din_precision.split(',')
  trainers = {p: cuda_trainer(p) for p in precs}
  key = lambda p: 'cuda' if p == 'fp32' else 'cuda_' + p
  arms = [(key(p), (lambda tr: lambda: tr.train_step(x, y))(tr), False)
          for p, tr in trainers.items()]
  try:
    step = torch_step_fn(x, y)
    arms += [('pytorch', step, False), ('pytorch_tf32', step, True)]
  except torch.cuda.OutOfMemoryError:
    res['pytorch'] = 'out of memory'
  secs = alternated(arms, args.steps, args.warmup, args.rounds)
  afwd, abwd = attention_flop(B, N, H, HS, L)
  for p, tr in trainers.items():
    sec = secs[key(p)]
    ph = phases(tr, x, y, max(20, args.steps))
    total = sum(ph.values())
    res[key(p)] = {'lists_per_s': round(B / sec, 1), 'step_ms': round(sec * 1e3, 3),
                   'timed_steps': args.steps * args.rounds, 'phases_ms': ph,
                   'din_share': round((ph['din_fwd'] + ph['din_bwd']) / total, 3),
                   'scorer_share': round((ph['scorer_fwd'] + ph['scorer_bwd']) / total, 3),
                   'attention_gflop': {'fwd': round(afwd / 1e9, 1), 'bwd': round(abwd / 1e9, 1)},
                   'attention_kernels': attention_kernels(lambda: tr.train_step(x, y), 10,
                                                          afwd, abwd)}
    if p == 'fp32':
      res['cross_kernels'] = cross_kernels(tr, x, y, 10)
  for name in ('pytorch', 'pytorch_tf32'):
    if name in secs:
      res[name] = {'lists_per_s': round(B / secs[name], 1),
                   'step_ms': round(secs[name] * 1e3, 3)}
  print(json.dumps(res))


if __name__ == '__main__':
  main()
