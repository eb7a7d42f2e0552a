"""Training-step throughput of DINRankingTrainer (csrc/din.cu + the scorer tower) at
config-2 shape: B = 1024 lists of N = 200 items, D = 136 features; DocumentInteractionAttention
with 2 layers x 2 heads x head_size 64, dropout 0; a [256, 128, 64] ReLU tower on [X | E]
(D + h = 200 inputs); ApproxNDCG; Adagrad 0.05.

Prints one JSON line: lists/s and ms/step of DINRankingTrainer.train_step (CUDA events); a
per-phase split of the step (DIN forward, tower forward, loss, tower backward with the input
gradient, DIN backward, optimizer), also with CUDA events; algorithmic FLOPs and bytes against
the FP32 data-sheet rate and HBM bandwidth; and lists/s of a batched PyTorch autograd
formulation of the same model (einsum projections, scaled_dot_product_attention, layer_norm,
fp32 with TF32 off, torch.optim.Adagrad) on the same card.  Needs a CUDA device.

--din_precision fp32,tf32 times the trainer with each DocumentInteractionAttention precision
('cuda', 'cuda_tf32'), and the PyTorch model runs with TF32 off ('pytorch') and on
('pytorch_tf32', torch.backends.cuda.matmul / cudnn allow_tf32): every arm is warmed up, then
the arms take turns for --rounds rounds of --steps steps.  Each trainer's attention kernels
are then timed with torch.profiler, in a run of its own, against the TF32 data-sheet bound of
their FLOPs.
  python tools/din_step.py [--steps 30] [--warmup 5] [--din_precision fp32[,tf32]]
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

B, N, D, H, HS, L, HIDDEN, LR = 1024, 200, 136, 2, 64, 2, [256, 128, 64], 0.05
FP32_PEAK = 67e12        # H100 SXM data sheet, dense FP32
TF32_PEAK = 495e12       # H100 SXM data sheet, dense TF32 (3xTF32 runs three such products)
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


def batch(seed):
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(B, N, D, generator=g)
  y = torch.randint(0, 5, (B, N), generator=g).float()
  y[:, N - 20:] = -1.0
  return x.cuda(), y.cuda()


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


def set_torch_tf32(on):
  torch.backends.cuda.matmul.allow_tf32 = on
  torch.backends.cudnn.allow_tf32 = on


def alternated(arms, steps, warmup, rounds):
  """{name: s per step} of arms [(name, step, torch_tf32)]: each warmed up, then `rounds`
  rounds in which every arm runs `steps` timed steps in turn."""
  for _, step, tf32 in arms:
    set_torch_tf32(tf32)
    for _ in range(warmup):
      step()
  tot = {name: 0.0 for name, _, _ in arms}
  for _ in range(rounds):
    for name, step, tf32 in arms:
      set_torch_tf32(tf32)
      tot[name] += timed(step, steps, 0) / rounds
  set_torch_tf32(False)
  return tot


ATTENTION_KERNELS = ('attn_fwd_kernel', 'attn_bwd_dq_kernel', 'attn_bwd_dkv_kernel',
                     'attn_fwd_tc_kernel', 'attn_bwd_dq_tc_kernel', 'attn_bwd_dkv_tc_kernel')


def attention_flop(b, n, heads, hs, layers):
  """Forward (q.k, P~ v) and backward (S and dP in both passes, dQ, dK, dV) FLOPs."""
  one = 2.0 * b * heads * n * n * hs * layers
  return 2 * one, 7 * one


def attention_kernels(step, steps, fwd_flop, bwd_flop):
  """ms per training step of the DIN's attention kernels (torch.profiler, CUDA activities,
  `steps` steps) and their share of the TF32 data-sheet bound of the attention FLOPs."""
  from torch.profiler import ProfilerActivity, profile
  for _ in range(3):
    step()
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(steps):
      step()
    torch.cuda.synchronize()
  us = dict.fromkeys(ATTENTION_KERNELS, 0.0)
  for evt in prof.events():
    for k in ATTENTION_KERNELS:
      if k + '<' in evt.name and evt.device_time > 0:
        us[k] += evt.device_time / steps
  fwd = sum(v for k, v in us.items() if 'fwd' in k)
  bwd = sum(v for k, v in us.items() if 'bwd' in k)
  out = {k: round(v / 1e3, 3) for k, v in us.items() if v > 0}
  out['fwd_ms'], out['bwd_ms'] = round(fwd / 1e3, 3), round(bwd / 1e3, 3)
  out['fwd_share_of_tf32_bound'] = round(fwd_flop / TF32_PEAK * 1e6 / fwd, 4) if fwd else None
  out['bwd_share_of_tf32_bound'] = round(bwd_flop / TF32_PEAK * 1e6 / bwd, 4) if bwd else None
  return out


def cuda_trainer(precision='fp32'):
  import ranking_b200 as tfr
  din = tfr.keras.layers.DocumentInteractionAttention(H, HS, L, dropout=0.0, seed=1,
                                                      precision=precision).build(D)
  tower = tfr.keras.layers.create_tower(HIDDEN, 1, activation='relu', use_batch_norm=False,
                                        dropout=0, input_dim=D + HS, seed=2,
                                        precision='tf32x3')
  return tfr.train.DINRankingTrainer(din, tower, tfr.keras.losses.get('approx_ndcg_loss'),
                                     optimizer='adagrad', learning_rate=LR)


def phases(tr, x, y, steps):
  """ms per phase of the fused step, CUDA events between the phases of train_step."""
  from ranking_b200 import _C
  names = ['din_fwd', 'tower_fwd', 'loss', 'tower_bwd', 'din_bwd', 'optimizer']
  acc = dict.fromkeys(names, 0.0)
  m = B * N
  for _ in range(steps + 1):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(names) + 1)]
    cfg = ctypes.byref(tr.tower._run_cfg(training=True))
    din, mlp = tr.din, tr.mlp
    st = _C.stream()
    lm = (y >= 0).reshape(-1).to(torch.uint8).contiguous()
    dcfg = ctypes.byref(din._run_cfg(training=True))
    ev[0].record()
    tr.xe.view(B, N, -1)[..., :D].copy_(x)
    _C.check(_C.lib.tfr_din_fwd(_C.ptr(x), _C.ptr(lm), B, N, dcfg, _C.ptr(din.flat.data),
                                _C.ptr(tr.din_ws), ctypes.c_void_p(tr.xe.data_ptr() + 4 * D),
                                D + HS, st))
    ev[1].record()
    _C.check(_C.lib.tfr_mlp_fwd(_C.ptr(tr.xe), m, cfg, _C.ptr(mlp.flat.data), None,
                                _C.ptr(tr.ws), _C.ptr(tr.scores), mlp._precision, st))
    ev[2].record()
    tr.loss.fused_fwd_bwd(y, tr.scores, None, tr.dscores, tr.per_list, tr.total2)
    ev[3].record()
    g = tr.grads
    _C.check(_C.lib.tfr_mlp_bwd(_C.ptr(tr.xe), m, cfg, _C.ptr(mlp.flat.data),
                                _C.ptr(tr.dscores), None, _C.ptr(tr.ws),
                                ctypes.c_void_p(g.data_ptr() + 4 * din.flat.numel()),
                                mlp._precision, st))
    _C.check(_C.lib.tfr_mlp_input_grad(cfg, m, _C.ptr(mlp.flat.data), _C.ptr(tr.ws), D, HS,
                                       _C.ptr(tr.d_emb), HS, mlp._precision, st))
    ev[4].record()
    _C.check(_C.lib.tfr_din_bwd(_C.ptr(x), _C.ptr(lm), B, N, dcfg, _C.ptr(din.flat.data),
                                _C.ptr(tr.d_emb), HS, _C.ptr(tr.din_ws), _C.ptr(g), st))
    ev[5].record()
    tr._apply(g)
    ev[6].record()
    torch.cuda.synchronize()
    if _ == 0:
      continue   # warm-up pass
    for i, n in enumerate(names):
      acc[n] += ev[i].elapsed_time(ev[i + 1]) / steps
  return {k: round(v, 3) for k, v in acc.items()}


def torch_step_fn(x, y):
  """What a PyTorch user would write: batched einsum projections, SDPA with an additive
  -1e9 mask, layer_norm, a Linear tower, the same ApproxNDCG, autograd, Adagrad."""
  import ranking_b200 as tfr
  dev = x.device

  def glorot(*shape, fan_in, fan_out):
    lim = (6.0 / (fan_in + fan_out)) ** 0.5
    return ((torch.rand(*shape, device=dev) * 2 - 1) * lim).requires_grad_()

  def zeros(*shape):
    return torch.zeros(*shape, device=dev, requires_grad=True)

  w_in, b_in = glorot(D, HS, fan_in=D, fan_out=HS), zeros(HS)
  lay = []
  for _ in range(L):
    lay.append([glorot(HS, H, HS, fan_in=H * HS, fan_out=HS * HS), zeros(H, HS),
                glorot(HS, H, HS, fan_in=H * HS, fan_out=HS * HS), zeros(H, HS),
                glorot(HS, H, HS, fan_in=H * HS, fan_out=HS * HS), zeros(H, HS),
                glorot(H, HS, HS, fan_in=H * HS, fan_out=H * HS), zeros(HS),
                torch.ones(HS, device=dev, requires_grad=True), zeros(HS)])
  dims = [D + HS] + HIDDEN + [1]
  tw = [glorot(dims[i], dims[i + 1], fan_in=dims[i], fan_out=dims[i + 1])
        for i in range(len(dims) - 1)]
  tb = [zeros(dims[i + 1]) for i in range(len(dims) - 1)]
  params = [w_in, b_in] + [p for ps in lay for p in ps] + tw + tb
  opt = torch.optim.Adagrad(params, lr=LR, initial_accumulator_value=0.1, eps=1e-7)
  loss_obj = tfr.keras.losses.get('approx_ndcg_loss')
  mask = y >= 0
  add = torch.where(mask, 0.0, -1e9).reshape(B, 1, 1, N)

  def step():
    z = torch.relu(x @ w_in + b_in)
    for wq, bq, wk, bk, wv, bv, wo, bo, gm, bt in lay:
      q = (torch.einsum('bnc,chd->bnhd', z, wq) + bq).transpose(1, 2)
      k = (torch.einsum('bnc,chd->bnhd', z, wk) + bk).transpose(1, 2)
      v = (torch.einsum('bnc,chd->bnhd', z, wv) + bv).transpose(1, 2)
      o = torch.nn.functional.scaled_dot_product_attention(q, k, v, attn_mask=add)
      yv = torch.einsum('bhnd,hde->bne', o, wo) + bo
      z = torch.nn.functional.layer_norm(yv + z, (HS,), gm, bt, eps=1e-12)
    h = torch.cat([x, z], -1)
    for i in range(len(tw)):
      h = h @ tw[i] + tb[i]
      if i + 1 < len(tw):
        h = torch.relu(h)
    logits = torch.where(mask, h.squeeze(-1), torch.full_like(y, -23.025850929940457))
    loss = loss_obj(y, logits)
    opt.zero_grad(set_to_none=True)
    loss.backward()
    opt.step()
  return step


def work():
  """Algorithmic FLOPs and minimum HBM bytes of one training step (fwd + bwd)."""
  m = B * N
  hh = H * HS
  proj = 2.0 * m * (D * HS + L * (HS * 3 * hh + hh * HS))       # forward GEMMs
  attn = 4.0 * B * H * N * N * HS * L                             # q.k and p.v, forward
  tower_dims = [D + HS] + HIDDEN + [1]
  tower = 2.0 * m * sum(a * b for a, b in zip(tower_dims, tower_dims[1:]))
  # backward: two GEMMs per projection / tower layer; attention backward recomputes q.k
  # and does dO.v, dS.k (dQ pass) and q.k, dO.v, dS.q, P.dO (dK / dV pass)
  gemm_flop = 3.0 * (proj + tower)
  attn_flop = attn + 3.0 * attn
  # activations written once and read back in the backward, fp32
  act = m * (HS + L * (3 * hh + hh + 2 * HS + 2) + sum(HIDDEN) + D + HS)
  return gemm_flop, attn_flop, 2.0 * 4 * act


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=30)
  ap.add_argument('--warmup', type=int, default=5)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--din_precision', default='fp32',
                  help='comma-separated DocumentInteractionAttention precisions: fp32, tf32')
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('din_step.py needs a CUDA device')
  set_torch_tf32(False)
  res = {'shape': {'B': B, 'N': N, 'D': D, 'heads': H, 'head_size': HS, 'layers': L,
                   'tower': HIDDEN}}
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
  gemm_flop, attn_flop, byts = work()
  afwd, abwd = attention_flop(B, N, H, HS, L)
  for p, tr in trainers.items():
    sec = secs[key(p)]
    gemm_rate = TF32_PEAK if p == 'tf32' else TF32_PEAK / 3
    attn_rate = TF32_PEAK if p == 'tf32' else FP32_PEAK
    bound = gemm_flop / gemm_rate + attn_flop / attn_rate
    res[key(p)] = {'lists_per_s': round(B / sec, 1), 'step_ms': round(sec * 1e3, 3),
                   'timed_steps': args.steps * args.rounds,
                   'gemm_gflop': round(gemm_flop / 1e9, 1),
                   'attention_gflop': round(attn_flop / 1e9, 1),
                   'bytes_gb': round(byts / 1e9, 2),
                   'compute_bound_ms': round(bound * 1e3, 3),
                   'hbm_bound_ms': round(byts / HBM_BW * 1e3, 3),
                   'share_of_bound': round(max(bound, byts / HBM_BW) / sec, 4),
                   'phases_ms': phases(tr, x, y, max(20, args.steps)),
                   'attention_kernels': attention_kernels(lambda: tr.train_step(x, y), 10,
                                                          afwd, abwd)}
  for name in ('pytorch', 'pytorch_tf32'):
    if name in secs:
      res[name] = {'lists_per_s': round(B / secs[name], 1),
                   'step_ms': round(secs[name] * 1e3, 3)}
  print(json.dumps(res))


if __name__ == '__main__':
  main()
