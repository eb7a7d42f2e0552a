"""Training-step throughput of the GAM ranking model (csrc/gam.cu) on the canned-GAM
recipe (examples/tf_ranking_canned_gam.py of the reference) at config-2 shape: B = 1024
lists of N = 200 items, 136 scalar features, [16, 8] ReLU towers, ApproxNDCG, Adagrad 0.05.

Prints one JSON line: lists/s of GAMRankingTrainer.train_step with BN + dropout 0.5 and
with neither; per-sweep kernel times (torch.profiler, a separate run); launches per step;
algorithmic FLOPs and bytes against the FP32 data-sheet rate and HBM bandwidth; and lists/s
of a batched PyTorch formulation of the same model (einsum over the feature axis, fp32,
autograd, torch.optim.Adagrad) on the same card.  Needs a CUDA device.
  python tools/gam_step.py [--steps 30] [--warmup 5]
"""
import argparse
import collections
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

B, N, F, HIDDEN, LR = 1024, 200, 136, [16, 8], 0.05
FP32_PEAK = 67e12        # H100 SXM data sheet, dense FP32
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
  x = torch.randn(B, N, F, generator=g)
  y = torch.randint(0, 5, (B, N), generator=g).float()
  y[:, N - 20:] = -1.0      # padded tail: circular padding runs with BN
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


def cuda_trainer(bn, dropout):
  import ranking_b200 as tfr
  gam = tfr.keras.layers.GAMLayer(F, HIDDEN, activation='relu', use_batch_norm=bn,
                                  dropout=dropout, seed=1)
  return tfr.train.GAMRankingTrainer(gam, tfr.keras.losses.get('approx_ndcg_loss'), [1] * F,
                                     optimizer='adagrad', learning_rate=LR)


def torch_step_fn(bn, dropout, x, y):
  """What a PyTorch user would write: all F towers as batched tensors over the feature
  axis, einsum / bmm, autograd, BN over every (feature, unit) channel."""
  import ranking_b200 as tfr
  dev = x.device
  dims = [1] + HIDDEN + [1]
  ws, bs = [], []
  for i in range(len(dims) - 1):
    lim = (6.0 / (dims[i] + dims[i + 1])) ** 0.5
    ws.append(((torch.rand(F, dims[i], dims[i + 1], device=dev) * 2 - 1) * lim).requires_grad_())
    bs.append(torch.zeros(F, dims[i + 1], device=dev, requires_grad=True))
  bns = [torch.nn.BatchNorm1d(F * h, eps=1e-3, momentum=1 - 0.999).to(dev) for h in HIDDEN]
  params = ws + bs + ([p for m in bns for p in m.parameters()] if bn else [])
  opt = torch.optim.Adagrad(params, lr=LR, initial_accumulator_value=0.1, eps=1e-7)
  loss_obj = tfr.keras.losses.get('approx_ndcg_loss')
  mask = y >= 0
  xf = x.reshape(B * N, F, 1)

  def step():
    h = xf
    for i in range(len(HIDDEN)):
      h = torch.einsum('mfk,fkh->mfh', h, ws[i]) + bs[i]
      if bn:
        h = bns[i](h.reshape(B * N, -1)).reshape(B * N, F, -1)
      h = torch.relu(h)
      if dropout:
        h = torch.nn.functional.dropout(h, dropout, training=True)
    s = (torch.einsum('mfk,fkh->mfh', h, ws[-1]) + bs[-1]).sum((1, 2))
    logits = torch.where(mask, s.reshape(B, N), torch.full_like(y, -23.025850929940457))
    loss = loss_obj(y, logits)
    opt.zero_grad(set_to_none=True)
    loss.backward()
    opt.step()
  return step


def sweep_times(trainer, x, y, steps=5):
  """Mean time per launch of each GAM kernel over `steps` steps (torch.profiler)."""
  from torch.profiler import profile, ProfilerActivity
  trainer.train_step(x, y)
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(steps):
      trainer.train_step(x, y)
    torch.cuda.synchronize()
  out = collections.OrderedDict()
  for e in prof.key_averages():
    name = e.key
    if 'gam_' not in name and 'reduce_partials' not in name and 'approx' not in name:
      continue
    short = name.replace('void ', '').replace('(anonymous namespace)::', '')
    short = short.replace('tfr::', '').split('(')[0]
    t = getattr(e, 'device_time_total', None)
    if t is None:
      t = e.cuda_time_total
    out[short] = {'ms_per_step': round(t / 1e3 / steps, 4), 'launches_per_step':
                  e.count // steps}
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=30)
  ap.add_argument('--warmup', type=int, default=5)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('gam_step.py needs a CUDA device')
  import ranking_b200 as tfr
  res = {'shape': {'B': B, 'N': N, 'features': F, 'hidden': HIDDEN}}
  res.update(card())
  x, y = batch(0)
  m = B * N
  fan = sum(a * b for a, b in zip([1] + HIDDEN, HIDDEN + [1]))
  fwd_flop = 2.0 * m * F * fan
  for tag, bn, dropout in (('bn_dropout', True, 0.5), ('plain', False, 0.0)):
    tr = cuda_trainer(bn, dropout)
    sec = timed(lambda: tr.train_step(x, y), args.steps, args.warmup)
    before = tfr._C.lib.tfr_launch_count()
    tr.train_step(x, y)
    torch.cuda.synchronize()
    launches = tfr._C.lib.tfr_launch_count() - before
    # sweeps over X: forward = one per BN layer + 1; backward = one per BN layer + 1
    sweeps = 2 * (len(HIDDEN) + 1) if bn else 2
    flop = 3.0 * fwd_flop           # forward + about twice that backward (algorithmic)
    byts = sweeps * m * F * 4.0 + 2 * m * F * 4.0   # X per sweep + sublogits write / read
    t_min = max(flop / FP32_PEAK, byts / HBM_BW)
    res[tag] = {
        'lists_per_s': round(B / sec, 1), 'step_ms': round(sec * 1e3, 3),
        'launches_per_step': int(launches), 'algorithmic_gflop': round(flop / 1e9, 2),
        'bytes_gb': round(byts / 1e9, 3), 'bound': 'fp32' if flop / FP32_PEAK >
        byts / HBM_BW else 'hbm', 'share_of_bound': round(t_min / sec, 4),
        'sweeps': sweeps, 'kernels': sweep_times(tr, x, y)}
    del tr
    torch.cuda.empty_cache()
    try:
      step = torch_step_fn(bn, dropout, x, y)
      res[tag]['pytorch_lists_per_s'] = round(B / timed(step, max(5, args.steps // 3),
                                                         args.warmup), 1)
      del step
    except torch.cuda.OutOfMemoryError:
      res[tag]['pytorch_lists_per_s'] = 'out of memory'
    torch.cuda.empty_cache()
  print(json.dumps(res))


if __name__ == '__main__':
  main()
