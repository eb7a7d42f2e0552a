"""Training-step throughput of ClickEMRankingTrainer (K3d, csrc/loss_click.cu) at config-2
shape: B = 1024 lists of N = 200 items, 136 features, a 256-128-64 ReLU tower in tf32x3,
Adagrad 0.05, clicks as labels, default positions (the row in the list).

Prints one JSON line: lists/s of the click EM step and of a RankingTrainer step with
SigmoidCrossEntropyLoss on the same tower shape and batch, timed alternately in the same
process; in a separate torch.profiler run, the K3d kernel time against its HBM bound (bytes
moved / data-sheet bandwidth) and the time per step of the position-table gather and
reduction (the embedding kernels); and the card name and power limit.  Needs a CUDA device.
  python tools/click_em_step.py [--steps 30] [--warmup 5] [--rounds 3]
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

B, N, D, HIDDEN, LR, POSITIONS = 1024, 200, 136, [256, 128, 64], 0.05, 200
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
  clicks = (torch.rand(B, N, generator=g) < 0.1).float()
  clicks[:, N - 20:] = -1.0
  return x.cuda(), clicks.cuda()


def timed(step, steps):
  torch.cuda.synchronize()
  t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  t0.record()
  for _ in range(steps):
    step()
  t1.record()
  torch.cuda.synchronize()
  return t0.elapsed_time(t1) / 1e3 / steps


def trainers():
  import ranking_b200 as tfr

  def tower():
    return tfr.keras.layers.create_tower(HIDDEN, 1, activation='relu', use_batch_norm=False,
                                         dropout=0, input_dim=D, seed=1, precision='tf32x3')
  click = tfr.train.ClickEMRankingTrainer(tower(), tfr.keras.losses.ClickEMLoss(), POSITIONS,
                                          seed=2, optimizer='adagrad', learning_rate=LR)
  sce = tfr.train.RankingTrainer(tower(), tfr.keras.losses.SigmoidCrossEntropyLoss(),
                                 optimizer='adagrad', learning_rate=LR)
  return click, sce


def profile_kernels(tr, x, y, steps=5):
  """Per-step device time of the embedding, K3d and weighted-sum kernels (torch.profiler)."""
  from torch.profiler import profile, ProfilerActivity
  tr.train_step(x, y)
  torch.cuda.synchronize()
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(steps):
      tr.train_step(x, y)
    torch.cuda.synchronize()
  out = collections.OrderedDict()
  total = 0.0
  for e in prof.key_averages():
    t = getattr(e, 'device_time_total', None)
    if t is None:
      t = e.cuda_time_total
    total += t
    name = e.key
    if not any(k in name for k in ('embed_fwd', 'bag_grad', 'radix_', 'exclusive_scan',
                                   'segment_bounds', 'chunk_', 'table_grad', 'click_em',
                                   'weighted_sum')):
      continue
    short = name.replace('void ', '').replace('(anonymous namespace)::', '')
    short = short.replace('tfr::', '').split('(')[0]
    out[short] = {'ms_per_step': round(t / 1e3 / steps, 4), 'launches_per_step':
                  e.count // steps}
  return out, total / 1e3 / steps


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=30)
  ap.add_argument('--warmup', type=int, default=5)
  ap.add_argument('--rounds', type=int, default=3)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('click_em_step.py needs a CUDA device')
  res = {'shape': {'B': B, 'N': N, 'D': D, 'hidden': HIDDEN, 'precision': 'tf32x3',
                   'num_positions': POSITIONS}}
  res.update(card())
  x, y = batch(0)
  click, sce = trainers()
  for _ in range(args.warmup):
    click.train_step(x, y)
    sce.train_step(x, y)
  t_click, t_sce = [], []
  for _ in range(args.rounds):      # alternate so that both see the same card state
    t_click.append(timed(lambda: click.train_step(x, y), args.steps))
    t_sce.append(timed(lambda: sce.train_step(x, y), args.steps))
  tc, ts = min(t_click), min(t_sce)
  res['click_em_lists_per_s'] = round(B / tc, 1)
  res['sigmoid_ce_lists_per_s'] = round(B / ts, 1)
  res['click_em_ms_per_step'] = round(tc * 1e3, 4)
  res['sigmoid_ce_ms_per_step'] = round(ts * 1e3, 4)
  res['click_over_sce_step_time'] = round(tc / ts, 4)
  res['step_ms_all_rounds'] = {'click_em': [round(t * 1e3, 4) for t in t_click],
                               'sigmoid_ce': [round(t * 1e3, 4) for t in t_sce]}
  kernels, prof_step_ms = profile_kernels(click, x, y)
  res['profiled_kernels'] = kernels
  res['profiled_device_ms_per_step'] = round(prof_step_ms, 4)
  # K3d reads exam, rel, labels (4 B each) and writes d exam, d rel (4 B each) per item, plus
  # the per-list loss and weight
  k3d = kernels['click_em_kernel']['ms_per_step'] / 1e3
  nbytes = B * N * 20 + B * 8
  res['k3d'] = {'us': round(k3d * 1e6, 2), 'bytes': nbytes,
                'hbm_bound_us': round(nbytes / HBM_BW * 1e6, 2),
                'share_of_hbm_bound': round(nbytes / HBM_BW / k3d, 3)}
  emb = sum(v['ms_per_step'] for k, v in kernels.items()
            if 'click_em' not in k and 'weighted_sum' not in k)
  res['embedding_ms_per_step'] = round(emb, 4)
  res['embedding_share_of_step'] = round(emb / prof_step_ms, 4)
  print(json.dumps(res))


if __name__ == '__main__':
  main()
