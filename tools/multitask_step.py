"""Step time of the multi-task fused step against the single-task one, on config 2's shape
(B = 1024 lists, N = 200 items, D = 136 features, 256-128-64 tf32x3 tower, Adagrad):

  single   RankingTrainer, softmax
  T=2      MultiTaskRankingTrainer, softmax + approx NDCG
  T=4      MultiTaskRankingTrainer, softmax + approx NDCG + sigmoid CE + pairwise logistic

The three are alternated in one process (CUDA events around `--steps` steps, median of
`--rounds` rounds), then one profiled step of each (torch.profiler, a separate run) gives the
output-layer forward / backward kernel times.  The card name, power limit and max SM clock are
read in the same call.  Prints one JSON line.

  python tools/multitask_step.py [--steps 50 --rounds 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

B, N, D = 1024, 200, 136
HIDDEN = [256, 128, 64]


def _card():
  q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm',
                      '--format=csv,noheader'], capture_output=True, text=True).stdout
  return q.strip().splitlines()[0] if q.strip() else 'unknown'


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=50)
  ap.add_argument('--rounds', type=int, default=5)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('multitask_step needs a CUDA device')
  import __graft_entry__ as entry
  entry.build()
  import ranking_b200 as tfr
  L = tfr.keras.losses
  g = torch.Generator().manual_seed(0)
  x = torch.randn(B, N, D, generator=g).cuda()
  y = torch.randint(0, 5, (B, N), generator=g).float()
  y[:, 150:] = -1.0
  y = y.cuda()
  clicks = torch.where(y >= 0, (y > 2).float(), y)
  names = ['softmax_loss', 'approx_ndcg_loss', 'sigmoid_cross_entropy_loss',
           'pairwise_logistic_loss']

  def tower(out):
    return tfr.keras.layers.create_tower(HIDDEN, out, activation='relu', use_batch_norm=False,
                                         dropout=0, input_dim=D, seed=1, precision='tf32x3')

  mask = y >= 0
  single = tfr.train.RankingTrainer(tower(1), L.get('softmax_loss'), learning_rate=0.01)
  runs = {'single': lambda: single.train_step(x, y, mask=mask)}
  for t in (2, 4):
    tr = tfr.train.MultiTaskRankingTrainer(
        tower(t), {'task%d' % i: L.get(names[i]) for i in range(t)}, learning_rate=0.01)
    labels = {'task%d' % i: (y if i % 2 == 0 else clicks) for i in range(t)}
    runs['T=%d' % t] = (lambda tr=tr, labels=labels: tr.train_step(x, labels, mask=mask))

  for fn in runs.values():        # warm up every shape
    for _ in range(5):
      fn()
  torch.cuda.synchronize()
  times = {k: [] for k in runs}
  for _ in range(args.rounds):
    for k, fn in runs.items():
      a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
      a.record()
      for _ in range(args.steps):
        fn()
      b.record()
      torch.cuda.synchronize()
      times[k].append(a.elapsed_time(b) / args.steps)
  step_ms = {k: statistics.median(v) for k, v in times.items()}

  from torch.profiler import ProfilerActivity, profile
  kernels = {}
  for k, fn in runs.items():
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
      for _ in range(5):
        fn()
      torch.cuda.synchronize()
    per = {}
    for ev in prof.key_averages():
      if 'out_layer' in ev.key or 'tower_fused_fwd' in ev.key:
        dev_us = getattr(ev, 'device_time_total', None)
        if dev_us is None:
          dev_us = ev.cuda_time_total
        per[ev.key] = round(dev_us / 5.0, 2)
    kernels[k] = per
  print(json.dumps({'card': _card(), 'shape': [B, N, D], 'tower': HIDDEN,
                    'step_ms_median': step_ms, 'step_ms_rounds': times,
                    'slowdown_T2_pct': round(100 * (step_ms['T=2'] / step_ms['single'] - 1), 2),
                    'slowdown_T4_pct': round(100 * (step_ms['T=4'] / step_ms['single'] - 1), 2),
                    'kernel_us_per_step': kernels}))


if __name__ == '__main__':
  main()
