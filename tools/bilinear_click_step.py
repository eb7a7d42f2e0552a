"""Training-step throughput of BilinearClickRankingTrainer (K14, csrc/bilinear.cu) at config-2
shape: B = 1024 lists of N = 200 items, 136 features, a 256-128-64 ReLU tower in tf32x3 with
output_units = E = 8 (the widest output layer the tower kernels take), 200 positions,
Bilinear(E, 1), SigmoidCrossEntropyLoss on the clicks, Adagrad 0.05, default positions.

Prints one JSON line: lists/s of the bilinear step and of a ClickEMRankingTrainer step on the
same hidden tower and batch, timed alternately in the same process; in a separate
torch.profiler run, the K14 forward and backward times against their HBM bounds (bytes moved,
computed from the shapes, over the data-sheet bandwidth) and the time per step of the
position-table gather and reduction (the embedding kernels); and the card name and power
limit.  Needs a CUDA device.
  python tools/bilinear_click_step.py [--steps 30] [--warmup 5] [--rounds 3]
"""
import argparse
import collections
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import torch  # noqa: E402

from click_em_step import B, N, D, HIDDEN, LR, POSITIONS, HBM_BW  # noqa: E402
from click_em_step import batch, card, timed  # noqa: E402

E = 8
_EMBED = ('embed_fwd', 'bag_grad', 'radix_', 'exclusive_scan', 'segment_bounds', 'chunk_',
          'table_grad')


def trainers():
  import ranking_b200 as tfr

  def tower(out):
    return tfr.keras.layers.create_tower(HIDDEN, out, activation='relu', use_batch_norm=False,
                                         dropout=0, input_dim=D, seed=1, precision='tf32x3')
  two = tfr.train.BilinearClickRankingTrainer(
      tower(E), tfr.keras.layers.Bilinear(E, 1, seed=3),
      tfr.keras.losses.SigmoidCrossEntropyLoss(), POSITIONS, seed=2, optimizer='adagrad',
      learning_rate=LR)
  click = tfr.train.ClickEMRankingTrainer(tower(1), tfr.keras.losses.ClickEMLoss(), POSITIONS,
                                          seed=2, optimizer='adagrad', learning_rate=LR)
  return two, click


def profile_kernels(tr, x, y, steps=5):
  """Per-step device time of the K14 and embedding kernels (torch.profiler)."""
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
    if 'bilinear' not in name and not any(k in name for k in _EMBED):
      continue
    short = name.replace('void ', '').replace('(anonymous namespace)::', '')
    short = short.replace('tfr::', '').split('(')[0]
    out[short] = {'ms_per_step': round(t / 1e3 / steps, 4), 'launches_per_step':
                  e.count // steps}
  return out, total / 1e3 / steps


def _bound(us, nbytes):
  return {'us': round(us, 2), 'bytes': nbytes, 'hbm_bound_us': round(nbytes / HBM_BW * 1e6, 2),
          'share_of_hbm_bound': round(nbytes / HBM_BW / (us * 1e-6), 3)}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=30)
  ap.add_argument('--warmup', type=int, default=5)
  ap.add_argument('--rounds', type=int, default=3)
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('bilinear_click_step.py needs a CUDA device')
  res = {'shape': {'B': B, 'N': N, 'D': D, 'hidden': HIDDEN, 'precision': 'tf32x3',
                   'E': E, 'num_positions': POSITIONS}}
  res.update(card())
  x, y = batch(0)
  two, click = trainers()
  for _ in range(args.warmup):
    two.train_step(x, y)
    click.train_step(x, y)
  t_two, t_click = [], []
  for _ in range(args.rounds):      # alternate so that both see the same card state
    t_two.append(timed(lambda: two.train_step(x, y), args.steps))
    t_click.append(timed(lambda: click.train_step(x, y), args.steps))
  tb, tc = min(t_two), min(t_click)
  res['bilinear_lists_per_s'] = round(B / tb, 1)
  res['click_em_lists_per_s'] = round(B / tc, 1)
  res['bilinear_ms_per_step'] = round(tb * 1e3, 4)
  res['click_em_ms_per_step'] = round(tc * 1e3, 4)
  res['bilinear_over_click_em_step_time'] = round(tb / tc, 4)
  res['step_ms_all_rounds'] = {'bilinear': [round(t * 1e3, 4) for t in t_two],
                               'click_em': [round(t * 1e3, 4) for t in t_click]}
  kernels, prof_step_ms = profile_kernels(two, x, y)
  res['profiled_kernels'] = kernels
  res['profiled_device_ms_per_step'] = round(prof_step_ms, 4)
  m = B * N
  # forward: reads v1, v2 [M, E], writes y [M]; backward: reads v1, v2 and dy, writes dv1,
  # dv2 (the per-CTA partials, a few hundred KB, are left out)
  fwd = kernels['bilinear_fwd_kernel']['ms_per_step'] * 1e3
  bwd = sum(v['ms_per_step'] for k, v in kernels.items() if 'bilinear_bwd' in k or
            'bilinear_reduce' in k) * 1e3
  res['k14_fwd'] = _bound(fwd, m * (8 * E + 4))
  res['k14_bwd'] = _bound(bwd, m * (16 * E + 4))
  emb = sum(v['ms_per_step'] for k, v in kernels.items() if 'bilinear' not in k)
  res['embedding_ms_per_step'] = round(emb, 4)
  res['embedding_share_of_step'] = round(emb / prof_step_ms, 4)
  print(json.dumps(res))


if __name__ == '__main__':
  main()
