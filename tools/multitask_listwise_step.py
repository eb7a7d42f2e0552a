"""Training-step time of the multi-task listwise trainers against their single-task
counterparts at DASALC's Web30K shape: B = 128 lists of N = 200 items, D = 136 features; a
4-layer, 2-head, head_size 100 DocumentInteractionAttention; DASALC with W = 512 (dropout 0.4,
input noise 1.5), and for the DIN trainer a [512, 256] ReLU tower in 3xTF32.  Every task uses
the softmax loss and Adagrad.

Per scorer (din, dasalc) the arms are the single-task trainer and the multi-task trainer with
T = 1, 2 and 4 tasks, alternated in the same process (tools/din_step.py's `alternated`).
Prints one JSON line: ms per step of every arm, T = 1 over the single-task trainer and T = 4
over T = 1, with the card's name and power limit.  Needs a CUDA device.
  python tools/multitask_listwise_step.py [--steps 20] [--warmup 5] [--rounds 3]
                                          [--din_precision fp32|tf32]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

import torch  # noqa: E402

from din_step import alternated, card  # noqa: E402

B, N, D, W, HS, H, L = 128, 200, 136, 512, 100, 2, 4
HIDDEN = [512, 256]
RATE, NOISE, MOM, LR = 0.4, 1.5, 0.9, 0.05
TASKS = (1, 2, 4)


def batch(seed, tasks):
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(B, N, D, generator=g) * 5
  ys = {}
  for t in range(tasks):
    y = torch.randint(0, 5, (B, N), generator=g).float()
    y[:, N - 20:] = -1.0
    ys['task%d' % t] = y.cuda()
  return x.cuda(), ys


def trainer(kind, tasks, din_precision):
  """tasks None: the single-task trainer."""
  import ranking_b200 as tfr
  from ranking_b200.research import dasalc
  din = tfr.keras.layers.DocumentInteractionAttention(H, HS, L, dropout=RATE,
                                                      input_noise_stddev=NOISE, seed=1,
                                                      precision=din_precision)
  units = tasks or 1
  if kind == 'dasalc':
    part = dasalc.DASALCScorer(D, W, HS, dropout=RATE, input_noise_stddev=NOISE,
                               batch_norm_moment=MOM, seed=2, output_units=units)
  else:
    part = tfr.keras.layers.create_tower(HIDDEN, units, activation='relu', input_dim=D + HS,
                                         seed=2, precision='tf32x3')
  kw = dict(optimizer='adagrad', learning_rate=LR)
  if tasks is None:
    cls = tfr.train.DASALCRankingTrainer if kind == 'dasalc' else tfr.train.DINRankingTrainer
    return cls(din, part, tfr.keras.losses.get('softmax_loss'), **kw)
  cls = (tfr.train.MultiTaskDASALCRankingTrainer if kind == 'dasalc'
         else tfr.train.MultiTaskDINRankingTrainer)
  losses = {'task%d' % t: tfr.keras.losses.get('softmax_loss') for t in range(tasks)}
  return cls(din, part, losses, **kw)


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--warmup', type=int, default=5)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--din_precision', default='fp32', choices=['fp32', 'tf32'])
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('needs a CUDA device')
  import __graft_entry__ as entry
  entry.build()
  out = {'shape': {'B': B, 'N': N, 'D': D, 'W': W, 'head_size': HS, 'heads': H, 'layers': L},
         'din_precision': args.din_precision, 'steps': args.steps, 'rounds': args.rounds}
  out.update(card())
  x, ys = batch(0, max(TASKS))
  for kind in ('din', 'dasalc'):
    arms = []
    for tasks in (None,) + TASKS:
      tr = trainer(kind, tasks, args.din_precision)
      if tasks is None:
        step = (lambda tr=tr: tr.train_step(x, ys['task0']))
        name = 'single'
      else:
        labels = {'task%d' % t: ys['task%d' % t] for t in range(tasks)}
        step = (lambda tr=tr, labels=labels: tr.train_step(x, labels))
        name = 'T%d' % tasks
      arms.append((name, step, False))
    sec = alternated(arms, args.steps, args.warmup, args.rounds)
    ms = {k: round(v * 1e3, 3) for k, v in sec.items()}
    out[kind] = {'ms_per_step': ms,
                 'T1_over_single': round(sec['T1'] / sec['single'], 4),
                 'T4_over_T1': round(sec['T4'] / sec['T1'], 4)}
  print(json.dumps(out))


if __name__ == '__main__':
  main()
