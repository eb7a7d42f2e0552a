"""Multi-task ranking from ELWC TFRecords: one tower, one score per task, a loss per task and
per-task loss weights (the reference's MultiTaskPipeline, keras/pipeline.py:733-824).

  python examples/multitask_train.py --train a.tfrecord --valid b.tfrecord \\
      --example_features f:136 --labels relevance=label,click=clicked \\
      --losses relevance=softmax_loss,click=sigmoid_cross_entropy_loss --loss_weights click=0.5

  python examples/multitask_train.py --synthetic     # seeded data, no files needed
  python examples/multitask_train.py --synthetic --scorer din      # listwise context
  python examples/multitask_train.py --synthetic --scorer dasalc

--scorer picks the model that carries a score plane per task: `dnn` (default) a create_tower
tower (MultiTaskRankingTrainer), `din` a DocumentInteractionAttention embedding feeding that
tower (MultiTaskDINRankingTrainer), `dasalc` the DIN and a DASALCScorer
(MultiTaskDASALCRankingTrainer; features go through log1p_cutoff first).

--synthetic writes TFRecords whose two labels come from two different linear utilities of
the same features (a graded relevance and a binary click), trains both tasks and prints each
task's validation NDCG.
"""
import argparse
import os
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def _pairs(s, cast=str):
  out = {}
  for part in filter(None, s.split(',')):
    k, v = part.split('=') if '=' in part else part.split(':')
    out[k] = cast(v)
  return out


def write_synthetic(directory, n_lists=768, list_size=20, dim=16, seed=0):
  from ranking_b200 import data
  g = torch.Generator().manual_seed(seed)
  u_rel, u_click = torch.randn(dim, generator=g), torch.randn(dim, generator=g)
  paths = []
  for split, count in (('train', n_lists), ('valid', n_lists // 4)):
    recs = []
    for _ in range(count):
      f = torch.randn(list_size, dim, generator=g)
      rel = torch.bucketize(f @ u_rel, torch.tensor([-1.0, 0.0, 1.0])).float()
      click = (f @ u_click > 0.5).float()
      recs.append(data.encode_elwc(None, [
          {'f': f[i].tolist(), 'label': [float(rel[i])], 'clicked': [float(click[i])]}
          for i in range(list_size)]))
    path = os.path.join(directory, split + '.tfrecord')
    data.write_tfrecords(path, recs)
    paths.append(path)
  return paths, {'f': (dim, 0.0), 'label': (1, -1.0), 'clicked': (1, -1.0)}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--train')
  ap.add_argument('--valid')
  ap.add_argument('--synthetic', action='store_true')
  ap.add_argument('--example_features', default='',
                  help='name:dim,... (label features too, they are removed from x)')
  ap.add_argument('--labels', default='relevance=label,click=clicked')
  ap.add_argument('--losses', default='relevance=softmax_loss,click=sigmoid_cross_entropy_loss')
  ap.add_argument('--loss_weights', default='')
  ap.add_argument('--list_size', type=int, default=20)
  ap.add_argument('--batch_size', type=int, default=32)
  ap.add_argument('--hidden', default='64,32', help='tower widths of --scorer dnn / din')
  ap.add_argument('--scorer', default='dnn', choices=['dnn', 'din', 'dasalc'])
  ap.add_argument('--din_heads', type=int, default=2)
  ap.add_argument('--din_head_size', type=int, default=16, help='also DASALC context_dim')
  ap.add_argument('--din_layers', type=int, default=1)
  ap.add_argument('--dasalc_hidden', type=int, default=64, help='DASALC hidden_dim W')
  ap.add_argument('--epochs', type=int, default=6)
  ap.add_argument('--steps_per_epoch', type=int, default=24)
  ap.add_argument('--learning_rate', type=float, default=0.1)
  ap.add_argument('--model_dir', default=None)
  ap.add_argument('--work_dir', default=None,
                  help='where --synthetic writes its records (default: a new temporary directory)')
  args = ap.parse_args()

  import __graft_entry__ as entry
  entry.build()
  import ranking_b200 as tfr
  from ranking_b200 import data, pipeline

  tmp = args.work_dir or tempfile.mkdtemp(prefix='multitask_')
  labels = _pairs(args.labels)
  if args.synthetic:
    (train, valid), ex_spec = write_synthetic(tmp, list_size=args.list_size)
  else:
    if not (args.train and args.valid and args.example_features):
      ap.error('--train, --valid and --example_features are required without --synthetic')
    train, valid = args.train, args.valid
    ex_spec = {k: (v, -1.0 if k in labels.values() else 0.0)
               for k, v in _pairs(args.example_features, int).items()}
  losses = _pairs(args.losses)
  if set(losses) != set(labels):
    ap.error('--losses and --labels must name the same tasks')
  losses = {t: losses[t] for t in labels}
  weights = _pairs(args.loss_weights, float) or None
  input_dim = sum(d for k, (d, _) in ex_spec.items() if k not in labels.values())
  hidden = [int(h) for h in args.hidden.split(',')]

  def batches(path):
    return lambda: data.elwc_multilabel_batches(path, args.batch_size, args.list_size, {},
                                                ex_spec, labels)

  hp = pipeline.PipelineHparams(
      model_dir=args.model_dir or os.path.join(tmp, 'model'), num_epochs=args.epochs,
      steps_per_epoch=args.steps_per_epoch, validation_steps=8,
      learning_rate=args.learning_rate, loss=losses, loss_weights=weights)
  def model():
    t = len(labels)
    if args.scorer == 'dnn':
      return tfr.keras.layers.create_tower(hidden, t, activation='relu', input_dim=input_dim,
                                           seed=1, precision='tf32x3')
    din = tfr.keras.layers.DocumentInteractionAttention(args.din_heads, args.din_head_size,
                                                        args.din_layers, dropout=0.0, seed=2)
    din.build(input_dim)
    if args.scorer == 'din':
      return din, tfr.keras.layers.create_tower(hidden, t, activation='relu',
                                                input_dim=input_dim + args.din_head_size,
                                                seed=1, precision='tf32x3')
    from ranking_b200.research import dasalc
    return din, dasalc.DASALCScorer(input_dim, args.dasalc_hidden, args.din_head_size,
                                    dropout=0.0, input_noise_stddev=0.0, seed=1,
                                    output_units=t)

  trainer_cls = {'dnn': None, 'din': tfr.train.MultiTaskDINRankingTrainer,
                 'dasalc': tfr.train.MultiTaskDASALCRankingTrainer}[args.scorer]
  p = pipeline.MultiTaskPipeline(model, batches(train), batches(valid), hp,
                                 trainer_cls=trainer_cls)
  hist = p.train_and_validate()
  last = hist[-1]
  print('scorer %s, epochs %d, validation loss %.5f' % (args.scorer, len(hist), last['loss']))
  for t in labels:
    print('%-12s loss %.5f  NDCG@1 %.4f  NDCG@5 %.4f  NDCG@10 %.4f  NDCG %.4f' % (
        t, last[t + '_loss'], last[t + '_metric/ndcg_1'], last[t + '_metric/ndcg_5'],
        last[t + '_metric/ndcg_10'], last[t + '_metric/ndcg']))


if __name__ == '__main__':
  main()
