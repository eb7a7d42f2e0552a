"""The reference's DASALC recipe (research/dasalc.py) on the fused GPU step: numeric features
through log1p_cutoff, a DocumentInteractionAttention over the list, and the latent-cross
scorer (DASALCRankingTrainer).  The defaults are the reference's Web30K settings; its
docstring's other two are reachable through the flags:

  Yahoo    --batch_size 256 --learning_rate 0.0001 --dropout_rate 0.7
           --input_noise_stddev 4.5 --num_attention_heads 4
  Istella  --hidden_layer_dims 3072 --input_noise_stddev 0.2 --num_attention_layers 2

  python examples/dasalc_train.py \
      --train_path tests/golden/numerical/train_numerical_elwc.tfrecord \
      --eval_path tests/golden/numerical/vali_numerical_elwc.tfrecord --num_train_steps 300

Input is numerical ELWC (example features custom_features_1..D, int label `utility`) or, with
--data_format libsvm, LibSVM text files.  The paper trained with Adam; this project has no Adam
optimizer, so the step uses Adagrad (default) or SGD.
"""
import argparse
import itertools
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np                        # noqa: E402
import torch                              # noqa: E402

import ranking_b200 as tfr                # noqa: E402
from ranking_b200 import data, pipeline   # noqa: E402
from ranking_b200.research import dasalc  # noqa: E402

_LABEL = 'utility'


def main():
  ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
  ap.add_argument('--train_path', required=True, nargs='+')
  ap.add_argument('--eval_path', required=True, nargs='+')
  ap.add_argument('--data_format', choices=['elwc', 'libsvm'], default='elwc')
  ap.add_argument('--model_dir')
  ap.add_argument('--batch_size', type=int, default=128)
  ap.add_argument('--num_train_steps', type=int, default=15000)
  ap.add_argument('--num_features', type=int, default=136)
  ap.add_argument('--list_size', type=int, default=200)
  ap.add_argument('--learning_rate', type=float, default=0.001)
  ap.add_argument('--optimizer', choices=['adagrad', 'sgd'], default='adagrad',
                  help='the paper used Adam, which this project does not implement')
  ap.add_argument('--dropout_rate', type=float, default=0.4)
  ap.add_argument('--hidden_layer_dims', type=int, default=512)
  ap.add_argument('--loss', default='softmax_loss')
  ap.add_argument('--batch_norm_moment', type=float, default=0.9)
  ap.add_argument('--input_noise_stddev', type=float, default=1.5)
  ap.add_argument('--num_attention_layers', type=int, default=4)
  ap.add_argument('--num_attention_heads', type=int, default=2)
  ap.add_argument('--head_size', type=int, default=100)
  ap.add_argument('--seed', type=int, default=1234)
  ap.add_argument('--din_precision', choices=('fp32', 'tf32'), default='fp32',
                  help='DocumentInteractionAttention precision: fp32, or tf32 tensor cores')
  args = ap.parse_args()

  d = args.num_features
  if args.data_format == 'elwc':
    spec = {'custom_features_%d' % (i + 1): (1, 0.0) for i in range(d)}
    spec[_LABEL] = (1, -1.0)

    def batches(paths):
      return data.elwc_batches(paths, args.batch_size, args.list_size, None, spec, _LABEL,
                               drop_remainder=False)
  else:
    sets = {}

    def batches(paths):
      key = tuple(paths)
      if key not in sets:
        xs, ys = zip(*[data.load_libsvm_data(p, args.list_size, d) for p in paths])
        sets[key] = (torch.from_numpy(np.concatenate(xs)),
                     torch.from_numpy(np.concatenate(ys)))
      x, y = sets[key]
      return ((x[i:i + args.batch_size], y[i:i + args.batch_size])
              for i in range(0, x.shape[0], args.batch_size))

  din = tfr.keras.layers.DocumentInteractionAttention(
      args.num_attention_heads, args.head_size, args.num_attention_layers,
      dropout=args.dropout_rate, input_noise_stddev=args.input_noise_stddev, seed=args.seed,
      precision=args.din_precision)
  scorer = dasalc.DASALCScorer(d, args.hidden_layer_dims, args.head_size,
                               dropout=args.dropout_rate,
                               input_noise_stddev=args.input_noise_stddev,
                               batch_norm_moment=args.batch_norm_moment, seed=args.seed)
  trainer = tfr.train.DASALCRankingTrainer(din, scorer, tfr.keras.losses.get(args.loss),
                                           optimizer=args.optimizer,
                                           learning_rate=args.learning_rate)
  train = itertools.chain.from_iterable(batches(args.train_path) for _ in itertools.count())
  step, loss = pipeline.fit(trainer, train, args.num_train_steps, checkpoint_dir=args.model_dir)
  metrics = pipeline.evaluate(trainer, batches(args.eval_path))
  print('step %d loss %.6f' % (step, loss))
  print({k: round(float(v), 6) for k, v in metrics.items()})


if __name__ == '__main__':
  main()
