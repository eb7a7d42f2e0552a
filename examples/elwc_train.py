"""Training on TFRecord files of ExampleListWithContext protos (the reference's
`tfr.keras.pipeline` input format) with the fused GPU step.

  python examples/elwc_train.py --train_path train.tfrecord --num_features 136 \
      --feature_name f --label_name utility --output_dir /tmp/out

The native decoder (`tfr_elwc_parse`) fills pinned host tensors; `RankingTrainer.train_step`
takes it from there.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import ranking_b200 as tfr          # noqa: E402
from ranking_b200 import data, pipeline   # noqa: E402


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--train_path', required=True, nargs='+')
  ap.add_argument('--output_dir')
  ap.add_argument('--feature_name', default='f',
                  help='dense float example feature holding the item vector')
  ap.add_argument('--label_name', default='utility')
  ap.add_argument('--num_features', type=int, default=136)
  ap.add_argument('--list_size', type=int, default=200)
  ap.add_argument('--batch_size', type=int, default=1024)
  ap.add_argument('--num_train_steps', type=int, default=1000)
  ap.add_argument('--learning_rate', type=float, default=0.05)
  ap.add_argument('--hidden_layer_dims', default='256,128,64')
  ap.add_argument('--loss', default='approx_ndcg_loss')
  ap.add_argument('--precision', default='tf32x3')
  args = ap.parse_args()

  hidden = [int(h) for h in args.hidden_layer_dims.split(',')]
  tower = tfr.keras.layers.create_tower(
      hidden, 1, activation='relu', use_batch_norm=False, dropout=0.0,
      input_dim=args.num_features, precision=args.precision)
  trainer = tfr.train.RankingTrainer(tower, tfr.keras.losses.get(args.loss),
                                     optimizer='adagrad', learning_rate=args.learning_rate)

  def batches():
    while True:
      yield from data.elwc_batches(
          args.train_path, args.batch_size, args.list_size, context_feature_spec=None,
          example_feature_spec={args.feature_name: (args.num_features, 0.0),
                                args.label_name: (1, -1.0)},
          label_feature=args.label_name)

  step, loss = pipeline.fit(trainer, batches(), args.num_train_steps,
                            checkpoint_dir=args.output_dir)
  print('finished at step', step, 'loss', loss)


if __name__ == '__main__':
  main()
