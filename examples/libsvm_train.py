"""Training on LibSVM ranking files with the fused GPU step: the workflow of
examples/tf_ranking_libsvm.py (hidden 256-128-64, pairwise_logistic_loss, Adagrad,
list_size 100, 136 features) through `ranking_b200`.

  python examples/libsvm_train.py --train_path train.txt --vali_path vali.txt \
      --output_dir /tmp/out --num_train_steps 1000

`--scorer gam` trains the neural additive model of examples/tf_ranking_canned_gam.py
instead: one tower per scalar feature (`--hidden_layer_dims 16,8` for that recipe), relu,
batch norm and `--dropout_rate`; the loss still comes from `--loss`.

`--scorer din` adds the listwise context of examples/keras/antique_kpl_din.py: a
DocumentInteractionAttention embedding (`--num_heads`, `--head_size`, `--num_layers`, dropout
`--dropout_rate`) of every item's features becomes an extra input block of the tower, which
then has hidden batch norm but no input batch norm.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import ranking_b200 as tfr          # noqa: E402
from ranking_b200 import data, pipeline   # noqa: E402


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--train_path', required=True)
  ap.add_argument('--vali_path')
  ap.add_argument('--output_dir')
  ap.add_argument('--train_batch_size', type=int, default=32)
  ap.add_argument('--num_train_steps', type=int, default=100000)
  ap.add_argument('--learning_rate', type=float, default=0.01)
  ap.add_argument('--dropout_rate', type=float, default=0.5)
  ap.add_argument('--hidden_layer_dims', default='256,128,64')
  ap.add_argument('--num_features', type=int, default=136)
  ap.add_argument('--list_size', type=int, default=100)
  ap.add_argument('--loss', default='pairwise_logistic_loss')
  ap.add_argument('--precision', default='tf32x3')
  ap.add_argument('--scorer', choices=('dnn', 'gam', 'din'), default='dnn')
  ap.add_argument('--num_heads', type=int, default=2)
  ap.add_argument('--head_size', type=int, default=64)
  ap.add_argument('--num_layers', type=int, default=2)
  ap.add_argument('--din_precision', choices=('fp32', 'tf32'), default='fp32',
                  help='DocumentInteractionAttention precision: fp32, or tf32 tensor cores')
  args = ap.parse_args()

  hidden = [int(h) for h in args.hidden_layer_dims.split(',')]
  x, y, info = data.load_libsvm_data(args.train_path, args.list_size, args.num_features)
  print('train:', info)
  loss = tfr.keras.losses.get(args.loss)
  if args.scorer == 'gam':
    tower = tfr.keras.layers.GAMLayer(args.num_features, hidden, activation='relu',
                                      use_batch_norm=True, dropout=args.dropout_rate)
    trainer = tfr.train.GAMRankingTrainer(tower, loss, [1] * args.num_features,
                                          optimizer='adagrad',
                                          learning_rate=args.learning_rate)
  elif args.scorer == 'din':
    din = tfr.keras.layers.DocumentInteractionAttention(
        args.num_heads, args.head_size, args.num_layers, dropout=args.dropout_rate,
        precision=args.din_precision)
    din.build(args.num_features)
    tower = tfr.keras.layers.create_tower(
        hidden, 1, activation='relu', use_batch_norm=True, dropout=args.dropout_rate,
        input_dim=args.num_features + args.head_size, precision=args.precision)
    trainer = tfr.train.DINRankingTrainer(din, tower, loss, optimizer='adagrad',
                                          learning_rate=args.learning_rate)
  else:
    tower = tfr.keras.layers.create_tower(
        hidden, 1, activation='relu', use_batch_norm=True, input_batch_norm=True,
        dropout=args.dropout_rate, input_dim=args.num_features, precision=args.precision)
    trainer = tfr.train.RankingTrainer(tower, loss, optimizer='adagrad',
                                       learning_rate=args.learning_rate)
  eval_fn = None
  if args.vali_path:
    vx, vy, vinfo = data.load_libsvm_data(args.vali_path, args.list_size,
                                          args.num_features)
    print('vali:', vinfo)
    eval_fn = lambda: data.batch_iterator(vx, vy, args.train_batch_size,
                                          drop_remainder=False)
  batches = data.batch_iterator(x, y, args.train_batch_size, shuffle=True, repeat=True)
  step, loss = pipeline.fit(trainer, batches, args.num_train_steps,
                            checkpoint_dir=args.output_dir, eval_batches_fn=eval_fn)
  print('finished at step', step, 'loss', loss)
  if eval_fn is not None:
    tower.eval()
    if args.scorer == 'din':
      din.eval()
    print(pipeline.evaluate(trainer, eval_fn()))


if __name__ == '__main__':
  main()
