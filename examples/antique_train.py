"""The reference's ANTIQUE text-ranking example (examples/keras/antique_kpl_din.py) on the fused
GPU step: `query_tokens` (context) and `document_tokens` (example) are bytes_list features,
mapped to ids with a vocabulary file, pooled (mean) through ONE shared embedding table, and
scored by a create_tower tower.  With --use_document_interaction 1 (the reference's default)
the pooled vectors are concatenated and run through a DocumentInteractionAttention, and the
tower scores [query_tokens | document_interaction_embedding | document_tokens]
(DINEmbeddingRankingTrainer); with 0 (the default here) the tower scores
[query_tokens | document_tokens] (EmbeddingRankingTrainer).

  python examples/antique_train.py --train_path tests/golden/antique/train_elwc.tfrecord \
      --eval_path tests/golden/antique/train_elwc.tfrecord \
      --vocab_file tests/golden/antique/vocab.txt --num_train_steps 20 \
      --use_document_interaction 1

Differences from the reference model: the tower has no input BatchNormalization (hidden BN,
ReLU and dropout as there), and a bag is cut to its first --max_query_tokens /
--max_document_tokens tokens (the decoder reports how many it cut).  An empty bag embeds to
zeros where the reference's ragged reduce_mean gives NaN.  With BN the padded items are
circularly padded before the DIN, where the reference pads after it.
"""
import argparse
import itertools
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import ranking_b200 as tfr                # noqa: E402
from ranking_b200 import data, pipeline   # noqa: E402

_LABEL = 'relevance'


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--train_path', required=True, nargs='+')
  ap.add_argument('--eval_path', required=True, nargs='+')
  ap.add_argument('--vocab_file', required=True)
  ap.add_argument('--model_dir')
  ap.add_argument('--vocab_size', type=int, default=30522,
                  help='rows of the shared embedding table')
  ap.add_argument('--embedding_dimension', type=int, default=20)
  ap.add_argument('--list_size', type=int, default=50)
  ap.add_argument('--max_query_tokens', type=int, default=16)
  ap.add_argument('--max_document_tokens', type=int, default=128)
  ap.add_argument('--train_batch_size', type=int, default=16)
  ap.add_argument('--eval_batch_size', type=int, default=64)
  ap.add_argument('--num_train_steps', type=int, default=15000)
  ap.add_argument('--learning_rate', type=float, default=0.005)
  ap.add_argument('--hidden_layer_dims', default='64,32')
  ap.add_argument('--use_batch_norm', type=int, default=1)
  ap.add_argument('--batch_normalization_moment', type=float, default=0.99)
  ap.add_argument('--dropout_rate', type=float, default=0.5)
  ap.add_argument('--loss', default='approx_ndcg_loss')
  ap.add_argument('--use_document_interaction', type=int, default=0,
                  help='1: a DocumentInteractionAttention over the pooled features')
  ap.add_argument('--num_attention_heads', type=int, default=1)
  ap.add_argument('--head_size', type=int, default=128)
  ap.add_argument('--num_attention_layers', type=int, default=1)
  ap.add_argument('--din_precision', choices=('fp32', 'tf32'), default='fp32',
                  help='DocumentInteractionAttention precision: fp32, or tf32 tensor cores')
  args = ap.parse_args()

  vocab = data.Vocabulary.from_file(args.vocab_file)
  if vocab.num_ids > args.vocab_size:
    raise SystemExit('the vocabulary has %d tokens, the table %d rows' %
                     (vocab.num_ids, args.vocab_size))
  spec = {'context': {'query_tokens': (args.max_query_tokens, vocab)},
          'example': {'document_tokens': (args.max_document_tokens, vocab)}}
  label_spec = {_LABEL: (1, -1)}

  def batches(paths, batch_size):
    return data.elwc_batches(paths, batch_size, args.list_size, None, label_spec, _LABEL,
                             drop_remainder=False, token_feature_spec=spec)

  e = args.embedding_dimension
  din_dim = args.head_size if args.use_document_interaction else 0
  shared = tfr.keras.layers.TokenEmbedding(args.vocab_size, e, combiner='mean', seed=1234)
  tower = tfr.keras.layers.create_tower(
      [int(h) for h in args.hidden_layer_dims.split(',')], 1, activation='relu',
      use_batch_norm=bool(args.use_batch_norm),
      batch_norm_moment=args.batch_normalization_moment, dropout=args.dropout_rate,
      input_dim=2 * e + din_dim, precision='tf32x3', seed=1234)
  tables = {'shared': shared}
  features = {'context': {'query_tokens': 'shared'}, 'example': {'document_tokens': 'shared'}}
  kw = dict(optimizer='adagrad', learning_rate=args.learning_rate)
  din = None
  if args.use_document_interaction:
    din = tfr.keras.layers.DocumentInteractionAttention(
        args.num_attention_heads, args.head_size, args.num_attention_layers,
        dropout=args.dropout_rate, seed=1234, precision=args.din_precision)
    trainer = tfr.train.DINEmbeddingRankingTrainer(
        tables, features, din, tower, tfr.keras.losses.get(args.loss), **kw)
  else:
    trainer = tfr.train.EmbeddingRankingTrainer(
        tables, features, tower, tfr.keras.losses.get(args.loss), **kw)
  train = itertools.chain.from_iterable(
      batches(args.train_path, args.train_batch_size) for _ in itertools.count())
  step, loss = pipeline.fit(trainer, train, args.num_train_steps,
                            checkpoint_dir=args.model_dir)
  trainer.check_ids()
  tower.eval()
  if din is not None:
    din.eval()
  metrics = pipeline.evaluate(trainer, batches(args.eval_path, args.eval_batch_size))
  print('step %d loss %.6f' % (step, loss))
  print({k: round(float(v), 6) for k, v in metrics.items()})


if __name__ == '__main__':
  main()
