"""The reference's TFR-BERT recipe (examples/keras/tfrbert_antique_train_config.yaml) on the
fused GPU step: softmax loss over lists of 10 (query, document) sequences of 64 tokens, a BERT
encoder (BERT-base by default; sizes by flag) with Dropout(0.1) + Dense(1) on the pooled output,
AdamW (weight decay 0.01, LayerNorm and biases excluded) at 3e-5 with linear warmup over the
first tenth of the steps and linear decay to 0, and the best checkpoint by MAP.

  python examples/tfrbert_train.py --train antique_train_seq_64_elwc.tfrecord \\
      --valid antique_test_seq_64_elwc.tfrecord --model_dir /tmp/tfrbert

Input is ELWC with example features `input_ids`, `input_mask`, `segment_ids` (int64,
seq_length each) and an int `relevance` label (--label).  The encoder starts from its
initialisation, or, as the recipe fine-tunes, from a pretrained BERT (--init_checkpoint: a TF2
BertEncoder checkpoint or a Hugging Face model; sizes from --bert_config_file or the
config.json beside it).  --gradient_clip_norm 1.0 is the recipe's AdamWeightDecay clipping.
--precision fp16 is the recipe's mixed_float16, the policy it names for GPUs, with dynamic
loss scaling (--loss_scale).
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ranking_b200 import pipeline, train        # noqa: E402
from ranking_b200.extension import tfrbert      # noqa: E402
from ranking_b200.keras import losses           # noqa: E402


def main():
  ap = argparse.ArgumentParser(description=__doc__.split('\n\n')[0])
  ap.add_argument('--train', required=True, nargs='+')
  ap.add_argument('--valid', nargs='+')
  ap.add_argument('--model_dir', required=True)
  ap.add_argument('--label', default='relevance')
  ap.add_argument('--batch_size', type=int, default=4)
  ap.add_argument('--list_size', type=int, default=10)
  ap.add_argument('--seq_length', type=int, default=64)
  ap.add_argument('--train_steps', type=int, default=10000)
  ap.add_argument('--warmup_steps', type=int, default=None,
                  help='default: a tenth of --train_steps')
  ap.add_argument('--steps_per_loop', type=int, default=50,
                  help='steps between validation and checkpoints')
  ap.add_argument('--learning_rate', type=float, default=3e-5)
  ap.add_argument('--weight_decay_rate', type=float, default=0.01)
  ap.add_argument('--dropout_rate', type=float, default=0.1)
  # encoder sizes: default BERT-base; with --bert_config_file / --init_checkpoint they come
  # from the config, and a size flag that disagrees with it is an error
  ap.add_argument('--vocab_size', type=int, default=None, help='default 30522')
  ap.add_argument('--hidden_size', type=int, default=None, help='default 768')
  ap.add_argument('--num_layers', type=int, default=None, help='default 12')
  ap.add_argument('--num_heads', type=int, default=None, help='default 12')
  ap.add_argument('--intermediate_size', type=int, default=None, help='default 3072')
  ap.add_argument('--init_checkpoint', default=None,
                  help='pretrained encoder: TF2 BertEncoder checkpoint prefix, Hugging Face '
                       'model.safetensors / pytorch_model.bin, or a directory holding one')
  ap.add_argument('--bert_config_file', default=None,
                  help='BERT / Hugging Face config.json (default: the one beside '
                       '--init_checkpoint)')
  ap.add_argument('--gradient_clip_norm', type=float, default=0.0,
                  help='clip gradients to this global norm before AdamW; 0 = off (the '
                       "reference recipe's AdamWeightDecay uses 1.0)")
  # the reference's runtime.mixed_precision_dtype: bf16 is 'mixed_bfloat16' (fp32 variables,
  # bf16 compute), fp16 is 'mixed_float16' (fp32 variables, fp16 compute, loss scaling)
  ap.add_argument('--precision', choices=('fp32', 'tf32', 'bf16', 'fp16'), default='fp32',
                  help="fp16 = the reference's mixed_float16, bf16 = its mixed_bfloat16")
  ap.add_argument('--loss_scale', default='dynamic',
                  help="fp16 only: 'dynamic' (Keras' dynamic loss scale, from 2^15) or a "
                       'fixed scale')
  ap.add_argument('--seed', type=int, default=1234)
  args = ap.parse_args()
  if args.gradient_clip_norm < 0:
    ap.error('--gradient_clip_norm must be >= 0')
  loss_scale = args.loss_scale
  if loss_scale != 'dynamic':
    try:
      loss_scale = float(loss_scale)
    except ValueError:
      ap.error("--loss_scale must be 'dynamic' or a number")

  sizes = {'vocab_size': args.vocab_size, 'hidden_size': args.hidden_size,
           'num_layers': args.num_layers, 'num_attention_heads': args.num_heads,
           'intermediate_size': args.intermediate_size}
  config_file = args.bert_config_file
  if config_file is None and args.init_checkpoint is not None:
    config_file = tfrbert.config_beside(args.init_checkpoint)
    if config_file is None:
      ap.error('no config.json beside --init_checkpoint; pass --bert_config_file')
  if config_file is not None:
    cfg = tfrbert.BertEncoderConfig.from_json(config_file)
    for field, value in sizes.items():
      if value is not None and value != getattr(cfg, field):
        ap.error('--%s %d disagrees with %s (%s %d)' %
                 (field if field != 'num_attention_heads' else 'num_heads', value,
                  config_file, field, getattr(cfg, field)))
  else:
    cfg = tfrbert.BertEncoderConfig(**{k: v for k, v in sizes.items() if v is not None})
  # the recipe's dropout rates (BERT's 0.1 by default) replace the config file's
  cfg.hidden_dropout_prob = cfg.attention_dropout_prob = args.dropout_rate
  encoder = tfrbert.BertEncoder(cfg, seed=args.seed, precision=args.precision)
  if args.init_checkpoint is not None:
    encoder.load_checkpoint(args.init_checkpoint)
  scorer = tfrbert.TFRBertScorer(encoder, bert_output_dropout=args.dropout_rate)
  warmup = args.train_steps // 10 if args.warmup_steps is None else args.warmup_steps
  schedule = train.PolynomialWarmUp(args.learning_rate, args.train_steps, warmup)
  trainer = tfrbert.TFRBertRankingTrainer(scorer, losses.get('softmax_loss'),
                                          learning_rate=schedule,
                                          weight_decay_rate=args.weight_decay_rate,
                                          gradient_clip_norm=args.gradient_clip_norm or None,
                                          loss_scale=loss_scale)

  def batches(paths, drop_remainder=True):
    return tfrbert.tfrbert_batches(paths, args.batch_size, args.list_size, args.seq_length,
                                   vocab_size=cfg.vocab_size,
                                   type_vocab_size=cfg.type_vocab_size,
                                   label_feature=args.label, drop_remainder=drop_remainder)

  def endless():
    while True:
      yield from batches(args.train)

  ckpt_dir = os.path.join(args.model_dir, 'ckpt')
  best_dir = os.path.join(args.model_dir, 'best_ckpt')
  train_it = endless()
  best = None
  step = 0
  while step < args.train_steps:
    target = min(step + args.steps_per_loop, args.train_steps)
    step, loss = pipeline.fit(trainer, train_it, target, checkpoint_dir=ckpt_dir,
                              steps_per_checkpoint=args.steps_per_loop, log_fn=print)
    msg = 'step %d loss %.6f' % (step, loss if loss is not None else float('nan'))
    if args.valid:
      logs = pipeline.evaluate(trainer, batches(args.valid, drop_remainder=False))
      msg += ' MAP %.4f NDCG %.4f' % (logs['metric/map'], logs['metric/ndcg'])
      if best is None or logs['metric/map'] > best:
        best = logs['metric/map']
        os.makedirs(best_dir, exist_ok=True)
        pipeline.save_checkpoint(trainer, os.path.join(best_dir, 'ckpt.pt'), step)
    print(msg, flush=True)
  trainer.check_ids()


if __name__ == '__main__':
  main()
