"""Learning to rank from position-biased clicks with click EM (Wang et al. 2018).

Graded relevance labels (a LibSVM file given by --train_path, or a seeded synthetic set)
are turned into click logs: a logging ranker orders each list, position p (0-based) is
examined with probability eta_p = (1 / (p + 1)) ** power, and an examined item is clicked
with probability P(rel) = (2^grade - 1) / (2^max_grade - 1).  Two models are trained on the
same clicks:

  * ClickEMRankingTrainer + ClickEMLoss: relevance tower and per-position examination
    propensities learned jointly;
  * RankingTrainer + SigmoidCrossEntropyLoss: the clicks taken as relevance labels;
  * with --bilinear_dim E, a third: BilinearClickRankingTrainer, a two-tower model whose
    relevance tower and position embeddings interact through a Bilinear(E, 1), scored with
    every item at position 0.

Both are evaluated with NDCG@{1,5,10} on the TRUE grades of held-out lists, and the learned
relative propensities are printed next to the planted ones.
  python examples/click_train.py [--train_path train.txt --num_features 136]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import ranking_b200 as tfr  # noqa: E402
from ranking_b200 import data, pipeline  # noqa: E402


def synthetic_grades(n_lists, list_size, num_features, seed):
  """Features N(0, 1); grade 0..4 from a noisy linear relevance score."""
  g = torch.Generator().manual_seed(seed)
  w = torch.randn(num_features, generator=g)
  w /= w.norm()
  x = torch.randn(n_lists, list_size, num_features, generator=g)
  score = x @ w + 0.3 * torch.randn(n_lists, list_size, generator=g)
  grades = torch.bucketize(score, torch.tensor([0.0, 0.8, 1.4, 2.0]))
  return x, grades.float()


def simulate_clicks(x, grades, power, seed):
  """Orders every list (padding last) by a logging ranker that scores items along a fixed
  random direction of the features, unrelated to relevance, then draws clicks from
  eta_p * P(rel)."""
  g = torch.Generator().manual_seed(seed)
  b, n, d = x.shape
  u = torch.randn(d, generator=g)
  logging = torch.where(grades >= 0, x @ u, torch.full_like(grades, -1e30))
  order = torch.argsort(logging, dim=1, descending=True, stable=True)
  x = torch.gather(x, 1, order.unsqueeze(2).expand(-1, -1, d))
  grades = torch.gather(grades, 1, order)
  top = float(grades.max().clamp(min=1))
  p_rel = (2 ** grades.clamp(min=0) - 1) / (2 ** top - 1)
  eta = (1.0 / (torch.arange(n, dtype=torch.float32) + 1)) ** power
  clicks = (torch.rand(b, n, generator=g) < eta * p_rel).float()
  clicks = torch.where(grades >= 0, clicks, torch.full_like(clicks, -1.))
  return x, grades, clicks, eta


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--train_path', default=None)
  ap.add_argument('--num_features', type=int, default=8)
  ap.add_argument('--list_size', type=int, default=10)
  ap.add_argument('--lists', type=int, default=8192, help='synthetic lists')
  ap.add_argument('--power', type=float, default=1.0)
  ap.add_argument('--batch_size', type=int, default=256)
  ap.add_argument('--epochs', type=int, default=25)
  ap.add_argument('--learning_rate', type=float, default=1.0)
  ap.add_argument('--hidden', default='', help='hidden layer widths, e.g. 64,32')
  ap.add_argument('--seed', type=int, default=0)
  ap.add_argument('--bilinear_dim', type=int, default=0,
                  help='E > 0 (at most 8) also trains a two-tower model whose relevance '
                       'tower and position embeddings of width E interact through a '
                       'Bilinear(E, 1) (BilinearClickRankingTrainer)')
  args = ap.parse_args()
  if args.train_path:
    x, grades = data.load_libsvm_data(args.train_path, args.list_size, args.num_features)[:2]
    x, grades = torch.as_tensor(x), torch.as_tensor(grades)
  else:
    x, grades = synthetic_grades(args.lists, args.list_size, args.num_features, args.seed)
  x, grades, clicks, eta = simulate_clicks(x, grades, args.power, args.seed + 1)
  n_test = max(1, x.shape[0] // 5)
  train = (x[n_test:].cuda(), clicks[n_test:].cuda())
  test = [(x[:n_test], grades[:n_test])]
  hidden = [int(h) for h in args.hidden.split(',') if h]

  def tower(units=1):
    return tfr.keras.layers.create_tower(hidden, units, activation='relu', use_batch_norm=False,
                                         dropout=0, input_dim=x.shape[2], seed=args.seed)
  em = tfr.train.ClickEMRankingTrainer(tower(), tfr.keras.losses.ClickEMLoss(),
                                       args.list_size, seed=args.seed,
                                       learning_rate=args.learning_rate)
  naive = tfr.train.RankingTrainer(tower(), tfr.keras.losses.SigmoidCrossEntropyLoss(),
                                   learning_rate=args.learning_rate)
  models = [('click_em', em), ('naive_sigmoid_ce', naive)]
  if args.bilinear_dim > 0:
    e = args.bilinear_dim
    models.append(('bilinear_two_tower', tfr.train.BilinearClickRankingTrainer(
        tower(e), tfr.keras.layers.Bilinear(e, 1, seed=args.seed),
        tfr.keras.losses.SigmoidCrossEntropyLoss(), args.list_size, seed=args.seed,
        learning_rate=args.learning_rate)))
  n_train = train[0].shape[0]
  for epoch in range(args.epochs):
    perm = torch.randperm(n_train, generator=torch.Generator().manual_seed(epoch)).cuda()
    for i in range(0, n_train - args.batch_size + 1, args.batch_size):
      idx = perm[i:i + args.batch_size]
      xb, cb = train[0][idx], train[1][idx]
      for _, tr in models:
        tr.train_step(xb, cb)
  for name, tr in models:
    res = pipeline.evaluate(tr, test)
    ndcg = {k.split('/')[-1]: float(v) for k, v in res.items()}
    print('%-17s ' % name + '  '.join('NDCG@%d %.4f' % (k, ndcg['ndcg_%d' % k])
                                       for k in (1, 5, 10)))
  learned = em.examination_propensity().cpu()
  print('position  planted eta_p/eta_0  learned')
  for p in range(args.list_size):
    print('%8d  %19.4f  %7.4f' % (p, float(eta[p] / eta[0]), float(learned[p] / learned[0])))


if __name__ == '__main__':
  main()
