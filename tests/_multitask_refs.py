"""The multi-task recovery experiment shared by tests/test_golden_multitask.py (CPU oracle,
which sets the threshold) and tests/test_multitask_gpu.py (the fused trainer).

Data: examples/multitask_train.py's seeded synthetic TFRecords, decoded with
`data.elwc_multilabel_batches`.  Both labels come from the same 16 features through two
independent linear utilities: a graded relevance (utility bucketed at -1, 0, 1) and a binary
click (the other utility above 0.5).  One tower with a plane per task is trained on both, and
each task's validation NDCG@5 is compared with a one-output model trained on the other task's
labels alone: a plane that learns its own objective ranks its task far better than a model of
the other utility does.
"""
import importlib.util
import os

import numpy as np
import torch

D, LIST_SIZE, HIDDEN, BATCH, EPOCHS, LR, SEED = 16, 20, [16], 32, 3, 0.1, 3
LABELS = {'relevance': 'label', 'click': 'clicked'}
LOSSES = {'relevance': 'softmax_loss', 'click': 'sigmoid_cross_entropy_loss'}
OTHER = {'relevance': 'click', 'click': 'relevance'}
TOP_K = 5

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _example():
  spec = importlib.util.spec_from_file_location(
      'multitask_train', os.path.join(_ROOT, 'examples', 'multitask_train.py'))
  mod = importlib.util.module_from_spec(spec)
  spec.loader.exec_module(mod)
  return mod


def synthetic(directory):
  """(train batches [(x [B, N, D], {task: y})], (x_valid, {task: y_valid}))."""
  import __graft_entry__ as entry
  entry.build()
  from ranking_b200 import data
  (train, valid), ex_spec = _example().write_synthetic(directory, list_size=LIST_SIZE, dim=D)

  def load(path, b):
    return [(x, y) for x, y, _, _ in data.elwc_multilabel_batches(
        path, b, LIST_SIZE, {}, ex_spec, LABELS, drop_remainder=False, pin_memory=False)]

  vx, vy = load(valid, 1 << 20)[0]
  return load(train, BATCH), (vx, vy)


def gains(task, y):
  y = np.asarray(torch.as_tensor(y).double().cpu())
  return np.maximum(np.power(2.0, y) - 1.0, 0.0) if task == 'relevance' else np.maximum(y, 0.0)


def ndcg_at(scores, gains_, k=TOP_K):
  """Mean NDCG@k, 1 / log2(rank + 1) discounts, ties by index."""
  s = np.asarray(torch.as_tensor(scores).detach().double().cpu())
  disc = 1.0 / np.log2(np.arange(2, k + 2))
  top = np.argsort(-s, axis=1, kind='stable')[:, :k]
  dcg = (np.take_along_axis(gains_, top, axis=1) * disc).sum(1)
  ideal = (-np.sort(-gains_, axis=1)[:, :k] * disc).sum(1)
  return float(np.mean(np.where(ideal > 0, dcg / np.where(ideal > 0, ideal, 1), 0)))


def oracle_train(tasks, batches):
  """fp64 oracle composition: create_tower (oracle/scorer.py), one loss per task on its output
  column (oracle/keras_losses), their sum, autograd, Adagrad.  Returns a scoring function
  x -> [B, N, len(tasks)]."""
  from oracle import keras_losses as OL
  from oracle import scorer as OS
  cls = {'softmax_loss': OL.SoftmaxLoss, 'sigmoid_cross_entropy_loss': OL.SigmoidCrossEntropyLoss}
  params = OS.init_tower_params(D, HIDDEN, len(tasks), seed=SEED, dtype=torch.float64)
  leaves = params['dense_w'] + params['dense_b']
  for p in leaves:
    p.requires_grad_()
  accum = [torch.full_like(p, 0.1) for p in leaves]

  def score(x):
    b, n, _ = x.shape
    return OS.tower_forward(x.double().reshape(b * n, D), params,
                            activation='relu').reshape(b, n, len(tasks))

  for _ in range(EPOCHS):
    for x, ys in batches:
      for p in leaves:
        p.grad = None
      s = score(x)
      total = sum(cls[LOSSES[t]]()(ys[t].double(), s[..., i]) for i, t in enumerate(tasks))
      total.backward()
      with torch.no_grad():
        for p, a in zip(leaves, accum):
          a.add_(p.grad * p.grad)
          p.sub_(LR * p.grad / (a.sqrt() + 1e-7))
  return lambda x: score(x).detach()


def margins(multi_scores, single_scores, valid_labels):
  """{task: NDCG@k of the multi-task plane - NDCG@k of the model trained on the other task}.
  multi_scores: {task: [B, N]}; single_scores: {task the model was trained on: [B, N]}."""
  out = {}
  for t in LABELS:
    g = gains(t, valid_labels[t])
    out[t] = (ndcg_at(multi_scores[t], g), ndcg_at(single_scores[OTHER[t]], g))
  return out
