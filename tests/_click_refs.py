"""Seeded click logs for the click EM recovery tests (tests/test_golden_click_losses.py on the
CPU oracle, tests/test_click_em_gpu.py on the GPU trainer).

Items have D = 8 Gaussian features and a true relevance P(rel | x) = sigmoid(3 w.x - 1).
A logging ranker sorts every list of 10 by u.x, with u mostly orthogonal to w, and the
list is logged in that order.  A user examines position p (0-based) with probability
eta_p = 1 / (p + 1) and clicks an examined item with probability P(rel | x).  A model
trained naively on the clicks learns the logger's direction u along with w; click EM
separates the two factors."""
import math

import numpy as np
import torch

D, N = 8, 10
# training budget shared by the oracle and the GPU trainer
TRAIN_LISTS, TEST_LISTS, BATCH_LISTS, STEPS, LR = 4096, 1024, 256, 600, 1.0


def eta(n=N):
  return np.array([1.0 / (p + 1) for p in range(n)])


def _directions():
  g = np.random.default_rng(1234)
  w = g.standard_normal(D)
  w /= np.linalg.norm(w)
  u = g.standard_normal(D)
  u -= (u @ w) * w
  u /= np.linalg.norm(u)
  return w, 0.3 * w + math.sqrt(1 - 0.09) * u


def click_logs(n_lists, seed):
  """(x [L, N, D] fp32, clicks [L, N] fp32, P(rel) [L, N] fp64), lists in logged order."""
  w, u = _directions()
  g = np.random.default_rng(seed)
  x = g.standard_normal((n_lists, N, D))
  order = np.argsort(-(x @ u), axis=1, kind='stable')
  x = np.take_along_axis(x, order[..., None], axis=1)
  p_rel = 1.0 / (1.0 + np.exp(-(3.0 * (x @ w) - 1.0)))
  clicks = (g.random((n_lists, N)) < eta()[None, :] * p_rel).astype(np.float32)
  return torch.from_numpy(x.astype(np.float32)), torch.from_numpy(clicks), p_rel


def ndcg_at(scores, gains, k):
  """Mean NDCG@k with linear gains and 1 / log2(rank + 1) discounts, ties by index."""
  s = np.asarray(torch.as_tensor(scores).detach().double().cpu())
  g = np.asarray(gains, dtype=np.float64)
  disc = 1.0 / np.log2(np.arange(2, k + 2))
  top = np.argsort(-s, axis=1, kind='stable')[:, :k]
  dcg = (np.take_along_axis(g, top, axis=1) * disc).sum(1)
  ideal = (-np.sort(-g, axis=1)[:, :k] * disc).sum(1)
  return float(np.mean(np.where(ideal > 0, dcg / np.where(ideal > 0, ideal, 1), 0)))


def batches(x, clicks, steps=STEPS, batch=BATCH_LISTS):
  """The same deterministic sweep of mini-batches for every trainer."""
  n = x.shape[0]
  for s in range(steps):
    i = (s * batch) % n
    yield x[i:i + batch], clicks[i:i + batch]


def relative_propensity(p):
  p = np.asarray(torch.as_tensor(p).detach().double().cpu())
  return p / p[0]
