"""Oracle restatement of the Bilinear layer (keras/layers.py:807-890) and of a two-tower
click training step around it:

  * bilinear(v1, v2, W, W1, W2, b): the layer's `call`, as einsums;
  * init_bilinear(E, K, seed): the layer's initialisers (RandomNormal(1/E) for W,
    RandomNormal(1/sqrt(E)) for W1 and W2, zeros for b), drawn as ranking_b200's
    keras.layers.Bilinear draws them;
  * BilinearClickTrainer: a relevance tower (scorer.tower_forward) and a position table
    [num_positions, E] whose rows interact through a Bilinear(E, 1) into the click logit
    (Yan et al., "Revisiting two tower models for unbiased learning to rank"), trained with the
    Keras SigmoidCrossEntropyLoss on the clicks, autograd and tf.keras Adagrad.

Test infrastructure only (see oracle/__init__.py).  Plain torch on the CPU; fp32 or fp64 by
the dtype of the tensors passed in.
"""
import math

import torch

from oracle import keras_losses
from oracle import scorer
from oracle import utils

LOG_EPSILON = math.log(1e-10)


def bilinear(v1, v2, W, W1, W2, b):
  """y[..., k] = sum_ij v1_i W_ijk v2_j + sum_i v1_i W1_ik + sum_j v2_j W2_jk + b_k."""
  return (torch.einsum('...i,ijk,...j->...k', v1, W, v2) + torch.einsum('...i,ik->...k', v1, W1)
          + torch.einsum('...j,jk->...k', v2, W2) + b)


def init_bilinear(E, K, seed):
  """[W [E, E, K], W1 [E, K], W2 [E, K], b [K]] (fp32)."""
  gen = torch.Generator().manual_seed(int(seed))
  w = (torch.randn(E * E * K, generator=gen, dtype=torch.float64) / E).float()
  w1 = (torch.randn(E * K, generator=gen, dtype=torch.float64) / math.sqrt(E)).float()
  w2 = (torch.randn(E * K, generator=gen, dtype=torch.float64) / math.sqrt(E)).float()
  return [w.reshape(E, E, K), w1.reshape(E, K), w2.reshape(E, K), torch.zeros(K)]


def abs_terms(v1, v2, W, W1, W2, b):
  """sum over the terms of y of their absolute values, [..., K]: the scale of y's rounding
  error."""
  return bilinear(v1.abs(), v2.abs(), W.abs(), W1.abs(), W2.abs(), b.abs())


class BilinearClickTrainer(object):
  """Relevance tower r = tower(x) [B, N, E], position embeddings p = table[position], click
  logit c = Bilinear(E, 1)((r, p)), ln(1e-10) where `mask` is False (RestoreList); Keras
  SigmoidCrossEntropyLoss on the clicks; autograd; tf.keras Adagrad over the table, the four
  bilinear weights and the tower parameters, in that order.  With BatchNormalization the padded
  slots of a list are filled circularly with its valid items before the tower."""

  def __init__(self, params, table, bil, activation='relu', use_batch_norm=False,
               bn_moving=None, learning_rate=0.001, epsilon=1e-7,
               initial_accumulator_value=0.1, reduction=keras_losses.Reduction.AUTO):
    self.params = params
    self.table = table
    self.bil = list(bil)
    self.activation = activation
    self.use_batch_norm = use_batch_norm
    self.bn_moving = bn_moving
    self.loss = keras_losses.SigmoidCrossEntropyLoss(reduction)
    self.lr = learning_rate
    self.eps = epsilon
    self.leaves = [table] + self.bil
    for w, b in zip(params['dense_w'], params['dense_b']):
      self.leaves += [w, b]
    for g, b in zip(params['bn_gamma'], params['bn_beta']):
      self.leaves += [g, b]
    for p in self.leaves:
      p.requires_grad_()
    self.accum = [torch.full_like(p, initial_accumulator_value) for p in self.leaves]

  def default_positions(self, b, n):
    p = torch.arange(n).clamp(max=self.table.shape[0] - 1)
    return p.unsqueeze(0).expand(b, n)

  def relevance(self, x, valid, training):
    """The relevance tower's embeddings [B, N, E]."""
    b, n, d = x.shape
    if self.use_batch_norm and training:
      idx, _ = utils.padded_nd_indices(valid)
      x = torch.gather(x, 1, idx.unsqueeze(2).expand(-1, -1, d))
    r = scorer.tower_forward(x.reshape(b * n, d), self.params, activation=self.activation,
                             use_batch_norm=self.use_batch_norm, training=training,
                             bn_moving=self.bn_moving)
    return r.reshape(b, n, -1)

  def logits(self, x, positions, valid, training, mask=None):
    r = self.relevance(x, valid, training)
    p = self.table[torch.as_tensor(positions, dtype=torch.int64)]
    c = bilinear(r, p, *self.bil)[..., 0]
    if mask is not None:
      c = torch.where(torch.as_tensor(mask, dtype=torch.bool), c,
                      torch.full_like(c, LOG_EPSILON))
    return c

  def train_step(self, x, clicks, positions=None, sample_weight=None, mask=None):
    b, n, _ = x.shape
    if positions is None:
      positions = self.default_positions(b, n)
    for p in self.leaves:
      p.grad = None
    valid = mask if mask is not None else clicks >= 0
    loss = self.loss(clicks, self.logits(x, positions, valid, True, mask), sample_weight)
    loss.backward()
    with torch.no_grad():
      for p, a in zip(self.leaves, self.accum):
        a.add_(p.grad * p.grad)
        p.sub_(self.lr * p.grad / (a.sqrt() + self.eps))
    return loss.detach()

  @torch.no_grad()
  def predict(self, x, serving_position=0, positions=None, mask=None):
    b, n, _ = x.shape
    if positions is None:
      positions = torch.full((b, n), serving_position, dtype=torch.int64)
    valid = torch.ones(b, n, dtype=torch.bool) if mask is None else mask
    return self.logits(x, positions, valid, False, mask)

  def flat_grad(self):
    return torch.cat([p.grad.reshape(-1) for p in self.leaves])

  def flat_params(self):
    return torch.cat([p.detach().reshape(-1) for p in self.leaves])
