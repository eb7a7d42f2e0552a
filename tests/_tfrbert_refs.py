"""fp64 reference of TFR-BERT (include/tfr_b200.h, K15) and of tfr_adamw_step, in torch, for
tests/test_tfrbert.py (CPU) and tests/test_tfrbert_gpu.py.

`forward` replays the kernels' dropout draws (oracle.din.uniform at the documented sites and
element indices) and the DIN's masking rule (logit - 1e9 for a masked key, so a sequence with no
valid token attends 1/L); gradients come from autograd over it.

Error bars (per parameter block, relative to the block's largest exact gradient; the scores
relative to their largest magnitude).  'fp32' runs every GEMM in 3xTF32 (~fp32) and the
attention core in fp32: the bar is 2e-5 on scores and 2e-4 on gradients, times the layer
count, tight enough that the erf GELU in place of the tanh one fails it.  'tf32' makes every
contraction one TF32 product; following tests/_din_tf32_refs.py a contraction of depth k
costs u(k) = u_p + k u_acc, u_p = 2^-9 + 2^-20, u_acc = 2^-23, and a quantity's bar is C = 2 times the sum of u over the contractions on its
longest path: per layer QKV, S, P~ V, Wo, W1, W2 (6) plus the pooler in the forward; the
backward adds per layer the same six and their input-side GEMMs (dO, dA, dX twice, dS, dQ /
dK / dV: 7) and the block's own dW.  With k = max(L, E, I, 3E).
"""
import math

import numpy as np
import torch

from oracle import din as odin

LN_EPS = 1e-12
U_P = 2.0 ** -9 + 2.0 ** -20
U_ACC = 2.0 ** -23
C_SAFETY = 2.0


def weight_shapes(V, E, I, NL, P, Tv):
  out = [('word', (V, E)), ('pos', (P, E)), ('type', (Tv, E)), ('ln_e_g', (E,)), ('ln_e_b', (E,))]
  for l in range(NL):
    out += [('wqkv%d' % l, (E, 3 * E)), ('bqkv%d' % l, (3 * E,)), ('wo%d' % l, (E, E)),
            ('bo%d' % l, (E,)), ('ln1_g%d' % l, (E,)), ('ln1_b%d' % l, (E,)),
            ('w1%d' % l, (E, I)), ('b1%d' % l, (I,)), ('w2%d' % l, (I, E)), ('b2%d' % l, (E,)),
            ('ln2_g%d' % l, (E,)), ('ln2_b%d' % l, (E,))]
  out += [('wp', (E, E)), ('bp', (E,)), ('ws', (E,)), ('bs', (1,))]
  return out


def param_count(V, E, I, NL, P, Tv):
  return sum(int(np.prod(s)) for _, s in weight_shapes(V, E, I, NL, P, Tv))


def unflatten(flat, V, E, I, NL, P, Tv):
  out, off = {}, 0
  for name, shape in weight_shapes(V, E, I, NL, P, Tv):
    n = int(np.prod(shape))
    out[name] = flat[off:off + n].reshape(shape)
    off += n
  assert off == flat.numel(), (off, flat.numel())
  return out


def keep(seed, site, n, rate, shape):
  """Keep factor (0 or 1 / (1 - rate)) of n draws at a site, fp64, reshaped."""
  if rate <= 0.0:
    return None
  k = ~(odin.uniform(seed, site, n) < np.float32(rate))
  return torch.from_numpy(k.astype(np.float64) / (1.0 - float(np.float32(rate)))).reshape(shape)


def layer_norm(z, g, b):
  mu = z.mean(-1, keepdim=True)
  var = ((z - mu) ** 2).mean(-1, keepdim=True)
  return (z - mu) / torch.sqrt(var + LN_EPS) * g + b


def gelu_tanh(u):
  return 0.5 * u * (1.0 + torch.tanh(math.sqrt(2.0 / math.pi) * (u + 0.044715 * u ** 3)))


def gelu_erf(u):   # the negative control
  return 0.5 * u * (1.0 + torch.erf(u / math.sqrt(2.0)))


def forward(wid, mask, tid, flat, V, E, H, I, NL, P, Tv, training=False, hdrop=0.0, adrop=0.0,
            sdrop=0.0, seed=0, gelu=gelu_tanh, mask_logits=True, probs=None):
  """scores [S] (fp64) of ids / mask / type ids [S, L] (CPU tensors) and flat params (fp64,
  may require grad).  Out-of-range ids add no row, as the kernels.  The -1e9 adder is summed
  in fp32, as the kernels (and Keras) do, so a sequence with no valid token attends 1/L while
  its logits stay below 32 in magnitude.  `probs` (a list) receives every layer's softmax."""
  S, L = wid.shape
  dh = E // H
  p = unflatten(flat, V, E, I, NL, P, Tv)
  if not training:
    hdrop = adrop = sdrop = 0.0
  wid = wid.long()
  tid = tid.long()
  wok = ((wid >= 0) & (wid < V)).unsqueeze(-1).double()
  kok = ((tid >= 0) & (tid < Tv)).unsqueeze(-1).double()
  z = (p['word'][wid.clamp(0, V - 1)] * wok + p['pos'][:L].unsqueeze(0) +
       p['type'][tid.clamp(0, Tv - 1)] * kok)
  x = layer_norm(z, p['ln_e_g'], p['ln_e_b'])
  k = keep(seed, 1, S * L * E, hdrop, (S, L, E))
  if k is not None:
    x = x * k
  to_mask = mask.reshape(S, 1, 1, L) != 0
  for l in range(NL):
    qkv = x @ p['wqkv%d' % l] + p['bqkv%d' % l]
    q, kk, v = [qkv[..., i * E:(i + 1) * E].reshape(S, L, H, dh).transpose(1, 2)
                for i in range(3)]
    logits = q @ kk.transpose(-1, -2) / math.sqrt(dh)
    if mask_logits:
      logits = torch.where(to_mask, logits, (logits.float() + -1e9).double())
    pr = torch.softmax(logits, -1)
    if probs is not None:
      probs.append(pr.detach())
    ka = keep(seed, 2 + 3 * l, S * H * L * L, adrop, (S, H, L, L))
    if ka is not None:
      pr = pr * ka
    o = (pr @ v).transpose(1, 2).reshape(S, L, E)
    y = o @ p['wo%d' % l] + p['bo%d' % l]
    k1 = keep(seed, 3 + 3 * l, S * L * E, hdrop, (S, L, E))
    if k1 is not None:
      y = y * k1
    x1 = layer_norm(y + x, p['ln1_g%d' % l], p['ln1_b%d' % l])
    a = gelu(x1 @ p['w1%d' % l] + p['b1%d' % l])
    y2 = a @ p['w2%d' % l] + p['b2%d' % l]
    k2 = keep(seed, 4 + 3 * l, S * L * E, hdrop, (S, L, E))
    if k2 is not None:
      y2 = y2 * k2
    x = layer_norm(y2 + x1, p['ln2_g%d' % l], p['ln2_b%d' % l])
  pooled = torch.tanh(x[:, 0] @ p['wp'] + p['bp'])
  ks = keep(seed, 2 + 3 * NL, S * E, sdrop, (S, E))
  if ks is not None:
    pooled = pooled * ks
  return pooled @ p['ws'] + p['bs'][0]


def adamw(p, g, m, v, step, lr, beta1=0.9, beta2=0.999, eps=1e-6, wd=0.01, decay_mask=None,
          grad_scale=1.0):
  """One tfr_adamw_step in fp64 (the header's rule); returns new (p, m, v).  The kernel
  computes in fp32: compare with a tolerance."""
  g = g * grad_scale
  m = beta1 * m + (1 - beta1) * g
  v = beta2 * v + (1 - beta2) * g * g
  dec = torch.ones_like(p) if decay_mask is None else decay_mask.double()
  p = p - lr * wd * p * dec
  step_size = lr * math.sqrt(1 - beta2 ** step) / (1 - beta1 ** step)
  p = p - step_size * m / (torch.sqrt(v) + eps)
  return p, m, v


def _u(L, E, I):
  return U_P + max(L, E, I, 3 * E) * U_ACC


def bars(precision, L, E, I, NL):
  """(score bar, gradient bar), relative (see the module docstring)."""
  if precision == 'fp32':
    return 2e-5 * NL, 2e-4 * NL
  u = _u(L, E, I)
  return C_SAFETY * (6 * NL + 1) * u, C_SAFETY * (13 * NL + 3) * u
