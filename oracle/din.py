"""fp64 restatement of DocumentInteractionAttention (keras/layers.py:420-588; the contract of
K11 in include/tfr_b200.h), autograd-able.  Random draws are inputs: `keep_masks` /
`noise` replay the kernels' counter hashes.  Test infrastructure only."""
import math

import numpy as np
import torch


def param_shapes(d, h, heads, layers):
  """(name, shape) in the flat layout (Keras get_weights() order)."""
  hh = heads * h
  out = [('w_in', (d, h)), ('b_in', (h,))]
  for l in range(layers):
    out += [('wq%d' % l, (h, hh)), ('bq%d' % l, (hh,)), ('wk%d' % l, (h, hh)),
            ('bk%d' % l, (hh,)), ('wv%d' % l, (h, hh)), ('bv%d' % l, (hh,)),
            ('wo%d' % l, (hh, h)), ('bo%d' % l, (h,)), ('gamma%d' % l, (h,)),
            ('beta%d' % l, (h,))]
  return out


def unflatten(flat, d, h, heads, layers):
  p, off = {}, 0
  for name, shape in param_shapes(d, h, heads, layers):
    n = int(np.prod(shape))
    p[name] = flat[off:off + n].reshape(shape)
    off += n
  assert off == flat.numel(), (off, flat.numel())
  return p


def uniform(seed, site, n):
  """u(s, e) for e = 0 .. n - 1, s = seed * 0x100000001B3 + site (the tower's hash)."""
  with np.errstate(over='ignore'):
    s = np.uint64(seed) * np.uint64(0x100000001B3) + np.uint64(site)
    idx = np.arange(n, dtype=np.uint64)
    z = s + np.uint64(0x9E3779B97F4A7C15) * (idx + np.uint64(1))
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z = z ^ (z >> np.uint64(31))
  return (z >> np.uint64(40)).astype(np.float32) * np.float32(1.0 / 16777216.0)


def keep_masks(seed, b, n, heads, h, layers, rate):
  """Per layer (attention keep [B, H, N, N], output keep [B, N, h]) as bool tensors."""
  out = []
  for l in range(layers):
    a = ~(uniform(seed, 2 + 2 * l, b * heads * n * n) < np.float32(rate))
    o = ~(uniform(seed, 3 + 2 * l, b * n * h) < np.float32(rate))
    out.append((torch.from_numpy(a.reshape(b, heads, n, n)),
                torch.from_numpy(o.reshape(b, n, h))))
  return out


def noise(seed, b, n, h, stddev):
  """sigma * g [B, N, h] (Box-Muller on the uniforms 2e, 2e + 1 of site 1), fp64."""
  u = uniform(seed, 1, 2 * b * n * h).astype(np.float64).reshape(-1, 2)
  g = np.sqrt(-2.0 * np.log(1.0 - u[:, 0])) * np.cos(2.0 * np.pi * u[:, 1])
  return torch.from_numpy(stddev * g.reshape(b, n, h))


def attention_logits(x, p, l, heads, h):
  """[B, H, N_query, N_key] logits of layer l (before the mask), Keras einsum layouts."""
  q = torch.einsum('bnc,chd->bnhd', x, p['wq%d' % l].reshape(h, heads, h)) + \
      p['bq%d' % l].reshape(heads, h)
  k = torch.einsum('bnc,chd->bnhd', x, p['wk%d' % l].reshape(h, heads, h)) + \
      p['bk%d' % l].reshape(heads, h)
  q = q * (1.0 / math.sqrt(float(h)))
  return torch.einsum('bjhd,bihd->bhij', k, q)


def forward(x, list_mask, flat, heads, h, layers, rate=0.0, keeps=None, noise_add=None,
            relu_gate=None):
  """x [B, N, D] (float64), list_mask [B, N] bool or None -> [B, N, h].  `keeps` (from
  keep_masks) applies dropout at `rate`; `noise_add` [B, N, h] is added after the ReLU.
  `relu_gate` [B, N, h] ({0, 1}), when given, multiplies the input projection in place of
  its ReLU: the gate decisions of a kernel call replayed."""
  b, n, d = x.shape
  p = unflatten(flat, d, h, heads, layers)
  if list_mask is None:
    list_mask = torch.ones(b, n, dtype=torch.bool, device=x.device)
  z = x @ p['w_in'] + p['b_in']
  x = torch.relu(z) if relu_gate is None else z * relu_gate
  if noise_add is not None:
    x = x + noise_add
  to_mask = list_mask.reshape(b, 1, 1, n)
  for l in range(layers):
    logits = attention_logits(x, p, l, heads, h)
    # The adder is summed in fp32, as Keras does: a list with no valid item attends uniformly.
    logits = torch.where(to_mask, logits, (logits.float() + -1e9).double())
    prob = torch.softmax(logits, -1)
    if keeps is not None:
      prob = prob * keeps[l][0] / (1.0 - rate)
    v = torch.einsum('bnc,chd->bnhd', x, p['wv%d' % l].reshape(h, heads, h)) + \
        p['bv%d' % l].reshape(heads, h)
    o = torch.einsum('bhij,bjhd->bihd', prob, v)
    y = torch.einsum('bihd,hde->bie', o, p['wo%d' % l].reshape(heads, h, h)) + p['bo%d' % l]
    if keeps is not None:
      y = y * keeps[l][1] / (1.0 - rate)
    z = y + x
    mean = z.mean(-1, keepdim=True)
    var = ((z - mean) ** 2).mean(-1, keepdim=True)
    x = (z - mean) / torch.sqrt(var + 1e-12) * p['gamma%d' % l] + p['beta%d' % l]
  return x
