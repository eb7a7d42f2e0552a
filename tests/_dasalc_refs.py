"""fp64 restatement of DASALC (research/dasalc.py:116-201; the contract of K13 in
include/tfr_b200.h), autograd-able.  Random draws are replayed from the documented counter
hashes (oracle/din.py's `uniform`).  Test infrastructure only."""
import numpy as np
import torch

from oracle import din as odin

EPS = 1e-3


def transform(x, cutoff=30.0):
  """clip(sign(x) log1p(|x|), -cutoff, cutoff)."""
  x = torch.as_tensor(x, dtype=torch.float64)
  return torch.clamp(torch.sign(x) * torch.log1p(x.abs()), -cutoff, cutoff)


def param_shapes(d, w, h):
  return [('w1', (d, w)), ('b1', (w,)), ('w2', (w, w)), ('b2', (w,)), ('wt', (w, w)),
          ('bt', (w,)), ('wc', (h, w)), ('bc', (w,)), ('wo', (w,)), ('bo', (1,)),
          ('g_in', (d,)), ('be_in', (d,)), ('g1', (w,)), ('be1', (w,)), ('g2', (w,)),
          ('be2', (w,)), ('gc', (h,)), ('bec', (h,))]


def state_shapes(d, w, h):
  return [(name, width) for name, width in (('in', d), ('1', w), ('2', w), ('c', h))]


def unflatten(flat, d, w, h):
  p, off = {}, 0
  for name, shape in param_shapes(d, w, h):
    n = int(np.prod(shape))
    p[name] = flat[off:off + n].reshape(shape)
    off += n
  assert off == flat.numel(), (off, flat.numel())
  return p


def draws(seed, m, d, w, rate, sigma):
  """(keep1, keep2, noise, keep_cross) of one training call; None where nothing is drawn."""
  k1 = k2 = kx = noise = None
  if rate > 0:
    k1, k2, kx = [torch.from_numpy(~(odin.uniform(seed, site, m * w) < np.float32(rate)))
                  .reshape(m, w) for site in (1, 2, 4)]
  if sigma > 0:
    u = odin.uniform(seed, 3, 2 * m * d).astype(np.float64).reshape(-1, 2)
    g = np.sqrt(-2.0 * np.log(1.0 - u[:, 0])) * np.cos(2.0 * np.pi * u[:, 1])
    noise = torch.from_numpy(sigma * g.reshape(m, d))
  return k1, k2, noise, kx


def _bn(x, gamma, beta, mean_var, training, stats):
  if training:
    mean = x.mean(0)
    var = ((x - mean) ** 2).mean(0)
    stats.append((mean.detach(), var.detach()))
  else:
    mean, var = mean_var
  return (x - mean) / torch.sqrt(var + EPS) * gamma + beta


def forward(x, e, flat, d, w, h, state=None, training=False, rate=0.0, sigma=0.0, seed=0,
            mask=None):
  """x [M, D] (transformed features), e [M, h], flat (fp64) -> (scores [M], batch stats).
  `state` is the bn_state vector (used in inference).  Batch stats: [(mean, var)] for
  BN_in, BN_1, BN_2, BN_c in training."""
  m = x.shape[0]
  p = unflatten(flat, d, w, h)
  moving = {}
  if state is not None:
    off = 0
    for name, width in state_shapes(d, w, h):
      moving[name] = (state[off:off + width].double(), state[off + width:off + 2 * width].double())
      off += 2 * width
  k1, k2, noise, kx = draws(seed, m, d, w, rate, sigma) if training else (None,) * 4
  stats = []
  a = _bn(x, p['g_in'], p['be_in'], moving.get('in'), training, stats)
  if noise is not None:
    a = a + noise
  for i, keep in ((1, k1), (2, k2)):
    a = torch.relu(a @ p['w%d' % i] + p['b%d' % i])
    a = _bn(a, p['g%d' % i], p['be%d' % i], moving.get(str(i)), training, stats)
    if keep is not None:
      a = a * keep / (1.0 - rate)
  t = a @ p['wt'] + p['bt']
  yc = _bn(e, p['gc'], p['bec'], moving.get('c'), training, stats)
  c = yc @ p['wc'] + p['bc']
  o = torch.relu(t * c + t)
  if kx is not None:
    o = o * kx / (1.0 - rate)
  s = o @ p['wo'] + p['bo']
  if mask is not None:
    s = torch.where(mask.reshape(-1), s, torch.full_like(s, float(np.log(1e-10))))
  return s, stats


def updated_state(state, stats, momentum=0.9):
  """bn_state after one training call: moving * momentum + batch * (1 - momentum)."""
  out, off = state.double().clone(), 0
  for mean, var in stats:
    width = mean.numel()
    out[off:off + width] = out[off:off + width] * momentum + mean * (1 - momentum)
    out[off + width:off + 2 * width] = out[off + width:off + 2 * width] * momentum + \
        var * (1 - momentum)
    off += 2 * width
  return out
