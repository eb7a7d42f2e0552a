"""fp64 restatement of DASALC (research/dasalc.py:116-201; the contract of K13 in
include/tfr_b200.h), autograd-able.  Random draws are replayed from the documented counter
hashes (oracle/din.py's `uniform`).  Test infrastructure only.

Gates.  `forward(..., gates=)` takes the three ReLUs' decisions from a kernel call instead of
deciding them itself, as tests/_tower_fp64.py does for the scorer tower: the two hidden ReLUs
from the sign words the GEMM epilogue stored, the cross ReLU from the sign of t c + t over
the kernel's own t and c (`kernel_gates`).  With the gates shared, every difference left
between kernel and reference is rounding error.

Gates taken from the kernel would also hide a kernel that gates wrongly, so each one is
judged layer by layer (`local_checks`): the reference recomputes every Dense layer in fp64
from the input the kernel itself stored for it, and the kernel's sign words must equal the
signs of those pre-activations except within one GEMM's error bound of 0, and its stored t
and c must equal the recomputed ones within the same bound.  One GEMM's bound is tight enough
to judge most gates at every width (`local_checks` reports the share it can judge); a bound
carried through the whole chain is not.  The cross gate is a function of t and c, and the
scores of t, c, w_o and b_o (`cross_scores`), which is checked at the bound of that one sum.
"""
import math
import types

import numpy as np
import torch

import _tower_fp64 as T
from oracle import din as odin

EPS = 1e-3
U24 = 2.0 ** -24


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


def draws(seed, m, d, w, rate, sigma, device=None):
  """(keep1, keep2, noise, keep_cross) of one training call; None where nothing is drawn."""
  k1 = k2 = kx = noise = None
  if rate > 0:
    k1, k2, kx = [torch.from_numpy(~(odin.uniform(seed, site, m * w) < np.float32(rate)))
                  .reshape(m, w) for site in (1, 2, 4)]
  if sigma > 0:
    u = odin.uniform(seed, 3, 2 * m * d).astype(np.float64).reshape(-1, 2)
    g = np.sqrt(-2.0 * np.log(1.0 - u[:, 0])) * np.cos(2.0 * np.pi * u[:, 1])
    noise = torch.from_numpy(sigma * g.reshape(m, d))
  return tuple(None if t is None else t.to(device) for t in (k1, k2, noise, kx))


def _bn(x, gamma, beta, mean_var, training, stats):
  if training:
    mean = x.mean(0)
    var = ((x - mean) ** 2).mean(0)
    stats.append((mean.detach(), var.detach()))
  else:
    mean, var = mean_var
  return (x - mean) / torch.sqrt(var + EPS) * gamma + beta


def _moving(state, d, w, h):
  moving = {}
  if state is not None:
    off = 0
    for name, width in state_shapes(d, w, h):
      moving[name] = (state[off:off + width].double(), state[off + width:off + 2 * width].double())
      off += 2 * width
  return moving


def forward(x, e, flat, d, w, h, state=None, training=False, rate=0.0, sigma=0.0, seed=0,
            mask=None, gates=None, pre=None):
  """x [M, D] (transformed features), e [M, h], flat (fp64) -> (scores [M], batch stats).
  `state` is the bn_state vector (used in inference).  Batch stats: [(mean, var)] for
  BN_in, BN_1, BN_2, BN_c in training.  Everything runs on x's device.

  gates: None (the ReLUs decide on the reference's own values), or {'hidden': [G_1, G_2],
  'cross': G_x}, [M, W] each, by which the three ReLUs' inputs are multiplied instead.
  pre: a list that receives {'a0', 'a1', 'a2', 'yc', 'z1', 'z2', 't', 'c', 'v'}: the inputs
  of the Dense layers W_1, W_2, W_t, W_c, the hidden ReLUs' inputs, t, c and v = t c + t, as
  live tensors of the graph."""
  m = x.shape[0]
  p = unflatten(flat, d, w, h)
  moving = {k: (a.to(x.device), b.to(x.device))
            for k, (a, b) in _moving(state, d, w, h).items()}
  k1, k2, noise, kx = draws(seed, m, d, w, rate, sigma, x.device) if training else (None,) * 4
  stats = []
  inner = {}
  a = _bn(x, p['g_in'], p['be_in'], moving.get('in'), training, stats)
  if noise is not None:
    a = a + noise
  for i, keep in ((1, k1), (2, k2)):
    inner['a%d' % (i - 1)] = a
    z = a @ p['w%d' % i] + p['b%d' % i]
    inner['z%d' % i] = z
    a = torch.relu(z) if gates is None else z * gates['hidden'][i - 1]
    a = _bn(a, p['g%d' % i], p['be%d' % i], moving.get(str(i)), training, stats)
    if keep is not None:
      a = a * keep / (1.0 - rate)
  t = a @ p['wt'] + p['bt']
  yc = _bn(e, p['gc'], p['bec'], moving.get('c'), training, stats)
  c = yc @ p['wc'] + p['bc']
  v = t * c + t
  inner.update(a2=a, yc=yc, t=t, c=c, v=v)
  o = torch.relu(v) if gates is None else v * gates['cross']
  if kx is not None:
    o = o * kx / (1.0 - rate)
  s = o @ p['wo'] + p['bo']
  if mask is not None:
    s = torch.where(mask.reshape(-1).to(s.device), s, torch.full_like(s, float(np.log(1e-10))))
  if pre is not None:
    pre.append(inner)
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


def param_count(d, w, h):
  return sum(int(np.prod(shape)) for _, shape in param_shapes(d, w, h))


def blocks(flat, d, w, h):
  """{name: 1-D view} of a flat parameter (or gradient) vector."""
  out, off = {}, 0
  for name, shape in param_shapes(d, w, h):
    n = int(np.prod(shape))
    out[name] = flat[off:off + n]
    off += n
  return out


def block_errors(got, want, d, w, h):
  """{name: relative L2 error} of every parameter block; a block whose reference is exactly 0
  counts its absolute error (so it must be 0 too)."""
  out = {}
  g, r = blocks(got.double().reshape(-1), d, w, h), blocks(want.double().reshape(-1), d, w, h)
  for name in g:
    a, b = g[name], r[name].to(g[name].device)
    out[name] = float((a - b).norm() / max(float(b.norm()), 1e-300)) if float(b.norm()) > 0 \
        else float((a - b).norm())
  return out


# ---------------------------------------------------------------- the kernel's plan ---
def _al64(n):
  return (n + 63) // 64 * 64


def _up128(n):
  return (n + 127) // 128 * 128


def dw_splits(d, w, m, sms):
  """make_plan's dW row splits (csrc/dasalc.cu): the tower's rule, about one split per SM,
  capped so the split-K partials stay within 64 M floats.  (rows_per_split, splits, capped)."""
  per_split = _up128(max(d, w)) * _up128(w)
  per = (m + sms - 1) // sms
  rows = 256 if per < 256 else _up128(per)
  max_splits = max(1, (64 << 20) // per_split)
  capped = m > 0 and (m + rows - 1) // rows > max_splits
  if capped:
    rows = _up128((m + max_splits - 1) // max_splits)
  return rows, ((m + rows - 1) // rows if m > 0 else 1), capped


def cross_layout(w):
  """cross_bwd_kernel's layout for width w (cross_cw): (cw, row lanes rl, the most column
  quads one thread owns, whether some quad lanes of a row lane are idle)."""
  w4 = w // 4
  cw = 32
  while cw < w4 and cw < 256:
    cw <<= 1
  return cw, 256 // cw, -(-w4 // cw), w4 % cw != 0


def workspace_layout(d, w, h, m, sms):
  """Float offsets of the workspace regions the gated reference reads (make_plan,
  csrc/dasalc.cu), from the first 256-byte boundary of the buffer: 'act' [2] (the hidden
  layers' outputs, the inputs of W_2 and W_t), 'bits' [2] (sign words [ceil(W / 32), M] of the
  hidden ReLUs), 'xin' (the input BN's output, the input of W_1), 'cxin' (BN_c(E), the input
  of W_c), 't', 'cc', and 'total' (ws_floats)."""
  n_params = param_count(d, w, h)
  lay, o = {'act': [], 'bits': []}, 0
  for _ in range(2):
    lay['act'].append(o)
    o += 2 * _al64(m * w)                    # activations, normalised pre-activations
    lay['bits'].append(o)
    o += _al64(m * ((w + 31) // 32)) + _al64(2 * w)
  lay['xin'] = o
  o += _al64(m * d) + _al64(2 * d)           # input BN output, its statistics
  max_bn = max(d, w, h)
  red_blocks = (m + 255) // 256 if m > 0 else 1
  o += red_blocks * _al64(2 * max_bn) + _al64(2 * max_bn)
  _, splits, _ = dw_splits(d, w, m, sms)
  o += splits * _al64(_up128(max(d, w)) * _up128(w))   # split-K partials
  o += 4 * _al64(n_params)                   # split weight copies
  o += splits * _al64(w)                     # column-sum tiles
  lay['cxin'] = o
  o += 2 * _al64(m * h) + _al64(2 * h)       # context BN output, its statistics, E copy
  lay['t'] = o
  o += _al64(m * w)
  lay['cc'] = o
  o += 5 * _al64(m * w) + _al64(m * d) + _al64(m * h)   # c, dt, dc, dh x2; da0; dyc
  xblocks = (m + 31) // 32 if m > 0 else 1
  o += xblocks * _al64((w + 1 + 3) // 4 * 4 + 2 * w)
  lay['total'] = o
  return lay


def kernel_gates(ws, d, w, h, m, sms):
  """What one kernel call stored, from its workspace (a uint8 tensor), as fp64 on the
  workspace's device: 'hidden' [G_1, G_2] from the sign words (bit n & 31 of word
  [(n >> 5) M + m]), 'cross' = [t c + t > 0] over the kernel's t and c (an fp32 fma rounds to
  the sign of the exact value, which fp64 holds exactly here), and the stored Dense inputs
  and outputs 'a0', 'a1', 'a2', 'yc', 't', 'c' (the names of forward's `pre`)."""
  lay = workspace_layout(d, w, h, m, sms)
  base = (-ws.data_ptr()) % 256
  f = ws[base:base + (ws.numel() - base) // 4 * 4].view(torch.float32)
  i = ws[base:base + (ws.numel() - base) // 4 * 4].view(torch.int32)
  nw = (w + 31) // 32
  shifts = torch.arange(32, device=ws.device, dtype=torch.int32)
  hidden = []
  for off in lay['bits']:
    words = i[off:off + nw * m].view(nw, m)
    bits = (words.unsqueeze(-1) >> shifts) & 1                  # [nw, M, 32]
    hidden.append(bits.permute(1, 0, 2).reshape(m, nw * 32)[:, :w].double())
  region = lambda off, n: f[off:off + m * n].view(m, n).double()
  out = {'hidden': hidden, 'a0': region(lay['xin'], d), 'a1': region(lay['act'][0], w),
         'a2': region(lay['act'][1], w), 'yc': region(lay['cxin'], h),
         't': region(lay['t'], w), 'c': region(lay['cc'], w)}
  out['cross'] = (out['t'] * out['c'] + out['t'] > 0).double()
  return out


def gate_ratio(gate, value, band):
  """How far a gate is from admissible: max |value| / band over the elements where the gate
  differs from [value > 0] (0 when none does).  Above 1 the gate is wrong."""
  bad = (gate > 0) != (value > 0)
  if not bool(bad.any()):
    return 0.0
  r = (value.abs() / band)[bad]
  return float(torch.nan_to_num(r, nan=math.inf).max())


def _gemm_u(precision, k):
  """u of one Dense layer of depth k on the GEMM engine (tests/_tower_fp64.py's accounting:
  u_p per product, (per_k k + 1) accumulator additions, the bias epilogue included)."""
  u_p, u_acc, per_k = T.PRECISIONS[precision]
  return u_p + (per_k * k + 1) * u_acc


def local_checks(stored, flat, d, w, h, precision='tf32x3'):
  """Each Dense layer of one kernel call recomputed in fp64 from the input the kernel stored
  for it, against what the kernel made of it.  `stored` holds kernel_gates' entries (or a
  stand-in's).  With Y = A W + b and its bound B = C u_gemm(k) (|A| |W| + |b|):

    'relu1', 'relu2'  gate_ratio of the sign words against Y_1, Y_2 (above 1: a gate the
                      stored input cannot explain)
    't', 'c'          max |stored - Y| / B (0 where equal)
    'judged1', 'judged2'  the share of ReLU gates with |Y| > B, i.e. the share a wrong gate
                      would be caught in

  Only one GEMM's rounding separates the kernel's value from Y, so the bound is that GEMM's:
  whatever came before is the same stored input on both sides."""
  dev = stored['t'].device
  p = {k: v.detach().to(dev) for k, v in unflatten(flat.detach(), d, w, h).items()}
  out = {}

  def dense(a, wname, bname, k):
    y = a @ p[wname] + p[bname]
    return y, T.C * _gemm_u(precision, k) * (a.abs() @ p[wname].abs() + p[bname].abs())

  for i, (a, k) in enumerate(((stored['a0'], d), (stored['a1'], w))):
    y, band = dense(a, 'w%d' % (i + 1), 'b%d' % (i + 1), k)
    out['relu%d' % (i + 1)] = gate_ratio(stored['hidden'][i].to(dev), y, band)
    out['judged%d' % (i + 1)] = float((y.abs() > band).double().mean()) if y.numel() else 1.0
  for name, a, wname, bname, k in (('t', stored['a2'], 'wt', 'bt', w),
                                   ('c', stored['yc'], 'wc', 'bc', h)):
    y, band = dense(a, wname, bname, k)
    err = (stored[name] - y).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / band)
    out[name] = float(torch.nan_to_num(r, nan=math.inf).max()) if r.numel() else 0.0
  return out


def cross_scores(t, c, flat, d, w, h, keep=None, rate=0.0):
  """The scores cross_fwd_kernel must make of the t and c it was given, in fp64, and the
  bound of that one sum: s = sum_j o_j w_o[j] + b_o with o = drop(relu(t c + t)).  The kernel
  forms each o_j with an fma, a max and the dropout scale (3 roundings), sums W / 32 of them in
  order per lane (at most W / 32 + 4), then 5 shuffle additions and b_o:
  C 2^-24 ((W / 32 + 14) sum_j |o_j w_o[j]|
  + |b_o|).  keep: the replayed cross dropout stream [M, W] (training)."""
  p = {k: v.detach().to(t.device) for k, v in unflatten(flat.detach(), d, w, h).items()}
  o = torch.relu(t * c + t)
  if keep is not None:
    o = o * keep.to(t.device) / (1.0 - rate)
  s = o @ p['wo'] + p['bo']
  bound = T.C * U24 * ((w // 32 + 14) * (o.abs() @ p['wo'].abs()) + p['bo'].abs())
  return s, bound
