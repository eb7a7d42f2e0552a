"""fp64 restatement of the scorer tower (`create_tower`, csrc/mlp_simt.cu, mlp_tc.cu, mlp_norm.cu)
that takes its ReLU / dropout gates from the hidden activations the kernel stored, and a
per-element error bound for every quantity the tower returns.

Gates.  Hidden layer d of the kernel stores H_d = drop(act(BN(Z_d))) in its workspace.  The
reference keeps element (m, j) of layer d where the kernel's own backward does
(`keep_mask`, mlp_norm.cu): H_d > 0 with ReLU, H_d != 0 with identity plus dropout, always
otherwise.  A pre-activation within rounding distance of 0 therefore takes the same branch in
both.  Where the kernel keeps an element it holds fl(Y) and the reference holds Y, so every
difference left is rounding error.

Gates taken from the kernel would also hide a kernel that writes 0 where it should not (a
tile never stored, the wrong layer's mask): the reference would zero the same elements.  So
`gate_ratio` checks that every gate is admissible: it must equal the exact layer's own
decision, the sign of the ungated Y_d and the kernel's dropout stream replayed
(`dropout_keep`), except where |Y_d| is within the forward bound of 0.

Workspace layout (make_mlp_plan, csrc/capi.cu): the base is the first 256-byte boundary of
the buffer; per hidden layer d come H_d [M, n_d], then its sign words [ceil(n_d / 32), M],
each region padded to a multiple of 64 floats; with BN the normalised pre-activations follow
all of them.

Error bound.  The chain is run a second time on magnitudes: |X|, |W|, |b|, |dS|, the same
gates, and for BatchNormalization the normalised magnitudes below.  Every magnitude is an
elementwise upper bound on the absolute value of the exact quantity, so the first-order
error of a computed dot product fl(sum_k a_k b_k), whose inputs carry errors at most
u_a mag(a) and u_b mag(b), is at most

    (u_a + u_b + u_p + n u_acc) sum_k mag(a_k) mag(b_k),

with n the length of the longest chain of additions the kernel performs for that output,
u_acc the unit roundoff of the accumulator and u_p the relative error of one product:

    fp32    u_p = 0,                      u_acc = 2^-24 (FFMA, round to nearest)
    tf32x3  u_p = 3 * 2^-21, u_acc = 2^-23, n counts 3 products per k
            (hi = RN-TF32(a) leaves |lo| <= 2^-11 |a|; truncating lo to TF32 costs
            2^-21 |a|; hi*lo' + lo'*hi + dropping lo*lo <= (2 + 2^-10 + 1/2) 2^-21 |ab|;
            the tensor core's accumulator is not guaranteed to round to nearest, so its
            additions are charged a full ulp)
    tf32    u_p = 2^-9 + 2^-20,          u_acc = 2^-23 (both operands truncated to TF32:
            (1 + 2^-10)^2 - 1)
CUDA-core parts of the TF32 paths (output layer, reductions, BN passes) are charged 2^-24 per
addition.  The u of a quantity is the sum along its path: a layer's output inherits the u of
its inputs and adds its own term (`Bound`); each elementwise fp32 operation adds one 2^-24.

The dW summation of a split GEMM is rows_per_split rows inside a split plus `splits` partials,
not M.  BN reductions are at most red_rows + 256 row additions inside a block (the row lanes'
partial sums, then the lanes) plus red_blocks partials.

BatchNormalization in training couples every row through the batch statistics.  With
xhat = (Z - mu) r, r = (var + eps)^-1/2 and an error dZ <= u mag(Z), first order gives
(in training; the batch mean and variance move with Z)

    d(xhat) = r (dZ - mean(dZ) - xhat mean(xhat dZ)),

so the forward magnitude of Y = gamma xhat + beta is taken as

    mag(Y) = |gamma| r (mag(Z) + |mu| + mean(mag(Z)) + |xhat| mean(|xhat| mag(Z)))
             + |gamma| |xhat| + |beta|

(the |mu| term covers Z - mu, the |gamma||xhat| term the rounding of r, the division and the
fma), and the backward dZ = gamma r (dY - mean(dY) - xhat mean(dY xhat)) by

    mag(dZ) = |gamma| r (mag(dY) + mean(mag(dY)) + |xhat| mean(|xhat| mag(dY))
                         + mag(xhat) |mean(dY xhat)| + |xhat| mean(|dY| mag(xhat)))
              + |dZ| (1 + r mean(|xhat| mag(Z)))

where the last term is the error of r itself.  In inference the statistics are constants:
the mean terms drop out.  u of the backward then adds the forward u of the layer, because
xhat carries it.

c.  Everything above is first order: sum_k |a_k b_k| (1 + u)^n - 1 <= n u / (1 - n u), and
the magnitudes are evaluated on the exact values rather than the computed ones, which differ
by a factor 1 + u.  For u <= 0.1 both stay below 1.12; c = 2 leaves the rest for the few-ulp
rounding of rsqrtf and of the dropout scale, which are charged 4 ulps each but computed to
~2.  The bound is never widened past c = 2 anywhere in the suite.
"""
import math

import torch

C = 2.0
LOG_EPSILON = -23.025850929940457   # ln(1e-10): RestoreList's fill for masked rows
_U24 = 2.0 ** -24

# precision -> (u_p, u_acc of the tensor-core GEMMs, products per k)
PRECISIONS = {
    'fp32': (0.0, _U24, 1),
    'tf32x3': (3 * 2.0 ** -21, 2.0 ** -23, 3),
    'tf32': (2.0 ** -9 + 2.0 ** -20, 2.0 ** -23, 1),
}


class Cfg:
  """The tower options the kernel plan reads (tfr_mlp_cfg)."""

  def __init__(self, dims, relu=True, use_bn=False, input_bn=False, training=True,
               dropout=0.0, eps=1e-3, momentum=0.999):
    self.dims = list(dims)
    self.L = len(dims) - 2                  # hidden layers
    self.relu = relu
    self.use_bn = bool(use_bn) and self.L > 0
    self.input_bn = bool(input_bn)
    self.training = bool(training)
    self.dropout = float(dropout) if self.L > 0 else 0.0
    self.eps = eps
    self.momentum = momentum

  @property
  def drop_active(self):
    return self.training and self.dropout > 0

  @property
  def post(self):
    return self.use_bn or self.drop_active


class Plan:
  """The parts of make_mlp_plan (csrc/capi.cu) that decide summation lengths."""

  def __init__(self, cfg, m, sms):
    self.m, self.sms = m, sms
    per = (m + sms - 1) // sms
    self.rows_per_split = 256 if per < 256 else (per + 127) // 128 * 128
    self.splits = (m + self.rows_per_split - 1) // self.rows_per_split if m > 0 else 1
    rows = ((m + 4 * sms - 1) // (4 * sms) + 3) // 4 * 4 if m > 0 else 4
    self.out_rows = max(rows, 16)
    self.out_slots = (m + self.out_rows - 1) // self.out_rows
    self.red_rows = 256
    self.red_blocks = (m + 255) // 256 if m > 0 else 1


def hidden_activations(ws, cfg, m):
  """[H_d] (fp32 views [M, n_d]) from the uint8 workspace tensor the kernel wrote: from the
  first 256-byte boundary, per hidden layer H_d then its sign words, each padded to 64 floats."""
  up = lambda n: (n + 63) // 64 * 64
  base = (-ws.data_ptr()) % 256
  flat = ws[base:base + (ws.numel() - base) // 4 * 4].view(torch.float32)
  out, w = [], 0
  for n in cfg.dims[1:-1]:
    out.append(flat[w:w + m * n].view(m, n))
    w += up(m * n) + up(m * ((n + 31) // 32))
  return out


def dropout_keep(seed, d, m, n, p, device=None):
  """The kernel's dropout decision for hidden layer d (post_fwd_kernel, mlp_norm.cu): element i
  of [M, n] is dropped where splitmix64 of (seed * 0x100000001B3 + d + 1, i) maps below p.
  True where kept."""
  import numpy as np
  u64 = np.uint64
  layer_seed = u64((seed * 0x100000001B3 + d + 1) & 0xFFFFFFFFFFFFFFFF)
  with np.errstate(over='ignore'):
    z = layer_seed + u64(0x9E3779B97F4A7C15) * (np.arange(m * n, dtype=u64) + u64(1))
    z = (z ^ (z >> u64(30))) * u64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> u64(27))) * u64(0x94D049BB133111EB)
    z ^= z >> u64(31)
  uniform = (z >> u64(40)).astype(np.float32) * np.float32(1.0 / 16777216.0)
  return torch.from_numpy(~(uniform < np.float32(p))).reshape(m, n).to(device)


def gates_from(hidden, cfg):
  """The kernel's keep rule on its stored activations, as fp64 {0, 1}."""
  out = []
  for h in hidden:
    if cfg.relu:
      g = h > 0
    elif cfg.drop_active:
      g = h != 0
    else:
      g = torch.ones_like(h, dtype=torch.bool)
    out.append(g.double())
  return out


def _bn_fwd(z, gamma, beta, mu, var, cfg, mag_z):
  """Y = gamma xhat + beta and its magnitude; also xhat, r and mag(xhat)."""
  r = (var + cfg.eps).rsqrt()
  xh = (z - mu) * r
  t = mag_z + mu.abs()
  if cfg.training:
    t = t + mag_z.mean(0) + xh.abs() * (xh.abs() * mag_z).mean(0)
  m_xh = r * t + xh.abs()
  return gamma * xh + beta, xh, r, m_xh, gamma.abs() * m_xh + beta.abs()


def forward_backward(x, params, cfg, gates, ds, mask=None, moving=None, dtype=torch.float64):
  """The tower on fp64 copies of everything, with the kernel's gates.

  params: {'w': [W_d [in, out]], 'b': [b_d], 'gamma': [..], 'beta': [..],
           'in_gamma': .., 'in_beta': ..};  moving: {'input' | d: (mean, var)} before the call.
  Returns a dict: 'scores', 'grads' (the tower's flat gradient layout), 'dx' (no input BN,
  at least one hidden layer), 'moving' (after the call, training BN only), and per hidden
  layer 'A' (the input of Dense d), 'Y' (hidden layer d before its gate: Z_d, or BN(Z_d)) and
  'dz' (dL/dZ_d); 'mag' holds the magnitudes of the same keys.  `dtype` = torch.float32 evaluates the same chain in fp32 (a stand-in for an
  honest fp32 kernel when the bound itself is tested)."""
  f = lambda t: None if t is None else t.detach().to(dtype)
  x, ds = f(x), f(ds)
  gates = [f(g) for g in gates]
  W =[f(w) for w in params['w']]
  B = [f(b) for b in params['b']]
  G = [f(g) for g in params.get('gamma', [])]
  Be = [f(b) for b in params.get('beta', [])]
  L, O = cfg.L, cfg.dims[-1]
  scale = 1.0 / (1.0 - cfg.dropout) if cfg.drop_active else 1.0
  mom = cfg.momentum
  out = {'A': [], 'Y': [], 'dz': [], 'moving': {}}
  mg = {'A': [], 'Y': [], 'dz': [], 'moving': {}}

  def stats(v, key):
    if cfg.training:
      return v.mean(0), v.var(0, unbiased=False)
    mu, var = moving[key]
    return f(mu), f(var)

  def update_moving(key, v, mag_v):
    if not cfg.training:
      return
    mu, var = v.mean(0), v.var(0, unbiased=False)
    m0, v0 = f(moving[key][0]), f(moving[key][1])
    out['moving'][key] = (m0 * mom + mu * (1 - mom), v0 * mom + var * (1 - mom))
    m_var = 2 * ((v - mu).abs() * mag_v).mean(0) + var
    mg['moving'][key] = (m0.abs() * mom + mag_v.mean(0) * (1 - mom),
                         v0.abs() * mom + m_var * (1 - mom))

  # ------------------------------------------------------------------ forward
  h, mh = x, x.abs()
  bn_in = None
  if cfg.input_bn:
    mu, var = stats(h, 'input')
    update_moving('input', h, mh)
    y, xh, r, m_xh, my = _bn_fwd(h, f(params['in_gamma']), f(params['in_beta']), mu, var, cfg,
                                 mh)
    bn_in = (xh, r, m_xh)
    h, mh = y, my
  bn = []
  for d in range(L):
    out['A'].append(h)
    mg['A'].append(mh)
    z = h @ W[d] + B[d]
    mz = mh @ W[d].abs() + B[d].abs()
    if cfg.use_bn:
      mu, var = stats(z, d)
      update_moving(d, z, mz)
      y, xh, r, m_xh, my = _bn_fwd(z, G[d], Be[d], mu, var, cfg, mz)
      bn.append((xh, r, m_xh, mz))
    else:
      y, my = z, mz
    out['Y'].append(y)
    mg['Y'].append(my)
    h = y * gates[d] * scale
    mh = my * gates[d] * scale
  out['A'].append(h)
  mg['A'].append(mh)
  s = h @ W[L] + B[L]
  ms = mh @ W[L].abs() + B[L].abs()
  live = None
  if mask is not None and O == 1:
    live = f(mask.reshape(-1, 1))
    s = torch.where(live > 0, s, torch.full_like(s, LOG_EPSILON))
    ms = torch.where(live > 0, ms, torch.zeros_like(ms))
  out['scores'], mg['scores'] = s, ms

  # ----------------------------------------------------------------- backward
  dsl = ds if live is None else ds * live
  mds = dsl.abs()
  gW, gB, mgW, mgB = [None] * (L + 1), [None] * (L + 1), [None] * (L + 1), [None] * (L + 1)
  gG, gBe, mgG, mgBe = [None] * L, [None] * L, [None] * L, [None] * L
  gW[L], gB[L] = h.t() @ dsl, dsl.sum(0)
  mgW[L], mgB[L] = mh.t() @ mds, mds.sum(0)
  dh, mdh = dsl @ W[L].t(), mds @ W[L].abs().t()
  dz_list, mdz_list = [None] * L, [None] * L
  for d in range(L - 1, -1, -1):
    dy = dh * gates[d] * scale
    mdy = mdh * gates[d] * scale
    if cfg.use_bn:
      xh, r, m_xh, mz = bn[d]
      g = G[d]
      gBe[d], gG[d] = dy.sum(0), (dy * xh).sum(0)
      mgBe[d] = mdy.sum(0)
      mgG[d] = (mdy * xh.abs()).sum(0) + (dy.abs() * m_xh).sum(0)
      if cfg.training:
        dz = g * r * (dy - dy.mean(0) - xh * (dy * xh).mean(0))
        t = (mdy + mdy.mean(0) + xh.abs() * (xh.abs() * mdy).mean(0) +
             m_xh * (dy * xh).mean(0).abs() + xh.abs() * (dy.abs() * m_xh).mean(0))
        mdz = g.abs() * r * t + dz.abs() * (1 + r * (xh.abs() * mz).mean(0))
      else:
        dz = g * r * dy
        mdz = g.abs() * r * mdy + dz.abs()
    else:
      dz, mdz = dy, mdy
    dz_list[d], mdz_list[d] = dz, mdz
    gW[d], gB[d] = out['A'][d].t() @ dz, dz.sum(0)
    mgW[d], mgB[d] = mg['A'][d].t() @ mdz, mdz.sum(0)
    dh, mdh = dz @ W[d].t(), mdz @ W[d].abs().t()
  out['dz'], mg['dz'] = dz_list, mdz_list
  if L > 0 and not cfg.input_bn:
    out['dx'], mg['dx'] = dh, mdh
  gin = mgin = None
  if cfg.input_bn:
    xh, r, m_xh = bn_in
    gin = [(dh * xh).sum(0), dh.sum(0)]
    mgin = [(mdh * xh.abs()).sum(0) + (dh.abs() * m_xh).sum(0), mdh.sum(0)]

  def flat(ws, bs, gs, bes, gi):
    parts = []
    for w, b in zip(ws, bs):
      parts += [w.reshape(-1), b.reshape(-1)]
    if gi is not None:
      parts += gi
    if cfg.use_bn:
      for g, be in zip(gs, bes):
        parts += [g, be]
    return torch.cat(parts)

  out['grads'] = flat(gW, gB, gG, gBe, gin)
  mg['grads'] = flat(mgW, mgB, mgG, mgBe, mgin)
  out['mag'] = mg
  return out


class Bound:
  """u per returned quantity for one precision and plan (see the module docstring)."""

  def __init__(self, cfg, plan, precision):
    u_p, u_tc, per_k = PRECISIONS[precision]
    tc = precision != 'fp32'
    u = _U24
    dims, L, O = cfg.dims, cfg.L, cfg.dims[-1]
    red = (plan.red_rows + 256 + plan.red_blocks) * u

    def gemm(k):
      return u_p + (per_k * k + 1) * (u_tc if tc else u)

    # forward: u of the input of Dense d (index d), and of the scores
    self.bn_stats = {}     # u of the moving statistics after the update
    a = 0.0
    if cfg.input_bn:
      self.bn_stats['input'] = red + 6 * u
      a = red + 8 * u
    fwd = [a]
    for d in range(L):
      z = fwd[d] + gemm(dims[d])
      if cfg.use_bn:
        self.bn_stats[d] = z + red + 6 * u
        z = z + red + 8 * u
      if cfg.drop_active:
        z += 4 * u
      fwd.append(z)
    self.fwd = fwd
    self.scores = fwd[L] + (dims[L] + 1) * u
    # backward
    if tc:
      out_len = plan.out_rows + 256 + plan.out_slots
      dw_len = lambda: u_p + per_k * plan.rows_per_split * u_tc + plan.splits * u
      cs_len = max(plan.rows_per_split + plan.splits, out_len,
                   plan.rows_per_split + 128 + 8 * plan.sms)
    else:
      out_len = plan.rows_per_split + plan.splits
      dw_len = lambda: (plan.rows_per_split + plan.splits) * u
      cs_len = plan.rows_per_split + plan.splits
    grads = [None] * (L + 1)
    bn_g = [None] * L
    grads[L] = (fwd[L] + out_len * u, out_len * u)
    dh = O * u
    for d in range(L - 1, -1, -1):
      dy = dh + (4 * u if cfg.drop_active else 0.0)
      if cfg.use_bn:
        bn_g[d] = dy + fwd[d + 1] + red
        dz = dy + fwd[d + 1] + red + 8 * u
      else:
        dz = dy
      grads[d] = (fwd[d] + dz + dw_len(), dz + cs_len * u)
      dh = dz + gemm(dims[d + 1])
    self.dx = dh
    self.input_bn_grads = dh + fwd[0] + red + 4 * u if cfg.input_bn else None
    self.layer_grads = grads
    self.bn_grads = bn_g

  def grads(self, cfg):
    """u for each entry of the flat gradient."""
    dims, L = cfg.dims, cfg.L
    parts = []
    for d in range(L + 1):
      uw, ub = self.layer_grads[d]
      parts += [torch.full((dims[d] * dims[d + 1],), uw), torch.full((dims[d + 1],), ub)]
    if cfg.input_bn:
      parts.append(torch.full((2 * dims[0],), self.input_bn_grads))
    if cfg.use_bn:
      for d in range(L):
        parts.append(torch.full((2 * dims[d + 1],), self.bn_grads[d]))
    return torch.cat(parts).double()


def err_ratio(got, want, mag, u):
  """max |got - want| / (C u mag) over the elements (0 where both sides are exactly 0), and
  the index of the worst element.  A ratio above 1 fails the bound."""
  got = got.detach().double().reshape(-1)
  want = want.detach().double().reshape(-1).to(got.device)
  mag = mag.detach().double().reshape(-1).to(got.device)
  u = torch.as_tensor(u, dtype=torch.float64, device=got.device).reshape(-1)
  err = (got - want).abs()
  bound = C * u * mag
  ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
  ratio = torch.nan_to_num(ratio, nan=math.inf, posinf=math.inf)
  i = int(ratio.argmax())
  return float(ratio[i]), i


def gate_ratio(hidden, ref, bound, cfg, dropout_seed=None):
  """How far the kernel's gates are from admissible, as a ratio like err_ratio's.  Gate
  (m, j) of layer d must be what the exact layer gives, keep = [Y_d > 0 with ReLU] and [not
  dropped by the kernel's stream], except where |Y_d| <= C u mag(Y_d): there rounding may
  decide the ReLU either way.  A kept element the stream drops is inadmissible outright.
  Returns (ratio, layer)."""
  worst, where = 0.0, None
  for d, h in enumerate(hidden):
    gate = gates_from([h], cfg)[0] > 0
    y, my = ref['Y'][d], ref['mag']['Y'][d]
    keep = torch.ones_like(gate)
    if cfg.drop_active:
      keep = dropout_keep(dropout_seed, d, *gate.shape, cfg.dropout, gate.device)
    want = keep & (y > 0) if cfg.relu else keep
    bad = gate != want
    if not bad.any():
      continue
    r = torch.where(keep, y.abs() / (C * bound.fwd[d + 1] * my),
                    torch.full_like(y, math.inf))[bad]
    r = float(torch.nan_to_num(r, nan=math.inf).max())
    if r > worst:
      worst, where = r, d
  return worst, where


def check(cfg, precision, plan, x, params, ds, got, mask=None, moving=None, dropout_seed=None):
  """The whole comparison of one tower call: `got` holds what the kernel returned, 'hidden'
  ([H_d] from its workspace), 'scores', 'grads', 'moving' ({key: (mean, var)} after a training
  call with BN) and 'dx' ([(col0, ncols, dX[:, :ncols])]).  The gates are taken from
  got['hidden'] and checked for admissibility.  Returns [(what, ratio)]; every ratio must
  be <= 1."""
  ref = forward_backward(x, params, cfg, gates_from(got['hidden'], cfg), ds, mask, moving)
  bound = Bound(cfg, plan, precision)
  mag = ref['mag']
  out = [('gates', gate_ratio(got['hidden'], ref, bound, cfg, dropout_seed)[0])]
  live = slice(None)
  if mask is not None and cfg.dims[-1] == 1:
    live = mask.reshape(-1).bool()
  out.append(('scores', err_ratio(got['scores'][live], ref['scores'][live],
                                  mag['scores'][live], bound.scores)[0]))
  for d, h in enumerate(got['hidden']):
    out.append(('H%d' % d, err_ratio(h, ref['A'][d + 1], mag['A'][d + 1], bound.fwd[d + 1])[0]))
  out.append(('grads', err_ratio(got['grads'], ref['grads'], mag['grads'], bound.grads(cfg))[0]))
  for key, (mu, var) in (got.get('moving') or {}).items():
    (m_mu, m_var), (r_mu, r_var) = mag['moving'][key], ref['moving'][key]
    out.append(('moving mean %s' % key, err_ratio(mu, r_mu, m_mu, bound.bn_stats[key])[0]))
    out.append(('moving var %s' % key, err_ratio(var, r_var, m_var, bound.bn_stats[key])[0]))
  for c0, nc, dx in got.get('dx', []):
    out.append(('dX[%d:%d]' % (c0, c0 + nc),
                err_ratio(dx, ref['dx'][:, c0:c0 + nc], mag['dx'][:, c0:c0 + nc], bound.dx)[0]))
  return out
