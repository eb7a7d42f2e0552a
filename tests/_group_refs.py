"""References of the folded groupwise tower (csrc/mlp_group.cu): rolling-window group formation,
and an fp64 forward / backward with a per-element error bound, built on tests/_tower_fp64.py.

Group formation (model.py:164-244 semantics; `permutation` as in ranking_b200/model.py).  The
valid-first order of list b holds its valid positions in order, then its invalid ones.  Shuffle s
reorders it by perm[s, b] (default: identity).  Group g of shuffle s (row s N + g) holds in slot j
the item at position (g + j) mod max(nv, 1) of that order, and is valid when g < nv.  inv[s, b,
i, j] is the row of shuffle s whose slot j holds item i (-1: none); cnt[b, i] counts the (s, j)
pairs with inv >= 0.

fp64 forward / backward.  With A_0 [B G, gs D] the member features of every group, slot after
slot, the group score function is the plain tower on A_0, and _tower_fp64.forward_backward runs
it with the kernel's gates.  Layer 0's gates come from the H_0 that group_gather_fwd_kernel wrote
at rows M = B G, the later layers' from the H_d the tower stored.  The logits are the mean of the
member scores each item received (0 for items in no valid group); the member-score gradient is
dgscore[b, g, j] = dlogits[b, idx] / cnt[b, idx] for valid groups and 0 otherwise; dP_j[b, i] is
the sum over s of dZ_0 at row inv[s, b, i, j].

Bound.  Notation of _tower_fp64: u = 2^-24, u_p / u_tc / per_k of the precision, gemm(k) = u_p +
(per_k k + 1) u_tc.  The kernel computes

  * Z_0 = fl(b_0 + sum_j fl(P_j)) with P_j = X W_0^(j) one GEMM of K = D (not gs D) per slot,
    then gs + 1 fp32 additions (bias first, then the slots in order):
        u(Z_0) = u_p + (per_k D + 1) u_tc + (gs + 1) u,
    against gemm(gs D) in the plain tower.  Every later forward u shifts by the difference.
  * logits: S gs additions of member scores and one division by cnt:
        u(logits) = u(scores) + (S gs + 1) u,  mag(logits) = sum of mag(scores) / cnt.
  * dgscore: one division, so every backward quantity carries one more u than in the plain
    tower, whose dS is exact.
  * dP_j: S additions of dZ_0 rows: u(dP) = u(dZ_0) + S u.
  * dW_0^(j) = X^T dP_j: the rows are B N, not M, split as tfr_group_mlp_bwd does: per = ceil(B N
    / sms), rows_per = max(256, ceil(per / 128) 128), splits = min(ceil(B N / rows_per),
    plan.splits); a split then holds at most max(rows_per, ceil(B N / splits)) rows, rounded up
    to 128:  u(dW_0) = u(dP) + u_p + per_k rows u_tc + splits u.
  * db_0: the column sums of the dZ_0 tail (the last dgrad's, or the output layer's when there is
    one hidden layer), over M rows as in the plain tower: u(db_0) = u(dZ_0) + cs_len u.
The mean-of-scores magnitude is an upper bound on |logits| and on the error of its sum, since
every term carries its own mag(scores).  C = 2 of _tower_fp64 covers the first-order terms.
"""
import torch

import _tower_fp64 as R

_U24 = 2.0 ** -24


def form_groups(is_valid, gs, perms=None, num_shuffles=1, wrap_at_n=False):
  """is_valid [B, N] bool; perms None or [S, B, N] integer permutations of the valid-first order.
  Returns idx [B, S N, gs], gmask [B, S N] bool, inv [S, B, N, gs] (-1: none) and cnt [B, N], all
  int64 but gmask.  wrap_at_n: the windows wrap at N instead of nv (a negative control)."""
  v = torch.as_tensor(is_valid).bool()
  B, N = v.shape
  dev = v.device
  S = num_shuffles if perms is None else len(perms)
  nv = v.sum(1)
  # valid positions in order, then invalid ones in order: a stable sort on "is invalid"
  order = torch.sort((~v).to(torch.int32), dim=1, stable=True).indices
  g = torch.arange(N, device=dev)
  slots = g[:, None] + torch.arange(gs, device=dev)[None, :]                  # [N, gs]
  wrap = torch.full_like(nv, N) if wrap_at_n else nv.clamp(min=1)
  pos = slots[None] % wrap[:, None, None]                                       # [B, N, gs]
  idx, gmask = [], []
  for s in range(S):
    p = pos.reshape(B, -1)
    if perms is not None:
      p = torch.gather(torch.as_tensor(perms[s]).to(dev).long(), 1, p)
    idx.append(torch.gather(order, 1, p).reshape(B, N, gs))
    gmask.append(g[None, :] < nv[:, None])
  idx, gmask = torch.cat(idx, 1), torch.cat(gmask, 1)
  inv = torch.full((S, B, N, gs), -1, dtype=torch.long, device=dev)
  b, row = gmask.nonzero(as_tuple=True)
  for j in range(gs):
    i = idx[b, row, j]
    flat = ((row // N) * B + b) * N + i
    assert flat.unique().numel() == flat.numel(), 'an item fills one slot of two groups'
    inv[row // N, b, i, j] = row
  cnt = (inv >= 0).sum((0, 3))
  return idx, gmask, inv, cnt


def gathered(x, idx):
  """A_0 [B G, gs D]: row b G + g holds the features of group g's members, slot after slot."""
  B, N, D = x.shape
  G, gs = idx.shape[1], idx.shape[2]
  return torch.gather(x, 1, idx.reshape(B, G * gs, 1).expand(-1, -1, D)).reshape(B * G, gs * D)


def exact_gates(a0, params, cfg):
  """The gates of the exact fp64 tower on A_0 (what an unambiguous kernel would store)."""
  h, out = a0.double(), []
  for d in range(cfg.L):
    h = h @ params['w'][d].double() + params['b'][d].double()
    g = (h > 0).double() if cfg.relu else torch.ones_like(h)
    out.append(g)
    h = h * g
  return out


def scatter_mean(scores, inv, cnt):
  """logits [B, N] = the mean of the member scores [B G, gs] each item received (0: none)."""
  S, B, N, gs = inv.shape
  sc = scores.reshape(B, -1, gs)
  acc = torch.zeros(B, N, dtype=sc.dtype, device=sc.device)
  bb = torch.arange(B, device=sc.device)[:, None].expand(B, N)
  for s in range(S):
    for j in range(gs):
      g = inv[s, :, :, j]
      acc = acc + torch.where(g >= 0, sc[bb, g.clamp(min=0), j], torch.zeros_like(acc))
  c = cnt.to(sc.dtype)
  return torch.where(c > 0, acc / c.clamp(min=1), torch.zeros_like(acc))


def member_grad(dlogits, idx, gmask, cnt):
  """dgscore [B G, gs]: dlogits[b, idx] / cnt[b, idx] for valid groups, 0 otherwise."""
  B, G, gs = idx.shape
  fi = idx.reshape(B, -1)
  v = torch.gather(dlogits, 1, fi) / torch.gather(cnt.to(dlogits.dtype), 1, fi)
  v = torch.where(gmask[:, :, None].expand(-1, -1, gs).reshape(B, -1), v, torch.zeros_like(v))
  return v.reshape(B * G, gs)


def slot_grads(dz0, inv):
  """dP_j [B N, h1] = sum over s of dZ_0 at row inv[s, b, i, j] (0 where there is none)."""
  S, B, N, gs = inv.shape
  dz = dz0.reshape(B, -1, dz0.shape[-1])
  bb = torch.arange(B, device=dz.device)[:, None].expand(B, N)
  out = []
  for j in range(gs):
    acc = torch.zeros(B, N, dz.shape[-1], dtype=dz.dtype, device=dz.device)
    for s in range(S):
      g = inv[s, :, :, j]
      acc = acc + torch.where((g >= 0)[..., None], dz[bb, g.clamp(min=0)], torch.zeros_like(acc))
    out.append(acc.reshape(B * N, -1))
  return out


def forward_backward(x, params, cfg, gates, groups, dlogits, defect=None):
  """The folded tower in fp64.  x [B, N, D]; groups = form_groups(...); gates per hidden layer at
  rows B G; dlogits [B, N].  Returns the _tower_fp64 dict of the tower on A_0 (its 'grads' are the
  parameter gradient) with 'logits', 'dgscore', 'dP' added; 'mag' holds their magnitudes.

  defect (negative controls): 'swap_slots' swaps W_0's slot blocks 0 and 1, 'divide_by_S_gs'
  divides by S gs instead of cnt, 'no_bias0' drops layer 0's bias."""
  idx, gmask, inv, cnt = groups
  S, B, N, gs = inv.shape
  dev = gates[0].device if gates else x.device
  x = x.to(dev).double()
  dlogits = dlogits.to(dev).double()
  p = {'w': [w.detach().to(dev).double() for w in params['w']],
       'b': [b.detach().to(dev).double() for b in params['b']]}
  D = x.shape[-1]
  if defect == 'swap_slots':
    w0 = p['w'][0].clone()
    w0[:D], w0[D:2 * D] = p['w'][0][D:2 * D], p['w'][0][:D]
    p['w'][0] = w0
  elif defect == 'no_bias0':
    p['b'][0] = torch.zeros_like(p['b'][0])
  if defect == 'divide_by_S_gs':
    cnt = torch.where(cnt > 0, torch.full_like(cnt, S * gs), cnt)
  a0 = gathered(x, idx.to(dev))
  ds = member_grad(dlogits, idx.to(dev), gmask.to(dev), cnt.to(dev))
  ref = R.forward_backward(a0, p, cfg, gates, ds)
  inv, cnt = inv.to(dev), cnt.to(dev)
  mag = ref['mag']
  ref['logits'] = scatter_mean(ref['scores'], inv, cnt)
  mag['logits'] = scatter_mean(mag['scores'], inv, cnt)
  ref['dgscore'], mag['dgscore'] = ds, ds.abs()
  ref['dP'] = slot_grads(ref['dz'][0], inv)
  mag['dP'] = slot_grads(mag['dz'][0], inv)
  return ref


def dw0_splits(bn, plan):
  """(rows in the longest split, splits) of tfr_group_mlp_bwd's dW_0^(j) GEMMs over B N rows."""
  per = (bn + plan.sms - 1) // plan.sms
  rows_per = 256 if per < 256 else (per + 127) // 128 * 128
  splits = min((bn + rows_per - 1) // rows_per, plan.splits)
  rows = max(rows_per, ((bn + splits - 1) // splits + 127) // 128 * 128)
  return rows, splits


class Bound(object):
  """u per quantity of the folded tower (see the module docstring).  `fwd[d]` is the u of the
  input of Dense d (fwd[1]: H_0), as in _tower_fp64.Bound, so that _tower_fp64.gate_ratio reads
  it."""

  def __init__(self, cfg, precision, B, N, S, gs, sms):
    u = _U24
    u_p, u_tc, per_k = R.PRECISIONS[precision]
    dims, L, O = cfg.dims, cfg.L, cfg.dims[-1]
    D = dims[0] // gs
    self.plan = plan = R.Plan(cfg, B * S * N, sms)
    gemm = lambda k: u_p + (per_k * k + 1) * u_tc
    fwd = [0.0, gemm(D) + (gs + 1) * u]
    for d in range(1, L):
      fwd.append(fwd[d] + gemm(dims[d]))
    self.fwd = fwd
    self.scores = fwd[L] + (dims[L] + 1) * u
    self.logits = self.scores + (S * gs + 1) * u
    self.dgscore = u
    out_len = plan.out_rows + 256 + plan.out_slots
    dw_len = u_p + per_k * plan.rows_per_split * u_tc + plan.splits * u
    cs_len = max(plan.rows_per_split + plan.splits, out_len,
                 plan.rows_per_split + 128 + 8 * plan.sms)
    rows, splits = dw0_splits(B * N, plan)
    grads = [None] * (L + 1)
    grads[L] = (fwd[L] + u + out_len * u, u + out_len * u)
    dh = u + O * u
    for d in range(L - 1, -1, -1):
      if d > 0:
        grads[d] = (fwd[d] + dh + dw_len, dh + cs_len * u)
      else:
        self.dP = dh + S * u
        grads[0] = (self.dP + u_p + per_k * rows * u_tc + splits * u, dh + cs_len * u)
      dh = dh + gemm(dims[d + 1])
    self.layer_grads = grads

  def grads(self, cfg):
    dims = cfg.dims
    parts = []
    for d, (uw, ub) in enumerate(self.layer_grads):
      parts += [torch.full((dims[d] * dims[d + 1],), uw), torch.full((dims[d + 1],), ub)]
    return torch.cat(parts).double()


def check(cfg, bound, ref, got):
  """[(what, err / bound)] of the kernel's results against the reference: the gates'
  admissibility, every stored H_d, the logits and the flat parameter gradient.  `got` holds
  'hidden' ([H_d] at rows B G), 'logits' and 'grads'."""
  mag = ref['mag']
  out = [('gates', R.gate_ratio(got['hidden'], ref, bound, cfg)[0])]
  for d, h in enumerate(got['hidden']):
    out.append(('H%d' % d, R.err_ratio(h, ref['A'][d + 1], mag['A'][d + 1], bound.fwd[d + 1])[0]))
  out.append(('logits', R.err_ratio(got['logits'], ref['logits'], mag['logits'],
                                    bound.logits)[0]))
  out.append(('grads', R.err_ratio(got['grads'], ref['grads'], mag['grads'],
                                   bound.grads(cfg).to(ref['grads'].device))[0]))
  return out

