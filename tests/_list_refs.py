"""Blocked fp64 references for the O(N^2) per-list losses.

The oracle states ApproxNDCG / ApproxMRR and the pairwise losses with [B, N, N] fp64 tensors
and autograd.  At N = 8192 one such tensor is 512 MB per list, and autograd keeps several, so
the large-list tests use these restatements of the same operations instead: blocks of
ROW_BLOCK rows against the whole list, with the gradients in closed form,

  approx ranks    r_i = 1/2 + sum_j sigmoid(z_j - z_i)
                  d sum_i c_i r_i / d z_k = sum_i (c_i - c_k) sigmoid'(z_k - z_i)
  pairwise        L = sum_i w_i sum_j P_ij phi(z_i - z_j)
                  dL/dz_i = sum_j P_ij w_i phi'(z_i - z_j) - sum_j P_ji w_j phi'(z_j - z_i)

with z = scores / temperature and P the (detached) pair weights: label order times the lambda
weight.  CircleLoss and the OPA metric are restated the same way (see their docstrings).
Peak memory is a few [B, ROW_BLOCK, N] fp64 blocks (about 100 MB at B = 1,
N = 8192).  tests/test_list_size_reference.py checks both against the oracle at N <= 512.
"""
import torch

from oracle import losses_impl as OL

ROW_BLOCK = 256


def _blocks(n):
  bs = ROW_BLOCK
  for a in range(0, n, bs):
    yield a, min(n, a + bs)


def _list_weights(labels, weights):
  """Listwise weight normalisation (losses_impl.py:1004-1015): sum(w l) / sum(l) over the
  label-valid items, [B]."""
  b = labels.shape[0]
  if weights is None:
    return torch.ones(b, dtype=labels.dtype)
  lab = torch.where(labels >= 0, labels, torch.zeros_like(labels))
  num = (weights.to(labels.dtype) * lab).sum(1)
  den = lab.sum(1)
  return torch.where(den != 0, num / torch.where(den != 0, den, torch.ones_like(den)),
                     torch.zeros_like(num))


def approx_ranks(z):
  """r_i = 1/2 + sum_j sigmoid(z_j - z_i) (the j == i term contributes 1/2)."""
  r = torch.empty_like(z)
  for a, e in _blocks(z.shape[1]):
    r[:, a:e] = torch.sigmoid(z.unsqueeze(1) - z[:, a:e].unsqueeze(2)).sum(-1) + 0.5
  return r


def _approx_rank_vjp(z, c):
  """g_k = d (sum_i c_i r_i) / d z_k = sum_i (c_i - c_k) sigmoid'(z_k - z_i)."""
  g = torch.empty_like(z)
  for a, e in _blocks(z.shape[1]):
    s = torch.sigmoid(z[:, a:e].unsqueeze(2) - z.unsqueeze(1))
    g[:, a:e] = ((c.unsqueeze(1) - c[:, a:e].unsqueeze(2)) * (s * (1. - s))).sum(-1)
  return g


def approx_loss(labels, scores, weights=None, mask=None, temperature=0.1, mode='ndcg'):
  """ApproxNDCGLoss / ApproxMRRLoss `compute(..., Reduction.SUM, mask)`: returns
  (sum_b weight_b loss_b, its gradient w.r.t. scores, per-list loss [B])."""
  labels, scores = labels.double(), scores.double()
  if weights is not None:
    weights = weights.double()
  if mask is None:
    mask = labels >= 0
  z = scores / temperature
  zz = torch.where(mask, z, z.min(dim=1, keepdim=True).values - 1e3)
  cl = torch.where(mask, labels, torch.zeros_like(labels))
  nonzero = cl.sum(1) > 0
  cl = torch.where(nonzero.unsqueeze(1), cl, torch.full_like(cl, 1e-10))
  r = approx_ranks(zz)
  if mode == 'ndcg':
    gains = OL._safe_default_gain_fn(cl)
    inv_max = OL.inverse_max_dcg(cl, gain_fn=OL._safe_default_gain_fn).reshape(-1)
    lg = torch.log1p(r)
    loss = -(gains / lg).sum(1) * inv_max
    c = inv_max.unsqueeze(1) * gains / ((1. + r) * lg * lg)        # d loss / d r
  else:
    s = cl.sum(1, keepdim=True)
    loss = -(cl / r).sum(1) / s.reshape(-1)
    c = cl / (r * r * s)
  w = _list_weights(labels, weights) * nonzero.double()
  gz = _approx_rank_vjp(zz, c)
  grad = torch.where(mask, gz, torch.zeros_like(gz)) * (w / temperature).unsqueeze(1)
  return (w * loss).sum(), grad, loss


def _phi(kind, x):
  """(phi(x), phi'(x)) of losses_impl.py:933-958; x = z_i - z_j."""
  if kind == 'logistic':
    return torch.relu(-x) + torch.log1p(torch.exp(-x.abs())), -torch.sigmoid(-x)
  if kind == 'hinge':
    return torch.relu(1. - x), -(1. - x > 0).double()
  if kind == 'soft_zero_one':
    s = torch.sigmoid(x)
    return 1. - s, -s * (1. - s)
  raise ValueError(kind)


def _pair_lambda_block(lam, labels, ranks, a, e, aux):
  """Rows a..e of lambda_weight.pair_weights(labels, ranks) (losses_impl.py:255-279,
  299-369, 410-454) for DCGLambdaWeight (incl. NDCG) and PrecisionLambdaWeight."""
  n = labels.shape[1]
  valid = labels >= 0
  vp = (valid[:, a:e].unsqueeze(2) & valid.unsqueeze(1)).double()
  ri, rj = ranks[:, a:e].unsqueeze(2), ranks.unsqueeze(1)
  if isinstance(lam, OL.PrecisionLambdaWeight):
    pos = aux['pos']
    diff = (pos[:, a:e].unsqueeze(2) - pos.unsqueeze(1)).abs() * vp
    return diff * ((ri <= lam._topn) ^ (rj <= lam._topn)).double()
  if isinstance(lam, OL.DCGLambdaWeight):
    g = aux['gain']
    pair_gain = (g[:, a:e].unsqueeze(2) - g.unsqueeze(1)).abs() * vp
    topn = lam._topn or n
    disc = lam._rank_discount_fn
    in_top = (ri <= topn) | (rj <= topn)
    diff = (ri - rj).abs().double()
    safe = torch.where(diff > 0, diff, torch.ones_like(diff))
    u = torch.where((diff > 0) & in_top, (disc(safe) - disc(safe + 1.)).abs(),
                    torch.zeros_like(diff))
    rd = aux['rank_disc']
    v = (rd[:, a:e].unsqueeze(2) - rd.unsqueeze(1)).abs()
    pd = ((1. - lam._smooth_fraction) * u + lam._smooth_fraction * v) * in_top.double()
    return pair_gain * pd * float(n)
  raise NotImplementedError(type(lam).__name__)


def _lambda_aux(lam, labels, ranks):
  """Per-item quantities of the lambda weight that need the whole list."""
  if lam is None:
    return None
  cl = torch.where(labels >= 0, labels, torch.zeros_like(labels))
  if isinstance(lam, OL.PrecisionLambdaWeight):
    return {'pos': lam._positive_fn(cl).double()}
  gain = lam._gain_fn(cl)
  if lam._normalized:
    gain = gain * OL.inverse_max_dcg(cl, gain_fn=lam._gain_fn,
                                     rank_discount_fn=lam._rank_discount_fn, topn=lam._topn)
  topn = lam._topn or labels.shape[1]
  rd = torch.where(ranks > topn, torch.zeros_like(ranks, dtype=torch.float64),
                   lam._rank_discount_fn(ranks.double()))
  return {'gain': gain, 'rank_disc': rd}


def pairwise_loss(labels, scores, weights=None, phi='logistic', lambda_weight=None,
                  temperature=1.0):
  """Keras pairwise loss before its reduction: returns (sum_b sum_i w_i sum_j P_ij loss_ij,
  its gradient w.r.t. scores).  `phi` is 'logistic' | 'hinge' | 'soft_zero_one' | 'mse'
  (PairwiseMSELoss: all ordered pairs of valid items off the diagonal).  The Keras AUTO
  reduction divides both by B * N."""
  labels, scores = labels.double(), scores.double()
  b, n = labels.shape
  valid = labels >= 0
  w = torch.ones_like(labels) if weights is None else (
      torch.ones_like(labels) * weights.double())
  w = torch.where(valid, w, torch.zeros_like(w))
  z = scores / temperature
  ranks = OL._compute_ranks(z, valid) if lambda_weight is not None else None
  aux = _lambda_aux(lambda_weight, labels, ranks)
  total = torch.zeros((), dtype=torch.float64)
  gz = torch.zeros_like(z)
  for a, e in _blocks(n):
    vp = (valid[:, a:e].unsqueeze(2) & valid.unsqueeze(1)).double()
    d = z[:, a:e].unsqueeze(2) - z.unsqueeze(1)
    if phi == 'mse':
      dl = labels[:, a:e].unsqueeze(2) - labels.unsqueeze(1)
      pw = vp.clone()
      idx = torch.arange(a, e)
      pw[:, idx - a, idx] = 0.
      f, df = (d - dl) ** 2, 2. * (d - dl)
    else:
      pw = (labels[:, a:e].unsqueeze(2) - labels.unsqueeze(1) > 0).double() * vp
      f, df = _phi(phi, d)
    if lambda_weight is not None:
      pw = pw * _pair_lambda_block(lambda_weight, labels, ranks, a, e, aux)
    m = w[:, a:e].unsqueeze(2) * pw
    total = total + (m * f).sum()
    mdf = m * df
    gz[:, a:e] += mdf.sum(2)
    gz -= mdf.sum(1)
  return total, gz / temperature


def circle_loss(labels, scores, weights=None, gamma=64., margin=0.25):
  """CircleLoss `compute(..., Reduction.SUM)` (losses_impl.py:1036-1116): returns
  (sum_b weight_b loss_b, its gradient w.r.t. scores).  With s = clip(scores, 0, 1),
  a_i = gamma alpha_i (1 - s_i - m), b_j = gamma alpha_j (s_j - m) (alpha detached), the pair
  sum factorises: S = sum_{i, j valid, l_i > l_j} e^(a_i + b_j), loss = log1p(S), and
  dS/ds_k = gamma alpha_k (e^(b_k) sum_{i: l_i > l_k} e^(a_i)
                           - e^(a_k) sum_{j: l_j < l_k} e^(b_j)).
  Every list must hold a valid pair (the reference's weight is 0 / 0 otherwise)."""
  labels, scores = labels.double(), scores.double()
  valid = labels >= 0
  s = scores.clamp(0., 1.)
  pa = (1. - s + margin).clamp(min=0.)
  pb = (s + margin).clamp(min=0.)
  a = torch.where(valid, gamma * pa * (1. - s - margin), torch.full_like(s, -torch.inf))
  bb = torch.where(valid, gamma * pb * (s - margin), torch.full_like(s, -torch.inf))
  ea, eb = a.exp(), bb.exp()
  above = torch.zeros_like(s)       # sum_{i: l_i > l_k} e^(a_i)
  below = torch.zeros_like(s)       # sum_{j: l_j < l_k} e^(b_j)
  for lo, hi in _blocks(s.shape[1]):
    gt = labels.unsqueeze(1) > labels[:, lo:hi].unsqueeze(2)      # [B, rows k, cols i]
    above[:, lo:hi] = (gt * ea.unsqueeze(1)).sum(2)
    lt = labels.unsqueeze(1) < labels[:, lo:hi].unsqueeze(2)
    below[:, lo:hi] = (lt * eb.unsqueeze(1)).sum(2)
  S = torch.where(valid, ea * below, torch.zeros_like(s)).sum(1)
  loss = torch.log1p(S)
  w = _list_weights(labels, weights)
  ds = gamma * (pb * eb * above - pa * ea * below)
  ds = torch.where(valid, ds, torch.zeros_like(ds))
  ds = torch.where((scores >= 0) & (scores <= 1), ds, torch.zeros_like(ds))
  return (w * loss).sum(), ds * (w / (1. + S)).unsqueeze(1)


def opa_metric(labels, predictions, weights=None, mask=None):
  """OPAMetric.compute (metrics_impl.py:708-743) counted on blocks of rows: returns
  (per-list OPA [B, 1], per-list weight [B, 1])."""
  labels, predictions = labels.double(), predictions.double()
  w = torch.ones_like(labels) if weights is None else (
      torch.ones_like(labels) * weights.double())
  if mask is None:
    mask = labels >= 0
  mask = mask & (w > 0)
  labels = torch.where(mask, labels, torch.zeros_like(labels))
  predictions = torch.where(mask, predictions,
                            predictions.min(dim=1, keepdim=True).values - 1e-6)
  num = torch.zeros(labels.shape[0], dtype=torch.float64)
  den = torch.zeros_like(num)
  for lo, hi in _blocks(labels.shape[1]):
    pw = ((labels[:, lo:hi].unsqueeze(2) > labels.unsqueeze(1)) &
          mask[:, lo:hi].unsqueeze(2) & mask.unsqueeze(1)).double() * w[:, lo:hi].unsqueeze(2)
    den += pw.sum((1, 2))
    num += (pw * (predictions[:, lo:hi].unsqueeze(2) > predictions.unsqueeze(1))).sum((1, 2))
  opa = torch.where(den != 0, num / torch.where(den != 0, den, torch.ones_like(den)),
                    torch.zeros_like(num))
  return opa.unsqueeze(1), den.unsqueeze(1)
