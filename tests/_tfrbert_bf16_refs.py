"""fp64 replay of TFR-BERT's bf16 mode (include/tfr_b200.h, K15, TFR_PREC_BF16), in torch, for
tests/test_tfrbert_bf16.py (CPU), tests/test_tfrbert_bf16_gpu.py and, for the attention core
alone (`attention`, `attn_bars`, `attn_lse`), tests/test_attn_bf16_gpu.py.

`forward` is _tfrbert_refs.forward with the header's bf16 rounding points replayed; gradients
come from autograd over it.  Three kinds of rounding, all to nearest even:
  round_both  (_RoundBoth)   the value and its gradient: the stored GEMM and attention outputs
                             (qkv, o, y, u, a, y2, pre), whose gradients the kernels also
                             store as bf16 (dqkv, dO, dy, du, da, dpre);
  round_grad  (_RoundGrad)   the gradient only: a GEMM input on the input-gradient side (x_l,
                             o, x', a, the [CLS] rows: dx, dO, d x', da, dCLS are bf16 GEMM
                             outputs) and the scaled logits (dS);
  round_value                the value only (straight-through gradient): the weight shadows,
                             the LayerNorm outputs (their gradient is the fp32 residual
                             gradient) and P~ (dP stays fp32).
One more term replays the kernels' D_i = dO_i . o_i over the stored bf16 o: autograd's softmax
backward uses D_i = dO_i . (P~ v) with the unrounded P~; a term (P~ v - o).detach() *
(lse - lse.detach()), zero in value, adds P_ij dO_i . (P~ v - o)_i to the logits' gradient,
which turns the one D_i into the other.
With rounding=False every rounding is the identity and the extra term is left out, so the
replay is _tfrbert_refs.forward op for op.

Error bars (`bars`), relative to the largest exact magnitude as in _tfrbert_refs.  Against the
replay the kernels differ only by fp32 (not fp64) accumulation, which can flip a bf16 rounding
that falls near a tie: one bf16 unit, 2^-8 relative, in that element.  A quantity's bar is
C = 2 times u = 2^-8 + k 2^-23 (the flip plus fp32 accumulation of depth k = max(L, E, I, 3E))
per rounding site on its longest path: x_0, then per layer qkv, P~, o, y, x', u, a, y2, x''
(9), then pre, for the scores; the gradients add per layer dy twice, du, da, d x', dO, dS, dx
(8) and dpre, dCLS.
"""
import math

import torch

from _tfrbert_refs import gelu_tanh
from _tfrbert_refs import keep
from _tfrbert_refs import layer_norm
from _tfrbert_refs import unflatten

U_BF16 = 2.0 ** -8
U_ACC = 2.0 ** -23
C_SAFETY = 2.0


def bf16(x):
  """x rounded to the nearest bf16 (ties to even), in x's dtype."""
  return x.to(torch.bfloat16).to(x.dtype)


class _RoundBoth(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x):
    return bf16(x)

  @staticmethod
  def backward(ctx, g):
    return bf16(g)


class _RoundGrad(torch.autograd.Function):

  @staticmethod
  def forward(ctx, x):
    return x.clone()

  @staticmethod
  def backward(ctx, g):
    return bf16(g)


def round_both(x):
  return _RoundBoth.apply(x)


def round_grad(x):
  return _RoundGrad.apply(x)


def round_value(x):
  return x + (bf16(x) - x).detach()


def _ident(x):
  return x


def attention(qkv, mask, H, adrop=0.0, seed=0, site=2, rounding=True, mask_logits=True,
              skip=(), ds_scaled_first=False, swap_ij=False):
  """o [S, L, E] (fp64) of the bf16 attention core (csrc/din_bf16.cu) on qkv [S, L, 3E]
  (fp64, may require grad; q, k, v blocks of H heads) and mask [S, L] (0 = padded key).
  Dropout keeps element ((s H + head) L + i) L + j of keep(seed, site, ...).  With rounding
  on: dS = round_grad of the scaled logits, P~ = round_value(dropout(P)), o = round_both(P~ v)
  and D_i over that o; rounding=False is the unrounded op, op for op.
  Negative controls: `skip` drops rounding sites ('p' P~, 'o' o's value, 'ds' dS, 'd_i' the
  D_i term), ds_scaled_first rounds dS after the 1 / sqrt(dh) scale, swap_ij draws keep(j, i)."""
  rb, rg, rv = (round_both, round_grad, round_value) if rounding else (_ident,) * 3
  S, L, E3 = qkv.shape
  E = E3 // 3
  dh = E // H
  q, kk, v = [qkv[..., i * E:(i + 1) * E].reshape(S, L, H, dh).transpose(1, 2) for i in range(3)]
  r_ds = _ident if 'ds' in skip else rg
  if ds_scaled_first:   # rounds the gradient of q k^T, i.e. dS / sqrt(dh)
    logits = r_ds(q @ kk.transpose(-1, -2)) / math.sqrt(dh)
  else:
    logits = r_ds(q @ kk.transpose(-1, -2) / math.sqrt(dh))
  if mask_logits:
    to_mask = mask.reshape(S, 1, 1, L).to(logits.device) != 0
    logits = torch.where(to_mask, logits, (logits.float() + -1e9).double())
  pr = torch.softmax(logits, -1)
  ka = keep(seed, site, S * H * L * L, adrop, (S, H, L, L))
  if ka is not None:
    if swap_ij:
      ka = ka.transpose(-1, -2)
    pr = pr * ka.to(pr.device)
  r_p = _ident if 'p' in skip else rv
  o = r_p(pr) @ v
  o = (round_grad if rounding and 'o' in skip else rb)(o)
  if rounding and 'd_i' not in skip:   # D_i over the stored o (see the module docstring)
    lse = torch.logsumexp(logits, -1, keepdim=True)
    o = o + (pr @ v - o).detach() * (lse - lse.detach())
  return o.transpose(1, 2).reshape(S, L, E)


def forward(wid, mask, tid, flat, V, E, H, I, NL, P, Tv, training=False, hdrop=0.0, adrop=0.0,
            sdrop=0.0, seed=0, rounding=True, mask_logits=True, attn_site_shift=0):
  """scores [S] (fp64) of the bf16 mode; arguments as _tfrbert_refs.forward.  `rounding`
  False gives the unrounded model; `attn_site_shift` moves the attention dropout's site (a
  negative control)."""
  rb, rg, rv = (round_both, round_grad, round_value) if rounding else (_ident,) * 3
  S, L = wid.shape
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
  x = rv(x)
  for l in range(NL):
    qkv = rb(rg(x) @ rv(p['wqkv%d' % l]) + p['bqkv%d' % l])
    o = attention(qkv, mask, H, adrop, seed, 2 + 3 * l + attn_site_shift, rounding=rounding,
                  mask_logits=mask_logits)
    y = rb(rg(o) @ rv(p['wo%d' % l]) + p['bo%d' % l])
    k1 = keep(seed, 3 + 3 * l, S * L * E, hdrop, (S, L, E))
    if k1 is not None:
      y = y * k1
    x1 = rv(layer_norm(y + x, p['ln1_g%d' % l], p['ln1_b%d' % l]))
    a = rb(gelu_tanh(rb(rg(x1) @ rv(p['w1%d' % l]) + p['b1%d' % l])))
    y2 = rb(rg(a) @ rv(p['w2%d' % l]) + p['b2%d' % l])
    k2 = keep(seed, 4 + 3 * l, S * L * E, hdrop, (S, L, E))
    if k2 is not None:
      y2 = y2 * k2
    x = rv(layer_norm(y2 + x1, p['ln2_g%d' % l], p['ln2_b%d' % l]))
  pooled = torch.tanh(rb(rg(x[:, 0]) @ rv(p['wp']) + p['bp']))
  ks = keep(seed, 2 + 3 * NL, S * E, sdrop, (S, E))
  if ks is not None:
    pooled = pooled * ks
  return pooled @ p['ws'] + p['bs'][0]


def _heads(x, H):
  S, L, E = x.shape
  return x.reshape(S, L, H, E // H).transpose(1, 2)


def _logits(qkv, mask, H):
  """(masked logits as the kernel forms them, scaled |q| |k|^T: each logit's magnitude sum),
  fp64 [S, H, L, L]."""
  E = qkv.shape[-1] // 3
  dh = E // H
  q, k = _heads(qkv[..., :E], H), _heads(qkv[..., E:2 * E], H)
  s = q @ k.transpose(-1, -2) / math.sqrt(dh)
  sabs = q.abs() @ k.abs().transpose(-1, -2) / math.sqrt(dh)
  if mask is not None:
    valid = mask.reshape(mask.shape[0], 1, 1, -1).to(s.device) != 0
    s = torch.where(valid, s, (s.float() + -1e9).double())
  return s, sabs


def attn_bars(qkv, mask, H, dO, O, adrop, seed, site):
  """Per-element bars {O, dQ, dK, dV} ([S, L, E] each) of the bf16 attention core against
  `attention`'s replay, for bf16 inputs qkv [S, L, 3E], dO [S, L, E] and the replay's O.

  The kernel and the replay round at the same points; they differ by fp32 (kernel) against
  fp64 (replay) arithmetic, which (a) can flip a bf16 rounding that falls near a tie, one bf16
  unit: at most 2^-7 of the rounded value, and (b) leaves fp32 errors of relative size
  2^-23 k (k the depth of a sum).  So every output X gets one bf16 unit of its own,
  2^-7 |X|, plus, on each term of the contraction that forms it, one bf16 unit where that
  term is a rounded quantity (P~ or dS) and the fp32 error of the term and of the sum:
    O  = P~ V          2^-7 |O|  + sum_j u_i |P~_ij| |V_j|
    dV = P~^T dO       2^-7 |dV| + sum_i u_i |P~_ij| |dO_i|
    dQ = scale dS K    2^-7 |dQ| + scale sum_j w_i A_ij |K_j|
    dK = scale dS^T Q  2^-7 |dK| + scale sum_i w_i A_ij |Q_i|
  P_ij = exp(x_ij - m_i) / l_i moves by twice the fp32 error of a logit, whose dot product of
  depth h has magnitude sum l_i = max_j scale |q_i| |k_j| (fp32 max subtraction, exp and the
  sum of N exponentials add 2^-23 (N + 4)); the contraction over N keys (or queries) adds
  N 2^-23:  u_i = 2^-7 + 2^-23 (2 N + 4 + h (1 + l_i)).
  dS_ij = P_ij (dP_ij keep_ij - D_i) is bounded by A_ij = P_ij (keep_ij |dO_i| |V_j| + D'_i),
  D'_i = sum |dO_i| |O_i|.  It carries its own flip (2^-7 A), P's error, fp32 dot products of
  depth h for dP and D (2 h 2^-23 A), and D_i over the kernel's stored O, whose elements may
  each sit one bf16 unit from the replay's (2^-7 A): w_i = 2^-6 + 2^-23 (2 N + 4 + h (3 + l_i)).
  """
  S, L, E3 = qkv.shape
  E = E3 // 3
  dh = E // H
  scale = 1.0 / math.sqrt(dh)
  q, k, v = [_heads(qkv[..., i * E:(i + 1) * E], H) for i in range(3)]
  g, o = _heads(dO, H), _heads(O, H)
  x, sabs = _logits(qkv, mask, H)
  p = torch.softmax(x, -1)
  ka = keep(seed, site, S * H * L * L, adrop, (S, H, L, L))
  ka = torch.ones_like(p) if ka is None else ka.to(p.device)
  pt = p * ka
  lrow = sabs.amax(-1, keepdim=True)
  u = 2.0 ** -7 + 2.0 ** -23 * (2 * L + 4 + dh * (1 + lrow))
  w = 2.0 ** -6 + 2.0 ** -23 * (2 * L + 4 + dh * (3 + lrow))
  dabs = (g.abs() * o.abs()).sum(-1, keepdim=True)
  a = p * (ka * (g.abs() @ v.abs().transpose(-1, -2)) + dabs)
  # fp64 values of the outputs, for their own bf16 unit
  dp = g @ v.transpose(-1, -2)
  ds = p * (dp * ka - (g * o).sum(-1, keepdim=True))
  t = {'O': (o, (u * pt.abs()) @ v.abs()),
       'dV': (pt.transpose(-1, -2) @ g, (u * pt.abs()).transpose(-1, -2) @ g.abs()),
       'dQ': (scale * ds @ k, scale * (w * a) @ k.abs()),
       'dK': (scale * ds.transpose(-1, -2) @ q, scale * (w * a).transpose(-1, -2) @ q.abs())}
  out = {}
  for name, (val, terms) in t.items():
    out[name] = (2.0 ** -7 * val.abs() + terms).transpose(1, 2).reshape(S, L, E)
  return out


def attn_lse(qkv, mask, H):
  """(row max, 1 / sum, their tolerances), fp64 [S, L, H], of the kernel's lse: the max of
  the fp32 masked logits, whose error is a dot product of depth h (h 2^-23 times its
  magnitude sum) and their fp32 roundings (2^-22 |m|); 1 / sum of N exponentials in fp32,
  relative 2^-23 (N + 8) plus twice the logits' and the max's error."""
  E = qkv.shape[-1] // 3
  dh = E // H
  x, sabs = _logits(qkv, mask, H)
  m = x.amax(-1)
  inv = 1.0 / torch.exp(x - m.unsqueeze(-1)).sum(-1)
  lrow = sabs.amax(-1)
  m_tol = dh * 2.0 ** -23 * lrow + 2.0 ** -22 * m.abs()
  inv_tol = inv * 2.0 ** -23 * (x.shape[-1] + 8 + 4 * dh * lrow + 4 * lrow)
  return (m.transpose(1, 2), inv.transpose(1, 2), m_tol.transpose(1, 2),
          inv_tol.transpose(1, 2))


def bars(L, E, I, NL):
  """(score bar, gradient bar) against the replay, relative (see the module docstring)."""
  u = U_BF16 + max(L, E, I, 3 * E) * U_ACC
  fwd_sites = 9 * NL + 2
  return C_SAFETY * fwd_sites * u, C_SAFETY * (fwd_sites + 8 * NL + 2) * u
