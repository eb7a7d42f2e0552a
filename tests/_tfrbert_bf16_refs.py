"""fp64 replay of TFR-BERT's bf16 mode (include/tfr_b200.h, K15, TFR_PREC_BF16), in torch, for
tests/test_tfrbert_bf16.py (CPU) and tests/test_tfrbert_bf16_gpu.py.

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


def forward(wid, mask, tid, flat, V, E, H, I, NL, P, Tv, training=False, hdrop=0.0, adrop=0.0,
            sdrop=0.0, seed=0, rounding=True, mask_logits=True, attn_site_shift=0):
  """scores [S] (fp64) of the bf16 mode; arguments as _tfrbert_refs.forward.  `rounding`
  False gives the unrounded model; `attn_site_shift` moves the attention dropout's site (a
  negative control)."""
  rb, rg, rv = (round_both, round_grad, round_value) if rounding else (_ident,) * 3
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
  x = rv(x)
  to_mask = mask.reshape(S, 1, 1, L) != 0
  for l in range(NL):
    qkv = rb(rg(x) @ rv(p['wqkv%d' % l]) + p['bqkv%d' % l])
    q, kk, v = [qkv[..., i * E:(i + 1) * E].reshape(S, L, H, dh).transpose(1, 2)
                for i in range(3)]
    logits = rg(q @ kk.transpose(-1, -2) / math.sqrt(dh))
    if mask_logits:
      logits = torch.where(to_mask, logits, (logits.float() + -1e9).double())
    pr = torch.softmax(logits, -1)
    ka = keep(seed, 2 + 3 * l + attn_site_shift, S * H * L * L, adrop, (S, H, L, L))
    if ka is not None:
      pr = pr * ka
    o = rb(rv(pr) @ v)
    if rounding:   # D_i over the stored o (see the module docstring)
      lse = torch.logsumexp(logits, -1, keepdim=True)
      o = o + (pr @ v - o).detach() * (lse - lse.detach())
    o = o.transpose(1, 2).reshape(S, L, E)
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


def bars(L, E, I, NL):
  """(score bar, gradient bar) against the replay, relative (see the module docstring)."""
  u = U_BF16 + max(L, E, I, 3 * E) * U_ACC
  fwd_sites = 9 * NL + 2
  return C_SAFETY * fwd_sites * u, C_SAFETY * (fwd_sites + 8 * NL + 2) * u
