"""fp64 replay of TFR-BERT's fp16 mode (include/tfr_b200.h, K15, TFR_PREC_FP16) and a pure-Python
model of the dynamic loss scale rule, for tests/test_tfrbert_fp16.py (CPU) and
tests/test_tfrbert_fp16_gpu.py.

The fp16 mode has the bf16 mode's rounding points with fp16 in place of bf16, so its replay is
_tfrbert_bf16_refs run with fp16 rounding: `F` is a second instance of that module (loaded from
the same file, so the bf16 tests' module is untouched) whose `bf16` rounding function is
replaced by `fp16`.  F.forward and F.attention are then the fp16 replays, and rounding=False
still gives _tfrbert_refs.forward op for op.

Bars, as _tfrbert_bf16_refs' with fp16's unit: u = 2^-11 + k 2^-23 per rounding site on the
longest path (k the accumulation depth max(L, E, I, 3E)), C = 2.  The attention core's
per-element bars (`attn_bars`) are _tfrbert_bf16_refs.attn_bars with one fp16 unit, 2^-10 of
the rounded value, where that has one bf16 unit, 2^-7.
"""
import importlib.util
import math
import os

import torch

import _tfrbert_bf16_refs as B
from _tfrbert_bf16_refs import _heads
from _tfrbert_bf16_refs import _logits
from _tfrbert_bf16_refs import keep

U_FP16 = 2.0 ** -11
U_ACC = B.U_ACC
C_SAFETY = B.C_SAFETY


def fp16(x):
  """x rounded to the nearest fp16 (ties to even, subnormals kept, past 65504: +-inf), in
  x's dtype.  Through fp32, as the kernels round their fp32 values."""
  return x.float().to(torch.float16).to(x.dtype)


_spec = importlib.util.spec_from_file_location(
    '_tfrbert_fp16_replay', os.path.join(os.path.dirname(os.path.abspath(__file__)),
                                         '_tfrbert_bf16_refs.py'))
F = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(F)
F.bf16 = fp16


def bars(L, E, I, NL):
  """(score bar, gradient bar) of the kernels against F.forward, relative."""
  u = U_FP16 + max(L, E, I, 3 * E) * U_ACC
  fwd_sites = 9 * NL + 2
  return C_SAFETY * fwd_sites * u, C_SAFETY * (fwd_sites + 8 * NL + 2) * u


def attn_bars(qkv, mask, H, dO, O, adrop, seed, site, unit=2.0 ** -10):
  """Per-element bars {O, dQ, dK, dV} of the 16-bit attention core against F.attention; the
  derivation is _tfrbert_bf16_refs.attn_bars' with `unit` (one unit of the rounded value:
  2^-10 for fp16, 2^-7 for bf16) in place of 2^-7 and 2 units in place of 2^-6."""
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
  u = unit + 2.0 ** -23 * (2 * L + 4 + dh * (1 + lrow))
  w = 2 * unit + 2.0 ** -23 * (2 * L + 4 + dh * (3 + lrow))
  dabs = (g.abs() * o.abs()).sum(-1, keepdim=True)
  a = p * (ka * (g.abs() @ v.abs().transpose(-1, -2)) + dabs)
  dp = g @ v.transpose(-1, -2)
  ds = p * (dp * ka - (g * o).sum(-1, keepdim=True))
  t = {'O': (o, (u * pt.abs()) @ v.abs()),
       'dV': (pt.transpose(-1, -2) @ g, (u * pt.abs()).transpose(-1, -2) @ g.abs()),
       'dQ': (scale * ds @ k, scale * (w * a) @ k.abs()),
       'dK': (scale * ds.transpose(-1, -2) @ q, scale * (w * a).transpose(-1, -2) @ q.abs())}
  return {name: (unit * val.abs() + terms).transpose(1, 2).reshape(S, L, E)
          for name, (val, terms) in t.items()}


class LossScale(object):
  """The header's dynamic loss scale rule (Keras' LossScaleOptimizer(dynamic=True)), one step
  at a time: `step(finite)` returns whether the update applies and advances t either way.
  growth_steps 0 is a fixed scale (never changes; a non-finite step is still skipped)."""

  def __init__(self, initial=2.0 ** 15, growth_steps=2000):
    self.scale = float(initial)
    self.good = 0
    self.t = 0
    self.growth_steps = growth_steps

  def step(self, finite):
    self.t += 1
    if self.growth_steps == 0:
      return finite
    if not finite:
      self.scale = max(self.scale / 2.0, 1.0)
      self.good = 0
      return False
    self.good += 1
    if self.good >= self.growth_steps:
      grown = float(torch.tensor(self.scale * 2.0, dtype=torch.float32))   # a float32 scale
      if math.isfinite(grown):
        self.scale = grown
      self.good = 0
    return True


def adamw_fp64(p, m, v, g, lr, t, beta1=0.9, beta2=0.999, eps=1e-6, wd=0.01, decay=None):
  """One AdamW step (tfr_adamw_step's formula) in fp64 on gradient g; returns (p, m, v)."""
  p, m, v, g = p.double(), m.double(), v.double(), g.double()
  m = beta1 * m + (1 - beta1) * g
  v = beta2 * v + (1 - beta2) * g * g
  d = torch.ones_like(p) if decay is None else decay.double()
  p = p - lr * wd * p * d
  step = lr * math.sqrt(1 - beta2 ** t) / (1 - beta1 ** t)
  return p - step * m / (v.sqrt() + eps), m, v
