"""TFR-BERT's fp16 mode on the CPU: the fp16 replay (tests/_tfrbert_fp16_refs.py) with its rounding
switched off is the unrounded reference and rounds to fp16 with it on; the precision plumbing and
the fp16 limits are rejected before any CUDA call; the loss-scaling entry points check their
arguments before any CUDA call; the trainer's loss-scale arguments; and the pure-Python model of
the dynamic loss scale rule over a scripted sequence of finite and non-finite steps."""
import ctypes
import math

import pytest
import torch

import _tfrbert_fp16_refs as H
import _tfrbert_refs as R
from ranking_b200 import _C
from ranking_b200 import train
from ranking_b200.extension import tfrbert
from ranking_b200.keras import losses

V, P, TV = 31, 16, 2
FAKE = ctypes.c_void_p(1 << 20)   # a device pointer that is never dereferenced


def _case(S=3, L=6, E=16, I=24, NL=2, seed=0):
  g = torch.Generator().manual_seed(seed)
  wid = torch.randint(0, V, (S, L), generator=g, dtype=torch.int32)
  tid = torch.randint(0, TV, (S, L), generator=g, dtype=torch.int32)
  mask = (torch.rand(S, L, generator=g) < 0.7).to(torch.uint8)
  mask[:, 0] = 1
  mask[-1] = 0
  flat = 0.3 * torch.randn(R.param_count(V, E, I, NL, P, TV), generator=g, dtype=torch.float64)
  return wid, mask, tid, flat


def _grad(fn, flat, dscores, **kw):
  f = flat.clone().requires_grad_()
  s = fn(f, **kw)
  (s * dscores).sum().backward()
  return s.detach(), f.grad


def test_replay_without_rounding_is_the_unrounded_reference():
  E, Hh, I, NL = 16, 2, 24, 2
  wid, mask, tid, flat = _case(E=E, I=I, NL=NL)
  dscores = torch.randn(wid.shape[0], generator=torch.Generator().manual_seed(1),
                        dtype=torch.float64)
  kw = dict(training=True, hdrop=0.1, adrop=0.2, sdrop=0.1, seed=77)
  s0, g0 = _grad(lambda f, **k: R.forward(wid, mask, tid, f, V, E, Hh, I, NL, P, TV, **k), flat,
                 dscores, **kw)
  s1, g1 = _grad(lambda f, **k: H.F.forward(wid, mask, tid, f, V, E, Hh, I, NL, P, TV,
                                            rounding=False, **k), flat, dscores, **kw)
  assert torch.equal(s0, s1)
  assert torch.equal(g0, g1)
  # the fp16 rounding moves both, less than bf16 rounding does
  s2, g2 = _grad(lambda f, **k: H.F.forward(wid, mask, tid, f, V, E, Hh, I, NL, P, TV, **k),
                 flat, dscores, **kw)
  s3, g3 = _grad(lambda f, **k: H.B.forward(wid, mask, tid, f, V, E, Hh, I, NL, P, TV, **k),
                 flat, dscores, **kw)
  d16 = float((s2 - s0).norm() / s0.norm()), float((g2 - g0).norm() / g0.norm())
  dbf = float((s3 - s0).norm() / s0.norm()), float((g3 - g0).norm() / g0.norm())
  assert 1e-7 < d16[0] < dbf[0] and 1e-7 < d16[1] < dbf[1], (d16, dbf)


def test_fp16_rounding_and_the_second_replay_module():
  x = torch.randn(1000, dtype=torch.float64, generator=torch.Generator().manual_seed(2)) * 7.0
  want = x.float().half().double()
  assert torch.equal(H.fp16(x), want)
  assert torch.equal(H.F.bf16(x), want)   # the replay module rounds to fp16 ...
  assert torch.equal(H.B.bf16(x), x.to(torch.bfloat16).double())   # ... the bf16 one is as it was
  # out of range and subnormal: inf past 65504 (from 65520 up), subnormals kept
  big = torch.tensor([65504.0, 65519.0, 65520.0, -1e6, 2.0 ** -24, 2.0 ** -25, 3 * 2.0 ** -26],
                     dtype=torch.float64)
  got = H.fp16(big)
  assert got[0] == 65504.0 and got[1] == 65504.0
  assert got[2] == math.inf and got[3] == -math.inf
  assert got[4] == 2.0 ** -24 and got[5] == 0.0 and got[6] == 2.0 ** -24
  xg = x.clone().requires_grad_()
  y = H.F.round_both(xg)
  y.backward(x)
  assert torch.equal(y.detach(), want) and torch.equal(xg.grad, want)


def test_bars_use_the_fp16_unit():
  s16, g16 = H.bars(64, 768, 3072, 2)
  sbf, gbf = H.B.bars(64, 768, 3072, 2)
  u16 = 2.0 ** -11 + 3072 * 2.0 ** -23
  assert s16 == 2 * 20 * u16 and g16 == 2 * (20 + 16 + 2) * u16
  assert s16 < sbf and g16 < gbf


def test_precision_plumbing_and_parameters():
  cfg = tfrbert.BertEncoderConfig(vocab_size=50, hidden_size=64, num_layers=2,
                                  num_attention_heads=4, intermediate_size=136,
                                  max_position_embeddings=32, type_vocab_size=2)
  a = tfrbert.BertEncoder(cfg, seed=4, device='cpu', precision='fp32')
  b = tfrbert.BertEncoder(cfg, seed=4, device='cpu', precision='fp16')
  assert _C.PREC_FP16 == 4
  assert b.precision == 'fp16' and b._precision == _C.PREC_FP16
  assert torch.equal(a.flat.detach(), b.flat.detach())
  assert torch.equal(a.decay_mask, b.decay_mask)
  a.set_precision('fp16')
  assert a.precision == 'fp16'
  a.set_precision('bf16')
  assert a.precision == 'bf16'
  with pytest.raises(ValueError):
    a.set_precision('float16')
  assert a.precision == 'bf16'


def test_fp16_limits_before_any_cuda_call():
  """E, I or the head size not a multiple of 8: ValueError in Python, TFR_INVALID_ARGUMENT from
  every entry, and no launch."""
  n0 = _C.lib.tfr_launch_count()
  for e, h, i in [(60, 3, 128), (64, 4, 100), (96, 8, 128)]:   # E, I, head size 12
    cfg = tfrbert.BertEncoderConfig(vocab_size=50, hidden_size=e, num_layers=1,
                                    num_attention_heads=h, intermediate_size=i,
                                    max_position_embeddings=32, type_vocab_size=2)
    with pytest.raises(ValueError, match='multiples of 8'):
      tfrbert.BertEncoder(cfg, seed=1, device='cpu', precision='fp16')
    enc = tfrbert.BertEncoder(cfg, seed=1, device='cpu', precision='fp32')
    with pytest.raises(ValueError, match='TFR_PREC_FP16'):
      enc.set_precision('fp16')
    assert enc.precision == 'fp32' and enc._precision == _C.PREC_FP32
    c = enc._make_cfg(0.0)
    c.precision = _C.PREC_FP16
    assert _C.lib.tfr_bert_param_count(ctypes.byref(c)) == 0
    assert _C.lib.tfr_bert_workspace_bytes(ctypes.byref(c), 2, 4) == 0
    assert _C.lib.tfr_bert_fwd(FAKE, FAKE, FAKE, 2, 4, ctypes.byref(c), FAKE, FAKE, FAKE, None,
                               None) == 1
    assert _C.lib.tfr_bert_bwd(FAKE, FAKE, FAKE, 2, 4, ctypes.byref(c), FAKE, FAKE, FAKE, FAKE,
                               None) == 1
  # an unknown precision is still refused, with FP16 among those named
  c.precision = 5
  assert _C.lib.tfr_bert_param_count(ctypes.byref(c)) == 0
  assert 'TFR_PREC_FP16 (4)' in _C.last_error()
  assert _C.lib.tfr_launch_count() == n0


def test_other_entry_points_refuse_fp16_before_any_cuda_call():
  n0 = _C.lib.tfr_launch_count()
  cfg = _C.MlpCfg()
  cfg.n_dense = 2
  for i, d in enumerate([16, 8, 1]):
    cfg.dims[i] = d
  assert _C.lib.tfr_mlp_fwd_tasks(FAKE, 4, ctypes.byref(cfg), FAKE, None, FAKE, FAKE,
                                  _C.PREC_FP16, None) == 1
  assert _C.lib.tfr_mlp_input_grad(ctypes.byref(cfg), 4, FAKE, FAKE, 0, 1, FAKE, 1,
                                   _C.PREC_FP16, None) == 1
  assert _C.lib.tfr_launch_count() == n0


def test_loss_scale_entries_check_arguments_before_any_cuda_call():
  n0 = _C.lib.tfr_launch_count()
  L = _C.lib
  assert L.tfr_loss_scale_mul(FAKE, 4, None, FAKE, None) == 1
  assert L.tfr_loss_scale_mul(None, 4, FAKE, FAKE, None) == 1
  assert L.tfr_loss_scale_mul(None, 0, FAKE, FAKE, None) == 0   # nothing to do
  good = [FAKE, FAKE, FAKE, FAKE, None, 8, 1e-3, 0.9, 0.999, 1e-6, 0.01, 1, 0.0, FAKE, FAKE, None]
  assert L.tfr_adamw_step_scaled(*good[:5], 0, *good[6:]) == 0   # n = 0: nothing to do
  for i, bad in [(0, None), (13, None), (14, None), (11, 0), (7, 1.0), (12, -1.0),
                 (12, float('inf')), (12, float('nan'))]:
    args = list(good)
    args[i] = bad
    assert L.tfr_adamw_step_scaled(*args) == 1, (i, bad)
  assert L.tfr_loss_scale_update(None, FAKE, FAKE, None, 2000, None) == 1
  assert L.tfr_loss_scale_update(FAKE, FAKE, None, None, 2000, None) == 1
  assert L.tfr_loss_scale_update(FAKE, None, FAKE, None, 2000, None) == 1   # dynamic needs c
  assert L.tfr_loss_scale_update(FAKE, FAKE, FAKE, None, -1, None) == 1
  assert L.tfr_launch_count() == n0


def _trainer(precision='fp16', **kw):
  cfg = tfrbert.BertEncoderConfig(vocab_size=50, hidden_size=64, num_layers=1,
                                  num_attention_heads=4, intermediate_size=128,
                                  max_position_embeddings=32, type_vocab_size=2)
  enc = tfrbert.BertEncoder(cfg, seed=1, device='cpu', precision=precision)
  return tfrbert.TFRBertRankingTrainer(tfrbert.TFRBertScorer(enc, 0.0),
                                       losses.get('softmax_loss'), **kw)


def test_trainer_loss_scale_arguments():
  tr = _trainer()
  assert float(tr.loss_scale) == 2.0 ** 15 and tr.loss_scale.dtype == torch.float32
  assert int(tr.good_steps) == 0 and tr.good_steps.dtype == torch.int64
  assert tr.dynamic_growth_steps == 2000
  tr = _trainer(loss_scale=128.0)
  assert float(tr.loss_scale) == 128.0 and tr.dynamic_growth_steps == 0
  tr = _trainer(initial_loss_scale=2 ** 10, dynamic_growth_steps=3)
  assert float(tr.loss_scale) == 1024.0 and tr.dynamic_growth_steps == 3
  tr.loss_scale.fill_(8.0)
  tr.good_steps.fill_(2)
  tr.reset_loss_scale()
  assert float(tr.loss_scale) == 1024.0 and int(tr.good_steps) == 0
  for kw in [dict(loss_scale='static'), dict(loss_scale=0.0), dict(loss_scale=float('inf')),
             dict(initial_loss_scale=0.5), dict(initial_loss_scale=float('nan')),
             dict(dynamic_growth_steps=0)]:
    with pytest.raises(ValueError):
      _trainer(**kw)


def test_trainer_fp16_needs_adamw():
  with pytest.raises(ValueError, match='adamw'):
    _trainer(optimizer='adagrad')
  _trainer(precision='bf16', optimizer='adagrad')   # the other precisions keep every optimizer


def test_loss_scale_rule_over_a_scripted_sequence():
  """Growth at the boundary, halving, the floor at 1, a fixed scale, and t advancing on a
  skipped step (with a schedule's learning rate, which is read at t)."""
  ls = H.LossScale(initial=8.0, growth_steps=3)
  applied = [ls.step(f) for f in (True, True)]
  assert applied == [True, True] and ls.scale == 8.0 and ls.good == 2
  assert ls.step(True) and ls.scale == 16.0 and ls.good == 0     # the third: doubles
  assert not ls.step(False) and ls.scale == 8.0 and ls.good == 0
  assert ls.step(True) and ls.step(True) and ls.good == 2
  assert not ls.step(False) and ls.scale == 4.0 and ls.good == 0  # a skip resets the count
  for _ in range(5):
    assert not ls.step(False)
  assert ls.scale == 1.0                                          # the floor
  assert ls.t == 12   # 5 applied, 7 skipped, every one counted
  # a schedule sees t advance through skipped steps: the next update's lr is lr(12), past
  # the warmup, not lr(5)
  sched = train.PolynomialWarmUp(1e-3, 100, 10)
  assert sched(ls.t) == pytest.approx(1e-3 * (1 - 12 / 100))
  # growth stops at the largest finite float32 power of two
  top = H.LossScale(initial=2.0 ** 127, growth_steps=1)
  assert top.step(True) and top.scale == 2.0 ** 127 and top.good == 0
  # a fixed scale never changes; a non-finite step is skipped
  fixed = H.LossScale(initial=100.0, growth_steps=0)
  assert [fixed.step(f) for f in (True, False, True)] == [True, False, True]
  assert fixed.scale == 100.0 and fixed.t == 3


def test_adamw_fp64_reference_matches_the_header_formula():
  p = torch.tensor([1.0, -2.0])
  g = torch.tensor([0.5, 0.25])
  p1, m1, v1 = H.adamw_fp64(p, torch.zeros(2), torch.zeros(2), g, 1e-2, 1, wd=0.1)
  m = (1 - 0.9) * g.double()
  v = (1 - 0.999) * g.double() ** 2
  want = p.double() * (1 - 1e-3) - 1e-2 * math.sqrt(1 - 0.999) / (1 - 0.9) * m / (v.sqrt() + 1e-6)
  assert torch.allclose(p1, want, rtol=0, atol=1e-15)
  assert torch.equal(m1, m) and torch.equal(v1, v)
