"""TFR-BERT's bf16 mode on the CPU: the fp64 replay (tests/_tfrbert_bf16_refs.py) with its
rounding switched off is the unrounded reference, its rounding functions round to bf16, and a
bf16 encoder has the fp32 encoder's parameters."""
import torch

import _tfrbert_bf16_refs as B
import _tfrbert_refs as R
from ranking_b200 import _C
from ranking_b200.extension import tfrbert

V, P, TV = 31, 16, 2


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
  E, H, I, NL = 16, 2, 24, 2
  wid, mask, tid, flat = _case(E=E, I=I, NL=NL)
  dscores = torch.randn(wid.shape[0], generator=torch.Generator().manual_seed(1),
                        dtype=torch.float64)
  kw = dict(training=True, hdrop=0.1, adrop=0.2, sdrop=0.1, seed=77)
  s0, g0 = _grad(lambda f, **k: R.forward(wid, mask, tid, f, V, E, H, I, NL, P, TV, **k), flat,
                 dscores, **kw)
  s1, g1 = _grad(lambda f, **k: B.forward(wid, mask, tid, f, V, E, H, I, NL, P, TV,
                                          rounding=False, **k), flat, dscores, **kw)
  assert torch.equal(s0, s1)
  assert torch.equal(g0, g1)
  # and the rounding moves both, by about the bf16 unit
  s2, g2 = _grad(lambda f, **k: B.forward(wid, mask, tid, f, V, E, H, I, NL, P, TV, **k), flat,
                 dscores, **kw)
  ds = float((s2 - s0).norm() / s0.norm())
  dg = float((g2 - g0).norm() / g0.norm())
  assert 1e-5 < ds < 0.1 and 1e-5 < dg < 0.1, (ds, dg)


def test_rounding_functions_round_trip_through_bfloat16():
  x = torch.randn(1000, dtype=torch.float64, generator=torch.Generator().manual_seed(2)) * 7.0
  want = x.to(torch.bfloat16).double()
  assert torch.equal(B.bf16(x), want)
  assert torch.equal(B.bf16(want), want)   # idempotent
  for fn, fwd_rounds, bwd_rounds in [(B.round_both, True, True), (B.round_grad, False, True),
                                     (B.round_value, True, False)]:
    xg = x.clone().requires_grad_()
    y = fn(xg)
    assert torch.equal(y.detach(), want if fwd_rounds else x)
    g = torch.randn(1000, dtype=torch.float64, generator=torch.Generator().manual_seed(3))
    y.backward(g)
    assert torch.equal(xg.grad, g.to(torch.bfloat16).double() if bwd_rounds else g)


def test_bf16_encoder_has_the_fp32_parameters():
  cfg = tfrbert.BertEncoderConfig(vocab_size=50, hidden_size=64, num_layers=2,
                                  num_attention_heads=4, intermediate_size=136,
                                  max_position_embeddings=32, type_vocab_size=2)
  a = tfrbert.BertEncoder(cfg, seed=4, device='cpu', precision='fp32')
  b = tfrbert.BertEncoder(cfg, seed=4, device='cpu', precision='bf16')
  assert b.precision == 'bf16' and b._precision == _C.PREC_BF16
  assert a.flat.numel() == b.flat.numel()
  assert torch.equal(a.flat.detach(), b.flat.detach())
  assert torch.equal(a.decay_mask, b.decay_mask)
  assert a.weight_names() == b.weight_names()
  assert a.flat.numel() == R.param_count(50, 64, 136, 2, 32, 2)
  a.set_precision('bf16')
  assert a.precision == 'bf16'


def test_bf16_limits_are_rejected_in_python():
  for e, h, i in [(60, 3, 128), (64, 4, 100), (96, 8, 128)]:   # E, I, head size 12
    cfg = tfrbert.BertEncoderConfig(vocab_size=50, hidden_size=e, num_layers=1,
                                    num_attention_heads=h, intermediate_size=i,
                                    max_position_embeddings=32, type_vocab_size=2)
    try:
      tfrbert.BertEncoder(cfg, seed=1, device='cpu', precision='bf16')
    except ValueError as err:
      assert 'multiples of 8' in str(err), err
    else:
      raise AssertionError('accepted E %d, I %d, heads %d in bf16' % (e, i, h))
    enc = tfrbert.BertEncoder(cfg, seed=1, device='cpu', precision='fp32')
    try:
      enc.set_precision('bf16')
    except ValueError:
      pass
    else:
      raise AssertionError('set_precision accepted bf16')
    assert enc.precision == 'fp32' and enc._precision == _C.PREC_FP32
