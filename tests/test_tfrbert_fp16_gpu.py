"""TFR-BERT's fp16 mode on the GPU (K15, TFR_PREC_FP16) and its dynamic loss scaling:

  * the fp16 GEMM entry (tfr_tc_gemm_f16) at the bf16 engine tests' tile edges, epilogues and
    split counts, against fp64 of the same fp16 inputs with fp16 output rounding;
  * the fp16 attention core (tfr_attn_f16_*) at every head bucket and N 1 .. 1024 with an
    all-padded list, against the fp16 replay with fp16-unit bars;
  * tfr_bert_fwd / _bwd in fp16 over the bf16 case table against the fp16 replay
    (tests/_tfrbert_fp16_refs.py), and negative controls: the bf16 replay, and a gradient left
    scaled, fail the bar;
  * loss scaling: an input whose fp16 backward signals underflow at S = 1 and not at 2^15;
    overflow skips the step bit for bit and halves S; growth after dynamic_growth_steps;
    clipped and unclipped scaled AdamW against the fp64 composition; determinism;
  * training, checkpoint resume with the scale, the hf_tiny fixture and the example script."""
import ctypes
import math

import pytest
import torch

import _tfrbert_fp16_refs as H
import _tfrbert_refs as R
import test_attn_bf16_gpu as A
import test_tc_gemm_bf16_gpu as G
import test_tfrbert_bf16_gpu as TB
import test_tfrbert_gpu as T
from ranking_b200 import _C
from ranking_b200 import pipeline
from ranking_b200 import train
from ranking_b200.extension import tfrbert

pytestmark = pytest.mark.gpu

V, P, TV = T.V, T.P, T.TV
U16 = 2.0 ** -11


# ------------------------------------------------------------------------- GEMM entry ---
def _gemm_kmajor(gm, gn, gk, epi=0, act=0, want_bits=False, want_colsum=False, seed=0, lda=None,
                 ldc=None):
  """mn = 0 through tfr_tc_gemm_f16 (G.run_kmajor with fp16): error past one fp16 rounding of
  the output, relative to |A||B|; columns past GN keep their sentinel."""
  g = torch.Generator().manual_seed(seed)
  lda, ldc = lda or gk, ldc or gn
  A_full = torch.randn(gm, lda, generator=g).half()
  A_full[:, gk:] = 1e4
  Am = A_full[:, :gk]
  Bm = torch.randn(gn, gk, generator=g).half()
  bias = torch.randn(gn, generator=g)
  keep = torch.rand(gm, gn, generator=g) > 0.4
  ref = Am.double() @ Bm.double().t()
  scale = Am.double().abs() @ Bm.double().abs().t()
  if epi == 1:
    ref = ref + bias.double()
    if act == 1:
      ref = torch.relu(ref)
  elif epi == 3:
    ref = torch.where(keep, ref, torch.zeros_like(ref))
  C = torch.full((gm, ldc), G.SENTINEL, dtype=torch.float16, device='cuda')
  C[:, :gn] = float('nan')
  bits_out = bits_in = colsum = None
  nslots = ctypes.c_int(0)
  if want_bits:
    bits_out = torch.full(((gn + 31) // 32, gm), -1, dtype=torch.int32, device='cuda')
  if epi == 3:
    bits_in = G._pack_bits(keep).cuda()
  stride = (gn + 63) // 64 * 64
  if want_colsum:
    colsum = torch.full((148 * 8, stride), float('nan'), device='cuda')
  a_d, b_d, bias_d = A_full.cuda(), Bm.cuda(), bias.cuda()
  _C.check(_C.lib.tfr_tc_gemm_f16(
      _C.ptr(a_d), lda, _C.ptr(b_d), gk, _C.ptr(C), ldc, gm, gn, gk, 0, epi, _C.ptr(bias_d),
      act, _C.ptr(bits_out), _C.ptr(bits_in), _C.ptr(colsum), stride,
      ctypes.cast(ctypes.byref(nslots), ctypes.c_void_p), 1, 0, _C.stream()))
  torch.cuda.synchronize()
  assert (C[:, gn:].float() == G.SENTINEL).all(), 'columns past GN written'
  out = C[:, :gn].double().cpu()
  err = float(((out - ref).abs() - U16 * ref.abs()).clamp(min=0).div(scale + 1e-30).max())
  if want_bits:
    assert torch.equal(bits_out.cpu(), G._pack_bits(C[:, :gn].float().cpu() > 0))
  if want_colsum:
    cs = colsum[:nslots.value, :gn].double().sum(0).cpu()
    assert float(((cs - ref.sum(0)).abs() / (scale.sum(0) + 1e-30)).max()) <= 1e-5
  return err


def _gemm_mnmajor(gm, gn, gk, splits, seed=0, lda=None, ldc=None):
  g = torch.Generator().manual_seed(seed)
  lda, ldc = lda or gm, ldc or gn
  A_full = torch.randn(gk, lda, generator=g).half()
  A_full[:, gm:] = 1e4
  Am = A_full[:, :gm]
  Bm = torch.randn(gk, gn, generator=g).half()
  ref = Am.double().t() @ Bm.double()
  scale = Am.double().abs().t() @ Bm.double().abs()
  rows = (gm + 127) // 128 * 128
  C = torch.full((splits, rows, ldc), G.SENTINEL, device='cuda')
  C[:, :gm, :gn] = float('nan')
  a_d, b_d = A_full.cuda(), Bm.cuda()
  _C.check(_C.lib.tfr_tc_gemm_f16(
      _C.ptr(a_d), lda, _C.ptr(b_d), gn, _C.ptr(C), ldc, gm, gn, gk, 1, 0, None, 0, None, None,
      None, 0, None, splits, rows * ldc, _C.stream()))
  torch.cuda.synchronize()
  assert (C[:, :, gn:] == G.SENTINEL).all(), 'columns past GN written'
  out = C[:, :gm, :gn].double().sum(0).cpu()
  return float(((out - ref).abs() / (scale + 1e-30)).max())


@pytest.mark.parametrize('shape', G.KM_SHAPES)
def test_f16_gemm_kmajor_and_epilogues(shape):
  s = sum(shape)
  errs = [_gemm_kmajor(*shape, seed=s),
          _gemm_kmajor(*shape, epi=1, act=1, want_bits=True, seed=1 + s),
          _gemm_kmajor(*shape, epi=1, act=0, seed=2 + s),
          _gemm_kmajor(*shape, epi=3, act=1, want_colsum=True, seed=3 + s)]
  assert max(errs) <= 1e-5, errs


@pytest.mark.parametrize('shape', G.MN_SHAPES)
def test_f16_gemm_mnmajor(shape):
  err = _gemm_mnmajor(*shape, seed=sum(shape))
  assert err <= 2e-6, err


@pytest.mark.parametrize('shape', G.BERT_KM, ids=G._bert_id)
def test_f16_gemm_kmajor_bert_calls(shape):
  gm, gn, gk, lda, ldc, bias = shape
  err = _gemm_kmajor(gm, gn, gk, epi=1 if bias else 0, seed=gm + gn + gk, lda=lda, ldc=ldc)
  assert err <= 1e-5, err


@pytest.mark.parametrize('shape', G.BERT_MN, ids=G._bert_id)
def test_f16_gemm_mnmajor_bert_calls(shape):
  gm, gn, gk, lda, ldc, splits = shape
  splits = splits or G.dw_splits(132, gm, gn, gk)
  err = _gemm_mnmajor(gm, gn, gk, splits, seed=gm + gn + gk, lda=lda, ldc=ldc)
  assert err <= 2e-6, err


def test_f16_gemm_overflow_is_inf_not_clamped():
  """A product past 65504 is stored as inf (bias epilogue and plain store), not clamped."""
  a = torch.full((128, 64), 64.0, dtype=torch.float16, device='cuda')
  b = torch.full((64, 64), 32.0, dtype=torch.float16, device='cuda')   # sums to 131072
  bias = torch.zeros(64, device='cuda')
  for epi in (0, 1):
    c = torch.zeros(128, 64, dtype=torch.float16, device='cuda')
    _C.check(_C.lib.tfr_tc_gemm_f16(_C.ptr(a), 64, _C.ptr(b), 64, _C.ptr(c), 64, 128, 64, 64, 0,
                                    epi, _C.ptr(bias), 0, None, None, None, 0, None, 1, 0,
                                    _C.stream()))
    torch.cuda.synchronize()
    assert torch.isinf(c.float()).all() and (c.float() > 0).all(), epi


# ----------------------------------------------------------------- attention core ---
# (B, N, H, h, mask, dropout, sigma): every head bucket (16 / 32 / 64 / 128, a padded head
# size in two), N 1, 63, 64, 65, 512 and 1024, ragged lists with an all-padded one
ATTN_CASES = [(3, 1, 2, 8, 'ragged', 0.0, 1.0),
              (3, 63, 2, 24, 'ragged', 0.2, 1.0),
              (2, 64, 3, 32, 'null', 0.0, 1.0),
              (3, 65, 2, 40, 'ragged', 0.1, 1.0),
              (2, 512, 4, 16, 'padded', 0.0, 1.0),
              (3, 65, 2, 120, 'ragged', 0.0, 4.0),
              (3, 512, 2, 128, 'ragged', 0.1, 1.0),
              (1, 1024, 16, 64, 'ragged', 0.1, 1.0)]


def _attn_inputs(case, seed=0):
  qkv, mask, dO = A._inputs(case, seed)
  return qkv.float().half(), mask, dO.float().half()


def _attn_kernel(case, qkv, mask, dO):
  b, n, H, h, _, drop, _ = case
  E, m = H * h, b * n
  seed, site = A._seed(case)
  q, d = qkv.cuda().contiguous(), dO.cuda().contiguous()
  lm = None if mask is None else mask.reshape(-1).cuda()
  O = torch.full((m * E,), float('nan'), dtype=torch.float16, device='cuda')
  lse = torch.full((m * H * 2,), float('nan'), device='cuda')
  dsum = torch.full((m * H,), float('nan'), device='cuda')
  dqkv = torch.full((m * 3 * E,), float('nan'), dtype=torch.float16, device='cuda')
  ds = A._dseed(seed, site)
  _C.check(_C.lib.tfr_attn_f16_fwd(_C.ptr(q), _C.ptr(lm), b, n, H, h, drop, ds, _C.ptr(O),
                                   _C.ptr(lse), _C.stream()))
  _C.check(_C.lib.tfr_attn_f16_bwd(_C.ptr(q), _C.ptr(lm), b, n, H, h, drop, ds, _C.ptr(O),
                                   _C.ptr(lse), _C.ptr(d), _C.ptr(dsum), _C.ptr(dqkv),
                                   _C.stream()))
  torch.cuda.synchronize()
  for t in (O, lse, dsum, dqkv):
    assert not torch.isnan(t.float()).any(), 'unwritten elements'
  return O.reshape(b, n, E), dqkv.reshape(b, n, 3 * E)


def _attn_replay(case, qkv, mask, dO, dev, attention=None, rounding=True):
  b, n, nh, _, _, drop, _ = case
  seed, site = A._seed(case)
  x = qkv.to(dev).double().requires_grad_()
  m = torch.ones(b, n, dtype=torch.uint8) if mask is None else mask
  o = (attention or H.F.attention)(x, m, nh, drop, seed, site, rounding=rounding)
  o.backward(dO.to(dev).double())
  g = H.fp16(x.grad) if rounding else x.grad
  return o.detach(), g


@pytest.mark.parametrize('case', ATTN_CASES, ids=A._id)
def test_f16_attention_core_against_the_fp16_replay(case):
  b, n, nh, h, kind, drop, _ = case
  E = nh * h
  qkv, mask, dO = _attn_inputs(case)
  got_o, got_g = _attn_kernel(case, qkv, mask, dO)
  again_o, again_g = _attn_kernel(case, qkv, mask, dO)
  assert torch.equal(got_o, again_o) and torch.equal(got_g, again_g)
  dev = A._dev(case)
  rep_o, rep_g = _attn_replay(case, qkv, mask, dO, dev)
  bars = H.attn_bars(qkv.to(dev).double(), mask, nh, dO.to(dev).double(), rep_o, drop,
                     *A._seed(case))
  gt = A._tensors(got_o.to(dev).double(), got_g.to(dev).double(), E)
  rt = A._tensors(rep_o, rep_g, E)
  worst = {}
  for k in gt:
    err = (gt[k] - rt[k]).abs()
    worst[k] = float((err / bars[k].clamp(min=1e-300)).max())
    assert (err <= bars[k]).all(), (k, worst[k])
  # the bf16 replay (rounding at the bf16 points) sits outside the fp16 bars somewhere (not
  # in the all-padded lists: P~ = 1 / N is exact in both, and O's bar is dominated there by
  # the fp32 terms of its N-term sum)
  if n > 1 and kind != 'padded':
    bo, bg = _attn_replay(case, qkv, mask, dO, dev, attention=H.B.attention)
    bt = A._tensors(bo, H.B.bf16(bg), E)
    assert any(((gt[k] - bt[k]).abs() > bars[k]).any() for k in gt)
  print('[attn fp16 %s] err/bar %s' % (A._id(case),
                                       ' '.join('%s %.3f' % kv for kv in worst.items())))


# --------------------------------------------------------------------- the encoder ---
def _cfg(E, Hh, I, NL, training, seed=1234, rates=T.RATES):
  return TB._cfg(E, Hh, I, NL, training, precision=_C.PREC_FP16, seed=seed, rates=rates)


def _replay(cfg, wid, mask, tid, flat, dscores, fwd=None, **kw):
  f = flat.double().clone().requires_grad_()
  s = (fwd or H.F.forward)(wid, mask, tid, f, V, cfg.hidden_size, cfg.num_heads,
                           cfg.intermediate_size, cfg.num_layers, P, TV,
                           training=bool(cfg.training), hdrop=cfg.hidden_dropout,
                           adrop=cfg.attention_dropout, sdrop=cfg.output_dropout, seed=cfg.seed,
                           **kw)
  (s * dscores.double()).sum().backward()
  return s.detach(), f.grad


# RMS ratio of the gradients, ||kernel - replay|| / ||unrounded - replay||.  fp16's rounding
# is 8x finer than bf16's while the roundings that flip between fp32 and fp64 accumulation stay
# one unit each, so the kernel's ratio is larger than in bf16 (the bf16 tests' 1/8 does not
# apply).  Measured over the case table on an H100 SXM (700 W power limit): kernel 0.001 -
# 0.86, the bf16 replay 7.3 - 9.5.
GRAD_RATIO = 2.0


@pytest.mark.parametrize('case', TB.CASES, ids=lambda c: 'S%d-L%d-E%d-H%d-I%d-NL%d' % c)
def test_forward_and_gradients_against_the_fp16_replay(case):
  """Loss-scaled, as the trainer calls it: dscores times S = 2^8 in, the gradient / S out,
  against the replay of the same scaled backward.  Negative controls: a gradient left scaled
  fails the bar; the bf16 replay lies within the max-error bars (they allow 2 fp16 units per
  rounding site on the longest path, about 5 bf16 units in all), so it is caught by the RMS
  ratio ||gradient - replay|| / ||unrounded - fp16 replay||: at most GRAD_RATIO for the
  kernel, more for the bf16 replay."""
  S, L, E, Hh, I, NL = case
  cfg = _cfg(E, Hh, I, NL, True)
  wid, mask, tid = T._inputs(S, L)
  flat = T._flat(E, I, NL)
  scale = 2.0 ** 8
  dscores = torch.randn(S, generator=torch.Generator().manual_seed(5))
  got_s, got_g, bad = T._run(cfg, wid, mask, tid, flat, dscores * scale)
  assert bad == 0 and torch.isfinite(got_s).all() and torch.isfinite(got_g).all()
  rep_s, rep_g = _replay(cfg, wid, mask, tid, flat, dscores * scale)
  sbar, gbar = H.bars(L, E, I, NL)
  es, eg = T._errors(cfg, got_s, got_g / scale, rep_s, rep_g / scale)
  worst = max(eg, key=eg.get)
  # negative controls: the bf16 replay, and the gradient left scaled
  bf_s, bf_g = _replay(cfg, wid, mask, tid, flat, dscores * scale, fwd=H.B.forward)
  ex_s, ex_g = T._reference(cfg, wid, mask, tid, flat, dscores * scale)

  def ratio(s, g):   # (scores, gradients) RMS distance over the fp16 rounding's own effect
    return (float((s.double() - rep_s).norm() / (ex_s - rep_s).norm()),
            float((g.double() - rep_g).norm() / (ex_g - rep_g).norm()))

  r_kernel = ratio(got_s, got_g)
  r_bf16 = (float((got_s.double() - bf_s).norm() / (ex_s - rep_s).norm()),
            float((got_g.double() - bf_g).norm() / (ex_g - rep_g).norm()))
  _, ueg = T._errors(cfg, got_s, got_g, rep_s, rep_g / scale)
  print('[bert fp16 %s] score err/bar %.3f, worst grad %s err/bar %.3f; RMS ratio kernel '
        '%.3f / %.3f, bf16 replay %.2f / %.2f; scaled gradient err/bar %.0f' %
        (case, es / sbar, worst, eg[worst] / gbar, r_kernel[0], r_kernel[1], r_bf16[0],
         r_bf16[1], max(ueg.values()) / gbar))
  assert es <= sbar, (es, sbar)
  assert eg[worst] <= gbar, (worst, eg[worst], gbar)
  assert r_kernel[1] <= GRAD_RATIO < r_bf16[1], (r_kernel, r_bf16)
  assert max(ueg.values()) > gbar
  g = R.unflatten(got_g, V, E, I, NL, P, TV)
  assert torch.equal(g['word'][12:], torch.zeros_like(g['word'][12:]))


def test_inference_and_determinism():
  S, L, E, Hh, I, NL = 4, 9, 64, 4, 136, 2
  cfg = _cfg(E, Hh, I, NL, False)
  wid, mask, tid = T._inputs(S, L)
  flat = T._flat(E, I, NL)
  dscores = torch.randn(S, generator=torch.Generator().manual_seed(6))
  s1, g1, _ = T._run(cfg, wid, mask, tid, flat, dscores)
  s2, g2, _ = T._run(cfg, wid, mask, tid, flat, dscores)
  assert torch.equal(s1, s2) and torch.equal(g1, g2)
  rep_s, rep_g = _replay(cfg, wid, mask, tid, flat, dscores)
  es, eg = T._errors(cfg, s1, g1, rep_s, rep_g)
  sbar, gbar = H.bars(L, E, I, NL)
  assert es <= sbar and max(eg.values()) <= gbar, (es, eg)


def test_loss_scale_lifts_underflowing_signals():
  """dscores of 2^-22: unscaled, the fp16 backward signals fall below fp16's normal range
  (2^-14) and lose their bits; at S = 2^15 they are normal.  Against the unrounded fp64
  gradient: within the bar at 2^15, outside it at 1."""
  S, L, E, Hh, I, NL = 4, 16, 64, 4, 136, 1
  cfg = _cfg(E, Hh, I, NL, False)
  wid, mask, tid = T._inputs(S, L)
  flat = T._flat(E, I, NL)
  dscores = torch.randn(S, generator=torch.Generator().manual_seed(7)) * 2.0 ** -22
  ex_s, ex_g = T._reference(cfg, wid, mask, tid, flat, dscores)
  _, gbar = H.bars(L, E, I, NL)
  err = {}
  for scale in (1.0, 2.0 ** 15):
    _, g, _ = T._run(cfg, wid, mask, tid, flat, dscores * scale)
    err[scale] = max(T._errors(cfg, ex_s, g / scale, ex_s, ex_g)[1].values())
  print('[bert fp16 underflow] grad err/bar: S = 1 %.2f, S = 2^15 %.3f' %
        (err[1.0] / gbar, err[2.0 ** 15] / gbar))
  assert err[2.0 ** 15] <= gbar
  assert err[1.0] > gbar


# ------------------------------------------------------------- the scaled update ---
def _norm(x):
  ws = torch.empty(_C.lib.tfr_global_norm_workspace_bytes(x.numel()), dtype=torch.uint8,
                   device='cuda')
  out = torch.zeros((), device='cuda')
  _C.check(_C.lib.tfr_global_norm(_C.ptr(x), x.numel(), _C.ptr(out), _C.ptr(ws), ws.numel(),
                                  _C.stream()))
  return out


@pytest.mark.parametrize('clip', [0.0, 1e-3, 1e9], ids=['unclipped', 'clipped', 'within'])
def test_scaled_adamw_against_fp64(clip):
  n = 100_003
  g = torch.Generator().manual_seed(11)
  p = torch.randn(n, generator=g)
  m = 0.01 * torch.randn(n, generator=g)
  v = 1e-4 * torch.rand(n, generator=g)
  gu = 1e-2 * torch.randn(n, generator=g)   # the unscaled gradient
  decay = (torch.rand(n, generator=g) < 0.7).to(torch.uint8)
  S = 2.0 ** 15
  gs = (gu.double() * S).float()            # exact: S is a power of two
  pd, md, vd, gd, dd = [t.cuda() for t in (p, m, v, gs, decay)]
  scale = torch.full((), S, device='cuda')
  norm = _norm(gd)
  lr, t = 1e-3, 7
  _C.check(_C.lib.tfr_adamw_step_scaled(_C.ptr(pd), _C.ptr(gd), _C.ptr(md), _C.ptr(vd),
                                        _C.ptr(dd), n, lr, 0.9, 0.999, 1e-6, 0.01, t, clip,
                                        _C.ptr(norm), _C.ptr(scale), _C.stream()))
  un = torch.full((), -1.0, device='cuda')
  good = torch.zeros((), dtype=torch.int64, device='cuda')
  _C.check(_C.lib.tfr_loss_scale_update(_C.ptr(scale), _C.ptr(good), _C.ptr(norm), _C.ptr(un),
                                        2000, _C.stream()))
  torch.cuda.synchronize()
  nu = float(gu.double().norm())
  assert abs(float(un) - nu) <= 1e-6 * nu
  assert float(scale) == S and int(good) == 1
  ge = gu.double()
  if clip > 0 and nu > clip:
    ge = ge * (clip / nu)
  pe, me, ve = H.adamw_fp64(p, m, v, ge, lr, t, decay=decay)
  for got, want in ((pd, pe), (md, me), (vd, ve)):
    err = float((got.cpu().double() - want).abs().max() / want.abs().max())
    assert err <= 1e-6, err
  if clip == 1e9:   # within the clip: the unclipped bits
    p2, m2, v2 = [t.cuda() for t in (p, m, v)]
    _C.check(_C.lib.tfr_adamw_step_scaled(_C.ptr(p2), _C.ptr(gd), _C.ptr(m2), _C.ptr(v2),
                                          _C.ptr(dd), n, lr, 0.9, 0.999, 1e-6, 0.01, t, 0.0,
                                          _C.ptr(norm), _C.ptr(scale), _C.stream()))
    assert torch.equal(p2, pd) and torch.equal(m2, md) and torch.equal(v2, vd)


def test_loss_scale_update_kernel_follows_the_rule():
  """The one-thread update against the Python model over a scripted norm sequence."""
  scale = torch.full((), 8.0, device='cuda')
  good = torch.zeros((), dtype=torch.int64, device='cuda')
  norm = torch.zeros((), device='cuda')
  model = H.LossScale(8.0, growth_steps=3)
  for x in [1.0, 2.0, 3.0, math.inf, 1.0, math.nan, 4.0, 4.0, 4.0, math.inf, math.inf,
            math.inf, math.inf, math.inf, 5.0]:
    norm.fill_(x)
    _C.check(_C.lib.tfr_loss_scale_update(_C.ptr(scale), _C.ptr(good), _C.ptr(norm), None, 3,
                                          _C.stream()))
    model.step(math.isfinite(x))
    assert float(scale) == model.scale and int(good) == model.good, x
  # a fixed scale (growth_steps 0) never changes
  norm.fill_(math.inf)
  _C.check(_C.lib.tfr_loss_scale_update(_C.ptr(scale), None, _C.ptr(norm), None, 0, _C.stream()))
  assert float(scale) == model.scale


# -------------------------------------------------------------------- the trainer ---
def _tr(dropout=0.0, seed=9, **kw):
  enc = T._small_encoder('fp16', seed=seed, dropout=dropout)
  return enc, tfrbert.TFRBertRankingTrainer(tfrbert.TFRBertScorer(enc, dropout), T._loss(),
                                            **kw)


def _state(tr):
  return [t.detach().clone() for t in (tr.scorer.flat, tr.accum)]


def test_overflow_skips_the_step_and_halves_the_scale():
  """A fixed huge initial scale overflows the fp16 backward (inf, not a fault): each such step
  leaves parameters and moments bit for bit, halves S, resets the count and still advances
  t; once S is small enough a step applies."""
  enc, tr = _tr(initial_loss_scale=2.0 ** 40, learning_rate=1e-3)
  wid, mask, tid, y = [t.cuda() for t in T._separable(2, 4, 8, seed=2)]
  skipped = 0
  for i in range(40):
    before = _state(tr)
    s0 = float(tr.loss_scale)
    tr.good_steps.fill_(1)
    tr.train_step(wid, mask, tid, y)
    torch.cuda.synchronize()
    assert tr.adam_step == i + 1
    after = _state(tr)
    if float(tr.loss_scale) == s0 / 2:
      assert all(torch.equal(a, b) for a, b in zip(before, after)), i
      assert int(tr.good_steps) == 0 and not math.isfinite(float(tr.grad_norm))
      skipped += 1
      continue
    assert float(tr.loss_scale) == s0 and int(tr.good_steps) == 2   # applied
    assert not torch.equal(before[0], after[0])
    break
  else:
    raise AssertionError('no step applied')
  print('[bert fp16 overflow] %d steps skipped from 2^40, applied at S = 2^%d' %
        (skipped, int(math.log2(float(tr.loss_scale)))))
  assert skipped >= 10


def test_scale_grows_after_growth_steps():
  _, tr = _tr(initial_loss_scale=2.0 ** 10, dynamic_growth_steps=3)
  wid, mask, tid, y = [t.cuda() for t in T._separable(2, 4, 8, seed=2)]
  seen = []
  for _ in range(7):
    tr.train_step(wid, mask, tid, y)
    seen.append((float(tr.loss_scale), int(tr.good_steps)))
  assert seen == [(1024.0, 1), (1024.0, 2), (2048.0, 0), (2048.0, 1), (2048.0, 2),
                  (4096.0, 0), (4096.0, 1)], seen


@pytest.mark.parametrize('clip', [None, 1e-4], ids=['unclipped', 'clipped'])
def test_trainer_step_is_the_fp64_composition_on_the_unscaled_gradient(clip):
  """One trainer step: the update equals the fp64 AdamW (clipped on the unscaled norm) of
  grads / S, and grad_norm is the unscaled norm."""
  enc, tr = _tr(gradient_clip_norm=clip, learning_rate=1e-3, initial_loss_scale=2.0 ** 10)
  wid, mask, tid, y = [t.cuda() for t in T._separable(2, 4, 8, seed=3)]
  p0 = tr.scorer.flat.detach().cpu().double()
  tr.train_step(wid, mask, tid, y)
  torch.cuda.synchronize()
  S = float(tr.loss_scale)
  g = tr.grads.cpu().double() / S
  nu = float(g.norm())
  assert abs(float(tr.grad_norm) - nu) <= 1e-5 * nu
  if clip is not None and nu > clip:
    g = g * (clip / nu)
  n = g.numel()
  pe, _, _ = H.adamw_fp64(p0, torch.zeros(n), torch.zeros(n), g, 1e-3, 1,
                          decay=tr.decay_mask.cpu())
  got = tr.scorer.flat.detach().cpu().double()
  # relative to the largest update, past the one fp32 rounding of the stored parameter
  err = float(((got - pe).abs() - 2.0 ** -24 * pe.abs()).clamp(min=0).max() /
              (pe - p0).abs().max())
  print('[bert fp16 step %s] update err %.2e, grad_norm %.4g' % (clip, err, nu))
  assert err <= 1e-4, err


def test_identical_runs_give_identical_bits():
  runs = []
  for _ in range(2):
    _, tr = _tr(dropout=0.1)
    wid, mask, tid, y = [t.cuda() for t in T._separable(2, 4, 8, seed=4)]
    for _ in range(3):
      tr.train_step(wid, mask, tid, y)
    runs.append(_state(tr) + [tr.loss_scale.clone()])
  assert all(torch.equal(a, b) for a, b in zip(*runs))


def _train(precision, steps=50):
  enc = T._small_encoder(precision)
  tr = tfrbert.TFRBertRankingTrainer(tfrbert.TFRBertScorer(enc, 0.0), T._loss(),
                                     learning_rate=train.PolynomialWarmUp(3e-3, 50, 5))
  wid, mask, tid, y = T._separable(4, 6, 10, seed=1)
  losses = [float(tr.train_step(wid.cuda(), mask.cuda(), tid.cuda(), y.cuda()))
            for _ in range(steps)]
  return enc, tr, losses


def test_training_tracks_fp32():
  _, _, l32 = _train('fp32')
  _, tr, l16 = _train('fp16')
  print('[bert fp16 train] fp32 loss %.4f -> %.4f, fp16 %.4f -> %.4f, final scale %g' %
        (l32[0], l32[-1], l16[0], l16[-1], float(tr.loss_scale)))
  assert l32[0] - l32[-1] > 0
  assert l16[0] - l16[-1] >= 0.9 * (l32[0] - l32[-1]), (l32, l16)
  assert max(abs(a - b) for a, b in zip(l32, l16)) <= 0.05 * l32[0]


def test_checkpoint_resume_is_bit_identical_in_fp16(tmp_path):
  wid, mask, tid, y = T._separable(2, 4, 8, seed=2)
  batches = [({'input_word_ids': wid, 'input_mask': mask, 'input_type_ids': tid}, y)] * 6

  def trainer():
    return _tr(dropout=0.1, learning_rate=train.PolynomialWarmUp(1e-3, 6, 2),
               initial_loss_scale=2.0 ** 30, dynamic_growth_steps=2)

  enc_a, a = trainer()
  pipeline.fit(a, iter(batches), 6, log_fn=lambda *_: None)
  enc_b, b = trainer()
  d = str(tmp_path / 'ck')
  pipeline.fit(b, iter(batches), 3, checkpoint_dir=d, log_fn=lambda *_: None)
  enc_c, c = trainer()
  enc_c._calls = enc_b._calls
  pipeline.fit(c, iter(batches), 6, checkpoint_dir=d, log_fn=lambda *_: None)
  assert c.adam_step == 6
  assert float(b.loss_scale) != 2.0 ** 30   # the scale moved before the checkpoint
  assert torch.equal(enc_a.flat.detach(), enc_c.flat.detach())
  assert torch.equal(a.accum, c.accum)
  assert torch.equal(a.loss_scale, c.loss_scale) and torch.equal(a.good_steps, c.good_steps)
  # a checkpoint without the scale (as written before fp16 existed) loads with the defaults
  path = str(tmp_path / 'old.pt')
  pipeline.save_checkpoint(c, path, 6)
  ck = torch.load(path, weights_only=True)
  assert float(ck['loss_scale']) == float(c.loss_scale)
  del ck['loss_scale'], ck['good_steps']
  torch.save(ck, path)
  pipeline.load_checkpoint(c, path)
  assert float(c.loss_scale) == 2.0 ** 30 and int(c.good_steps) == 0


def test_predict_does_not_scale_and_switching_an_fp32_encoder():
  enc, _, _ = _train('fp32', steps=20)
  tr = tfrbert.TFRBertRankingTrainer(tfrbert.TFRBertScorer(enc, 0.0), T._loss())
  wid, mask, tid, y = T._separable(4, 6, 10, seed=3)
  s32 = tr.predict(wid.cuda(), mask.cuda(), tid.cuda()).detach().cpu().double()
  enc.set_precision('fp16')
  tr.loss_scale.fill_(2.0 ** 20)   # predict ignores it
  s16 = tr.predict(wid.cuda(), mask.cuda(), tid.cuda()).detach().cpu().double()
  enc.set_precision('bf16')
  sbf = tr.predict(wid.cuda(), mask.cuda(), tid.cuda()).detach().cpu().double()
  c = enc.config
  sbar, _ = H.bars(10, c.hidden_size, c.intermediate_size, c.num_layers)
  top = s32.abs().max()
  e16 = float((s16 - s32).abs().max() / top)
  ebf = float((sbf - s32).abs().max() / top)
  print('[bert fp16 switch] max |fp16 - fp32| / max |fp32| = %.5f (bf16 %.5f, bar %.4f)' %
        (e16, ebf, sbar))
  assert e16 <= sbar and e16 < ebf


def test_hf_fixture_scores_against_fp64():
  import test_bert_checkpoint_gpu as C
  enc = tfrbert.BertEncoder.from_pretrained(C.HF, seed=5, precision='fp16')
  c = enc.config
  with torch.no_grad():
    enc.flat[-c.hidden_size - 1:] = torch.linspace(-1.0, 1.0, c.hidden_size + 1).cuda()
  wid, mask, tid = C._hf_rows()
  tr = tfrbert.TFRBertRankingTrainer(tfrbert.TFRBertScorer(enc, 0.0), C._loss())
  got = tr.predict(wid[None].cuda(), mask[None].cuda(), tid[None].cuda())[0].cpu().double()
  flat = enc.flat.detach().cpu().double()
  Vv, E, Hh, I, NL, Pp, Tv = C._sizes(c)
  ref = H.F.forward(wid, mask, tid, flat, Vv, E, Hh, I, NL, Pp, Tv)
  exact = R.forward(wid, mask, tid, flat, Vv, E, Hh, I, NL, Pp, Tv)
  bar, _ = H.bars(wid.shape[1], E, I, NL)
  err = float((got - ref).abs().max() / ref.abs().max())
  err64 = float((got - exact).abs().max() / exact.abs().max())
  print('[bert fp16 hf fixture] score err %.3g against the replay, %.3g against fp64, bar %.3g'
        % (err, err64, bar))
  assert err <= bar and err64 <= bar


def test_example_runs_two_steps_in_fp16(tmp_path):
  import os
  import subprocess
  import sys

  import numpy as np

  from ranking_b200 import data
  seq, n = 16, 4
  g = np.random.RandomState(0)
  recs = []
  for _ in range(8):
    exs = []
    for j in range(n - 1):
      ids = [101] + list(g.randint(1000, 2000, seq - 2)) + [102]
      exs.append({'input_ids': [int(i) for i in ids], 'input_mask': [1] * seq,
                  'segment_ids': [0] * (seq // 2) + [1] * (seq // 2), 'label': [int(j == 0)]})
    recs.append(data.encode_elwc(None, exs))
  path = str(tmp_path / 'train.tfrecord')
  data.write_tfrecords(path, recs)
  for ls in ('dynamic', '1024'):
    cmd = [sys.executable, os.path.join(T.ROOT, 'examples', 'tfrbert_train.py'), '--train', path,
           '--valid', path, '--label', 'label', '--model_dir', str(tmp_path / ('model' + ls)),
           '--train_steps', '2', '--steps_per_loop', '1', '--seq_length', str(seq),
           '--list_size', str(n), '--vocab_size', '2048', '--hidden_size', '64',
           '--num_layers', '1', '--num_heads', '2', '--intermediate_size', '128',
           '--precision', 'fp16', '--loss_scale', ls]
    out = subprocess.run(cmd, capture_output=True, text=True, cwd=T.ROOT, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert 'step 2' in out.stdout
