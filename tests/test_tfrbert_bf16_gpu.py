"""TFR-BERT's bf16 mode on the GPU (K15, TFR_PREC_BF16): scores and every parameter gradient
against the fp64 replay of the header's bf16 rounding points (tests/_tfrbert_bf16_refs.py),
dropout replayed; negative controls, the bf16-only limits, determinism and bad ids, the
workspace size, and training (loss, checkpoint resume, switching a trained fp32 encoder)."""
import ctypes

import pytest
import torch

import _tfrbert_bf16_refs as B
import _tfrbert_refs as R
from ranking_b200 import _C
from ranking_b200 import pipeline
from ranking_b200 import train
from ranking_b200.extension import tfrbert

import test_tfrbert_gpu as T

pytestmark = pytest.mark.gpu

V, P, TV = T.V, T.P, T.TV

#        S, L,   E,    H,  I,    NL    (dh = E / H); every case has an all-padded item.  The
# head sizes cover every bucket of the bf16 attention core (16 / 32 / 64 / 128) and a padded one
# in each.
CASES = [(6, 7, 64, 4, 520, 1),        # dh 16, I not a multiple of 64
         (4, 65, 200, 5, 520, 2),      # dh 40 (bucket 64), E 200, L past one 64-row tile
         (3, 64, 128, 2, 1032, 3),     # dh 64, three layers
         (5, 1, 64, 1, 136, 1),        # L 1
         (2, 128, 256, 2, 520, 1),     # dh 128, L 128
         (2, 16, 768, 12, 3072, 1),    # BERT-base widths
         (2, 8, 1024, 16, 1032, 1),    # E 1024
         (2, 512, 64, 4, 136, 1),      # L 512
         (4, 33, 64, 8, 64, 1),        # dh 8 (half of bucket 16 is padding)
         (3, 130, 96, 4, 136, 1),      # dh 24 (bucket 32), L past two 64-row tiles
         (3, 130, 64, 2, 136, 1),      # dh 32
         (2, 70, 240, 2, 248, 1)]      # dh 120 (a partly padded bucket 128)
# RMS check: the kernels against the replay, at most 1/8 of the rounding's own effect (the
# replay against the unrounded reference).  What separates the kernels from the replay are
# roundings that flip between fp32 and fp64 accumulation, one bf16 unit each, and their RMS
# share grows as sqrt(flip rate).  The wgmma accumulator flips more often than fp32
# round-to-nearest: measured on the engine's bias GEMM (512 x 768, bf16 inputs), 3e-5 / 8e-5 /
# 4.1e-4 / 1.8e-3 of the outputs at K 64 / 256 / 768 / 3072, against 5e-5 / 9e-5 / 1.3e-4 /
# 1.6e-4 for fp32 round-to-nearest.  Past K 520 that puts the expected ratio at 0.15-0.3 and
# a few flips at the narrow [CLS] sites (pre, dpre: S x E elements) can exceed 1 with no
# rounding point misplaced (replays with one rounding site dropped lie further from the
# kernels).  So the ratio is asserted where the deepest contraction max(E, I, 3E) is at most
# 520 and printed everywhere; the max-error bar holds in every case.
RATIO = 1.0 / 8.0
RATIO_MAX_K = 520


def _cfg(E, H, I, NL, training, precision=_C.PREC_BF16, seed=1234, rates=T.RATES):
  c = T._cfg(E, H, I, NL, training, 'fp32', seed=seed, rates=rates)
  c.precision = precision
  return c


def _replay(cfg, wid, mask, tid, flat, dscores, **kw):
  f = flat.double().clone().requires_grad_()
  s = B.forward(wid, mask, tid, f, V, cfg.hidden_size, cfg.num_heads, cfg.intermediate_size,
                cfg.num_layers, P, TV, training=bool(cfg.training), hdrop=cfg.hidden_dropout,
                adrop=cfg.attention_dropout, sdrop=cfg.output_dropout, seed=cfg.seed, **kw)
  (s * dscores.double()).sum().backward()
  return s.detach(), f.grad


def _rel_fro(a, b):
  return float((a.double() - b).norm() / b.norm())


@pytest.mark.parametrize('training', [True, False], ids=['train', 'infer'])
@pytest.mark.parametrize('case', CASES, ids=lambda c: 'S%d-L%d-E%d-H%d-I%d-NL%d' % c)
def test_forward_and_gradients_against_the_bf16_replay(case, training):
  S, L, E, H, I, NL = case
  cfg = _cfg(E, H, I, NL, training)
  wid, mask, tid = T._inputs(S, L)
  flat = T._flat(E, I, NL)
  dscores = torch.randn(S, generator=torch.Generator().manual_seed(5))
  got_s, got_g, bad = T._run(cfg, wid, mask, tid, flat, dscores)
  assert bad == 0
  assert torch.isfinite(got_s).all() and torch.isfinite(got_g).all()
  rep_s, rep_g = _replay(cfg, wid, mask, tid, flat, dscores)
  ex_s, ex_g = T._reference(cfg, wid, mask, tid, flat, dscores)   # unrounded fp64
  es, eg = T._errors(cfg, got_s, got_g, rep_s, rep_g)
  sbar, gbar = B.bars(L, E, I, NL)
  worst = max(eg, key=eg.get)
  # RMS: the kernels against the replay, a fraction of the rounding's own effect
  rs = _rel_fro(got_s, rep_s) / _rel_fro(ex_s, rep_s)
  rg = _rel_fro(got_g, rep_g) / _rel_fro(ex_g, rep_g)
  print('[bert bf16 %s %s] score err/bar %.3f, worst grad %s err/bar %.3f; replay/rounding '
        'RMS ratio: scores %.4f, gradients %.4f (limit %.3f)' %
        ('train' if training else 'infer', case, es / sbar, worst, eg[worst] / gbar, rs, rg,
         RATIO))
  assert es <= sbar, (es, sbar)
  assert eg[worst] <= gbar, (worst, eg[worst], gbar)
  if max(E, I, 3 * E) <= RATIO_MAX_K:
    assert rs <= RATIO and rg <= RATIO, (rs, rg)
  g = R.unflatten(got_g, V, E, I, NL, P, TV)
  assert torch.equal(g['word'][12:], torch.zeros_like(g['word'][12:]))
  assert torch.equal(g['pos'][L:], torch.zeros_like(g['pos'][L:]))


@pytest.mark.parametrize('control', ['no_mask', 'attn_site_off_by_one'])
def test_negative_control_fails_the_bf16_bar(control):
  S, L, E, H, I, NL = 4, 16, 64, 4, 136, 1
  cfg = _cfg(E, H, I, NL, True, rates=(0.1, 0.3, 0.1))
  wid, mask, tid = T._inputs(S, L)
  flat = T._flat(E, I, NL)
  dscores = torch.randn(S, generator=torch.Generator().manual_seed(5))
  got_s, got_g, _ = T._run(cfg, wid, mask, tid, flat, dscores)
  kw = {'mask_logits': False} if control == 'no_mask' else {'attn_site_shift': 1}
  ref_s, ref_g = _replay(cfg, wid, mask, tid, flat, dscores, **kw)
  es, eg = T._errors(cfg, got_s, got_g, ref_s, ref_g)
  sbar, gbar = B.bars(L, E, I, NL)
  print('[bert bf16 control %s] score err/bar %.2f, worst grad err/bar %.2f' %
        (control, es / sbar, max(eg.values()) / gbar))
  assert es > sbar or max(eg.values()) > gbar


def test_bf16_limits_before_any_cuda_call():
  S, L = 2, 4
  wid, mask, tid = [t.cuda() for t in T._inputs(S, L)]
  n0 = _C.lib.tfr_launch_count()
  for E, H, I in [(60, 3, 64), (64, 4, 100), (96, 8, 64)]:   # E, I, head size 12
    bad = _cfg(E, H, I, 1, False)
    assert _C.lib.tfr_bert_param_count(ctypes.byref(bad)) == 0
    assert _C.lib.tfr_bert_workspace_bytes(ctypes.byref(bad), S, L) == 0
    n = _C.lib.tfr_bert_param_count(ctypes.byref(_cfg(E, H, I, 1, False, _C.PREC_FP32)))
    params = torch.zeros(n, device='cuda')
    ws = torch.empty(1 << 20, dtype=torch.uint8, device='cuda')
    out = torch.empty(S, device='cuda')
    assert _C.lib.tfr_bert_fwd(_C.ptr(wid), _C.ptr(mask), _C.ptr(tid), S, L, ctypes.byref(bad),
                               _C.ptr(params), _C.ptr(ws), _C.ptr(out), None,
                               _C.stream()) == 1   # TFR_INVALID_ARGUMENT
    assert _C.lib.tfr_bert_bwd(_C.ptr(wid), _C.ptr(mask), _C.ptr(tid), S, L, ctypes.byref(bad),
                               _C.ptr(params), _C.ptr(out), _C.ptr(ws), _C.ptr(params),
                               _C.stream()) == 1
  assert _C.lib.tfr_launch_count() == n0
  # the same sizes run in fp32
  for E, H, I in [(60, 3, 64), (64, 4, 100), (96, 8, 64)]:
    c = _cfg(E, H, I, 1, False, _C.PREC_FP32)
    w2, m2, t2 = T._inputs(S, L)
    s, g, _ = T._run(c, w2, m2, t2, T._flat(E, I, 1), torch.ones(S))
    assert torch.isfinite(s).all() and torch.isfinite(g).all()


def test_determinism_and_bad_ids():
  S, L, E, H, I, NL = 4, 9, 64, 4, 136, 2
  cfg = _cfg(E, H, I, NL, True)
  wid, mask, tid = T._inputs(S, L)
  flat = T._flat(E, I, NL)
  dscores = torch.randn(S, generator=torch.Generator().manual_seed(6))
  s1, g1, _ = T._run(cfg, wid, mask, tid, flat, dscores)
  s2, g2, _ = T._run(cfg, wid, mask, tid, flat, dscores)
  assert torch.equal(s1, s2) and torch.equal(g1, g2)
  wid[0, 1] = V
  wid[1, 2] = -3
  tid[1, 3] = TV
  got_s, got_g, bad = T._run(cfg, wid, mask, tid, flat, dscores)
  assert bad == 3
  ref_s, ref_g = _replay(cfg, wid, mask, tid, flat, dscores)
  es, eg = T._errors(cfg, got_s, got_g, ref_s, ref_g)
  sbar, gbar = B.bars(L, E, I, NL)
  assert es <= sbar and max(eg.values()) <= gbar, (es, eg)


def test_workspace_is_smaller_than_tf32():
  S, L = 32 * 10, 64   # BERT-base, 32 lists of 10 sequences of 64 tokens
  sizes = {}
  for name, prec in [('tf32', _C.PREC_TF32), ('bf16', _C.PREC_BF16)]:
    c = _cfg(768, 12, 3072, 12, True, prec)
    c.vocab_size = 30522
    sizes[name] = _C.lib.tfr_bert_workspace_bytes(ctypes.byref(c), S, L)
  print('[bert workspace] BERT-base, 32 x 10 x 64: tf32 %.2f GB, bf16 %.2f GB' %
        (sizes['tf32'] / 1e9, sizes['bf16'] / 1e9))
  assert 0 < sizes['bf16'] < sizes['tf32']


def _train(precision, steps=50):
  enc = T._small_encoder(precision)
  tr = tfrbert.TFRBertRankingTrainer(tfrbert.TFRBertScorer(enc, 0.0), T._loss(),
                                     learning_rate=train.PolynomialWarmUp(3e-3, 50, 5))
  wid, mask, tid, y = T._separable(4, 6, 10, seed=1)
  losses = [float(tr.train_step(wid.cuda(), mask.cuda(), tid.cuda(), y.cuda()))
            for _ in range(steps)]
  return enc, losses


def test_training_reduces_loss_like_fp32():
  _, l32 = _train('fp32')
  _, l16 = _train('bf16')
  drop32, drop16 = l32[0] - l32[-1], l16[0] - l16[-1]
  print('[bert bf16 train] fp32 loss %.4f -> %.4f, bf16 %.4f -> %.4f' %
        (l32[0], l32[-1], l16[0], l16[-1]))
  assert drop32 > 0
  assert drop16 >= 0.9 * drop32, (l32, l16)


def test_checkpoint_resume_is_bit_identical_in_bf16(tmp_path):
  wid, mask, tid, y = T._separable(2, 4, 8, seed=2)
  batches = [({'input_word_ids': wid, 'input_mask': mask, 'input_type_ids': tid}, y)] * 6

  def trainer():
    enc = T._small_encoder('bf16', seed=9, dropout=0.1)
    return enc, tfrbert.TFRBertRankingTrainer(tfrbert.TFRBertScorer(enc, 0.1), T._loss(),
                                              learning_rate=train.PolynomialWarmUp(1e-3, 6, 2))

  enc_a, a = trainer()
  pipeline.fit(a, iter(batches), 6, log_fn=lambda *_: None)
  enc_b, b = trainer()
  d = str(tmp_path / 'ck')
  pipeline.fit(b, iter(batches), 3, checkpoint_dir=d, log_fn=lambda *_: None)
  enc_c, c = trainer()
  enc_c._calls = enc_b._calls
  pipeline.fit(c, iter(batches), 6, checkpoint_dir=d, log_fn=lambda *_: None)
  assert c.adam_step == 6
  assert torch.equal(enc_a.flat.detach(), enc_c.flat.detach())
  assert torch.equal(a.accum, c.accum)


def test_switching_a_trained_fp32_encoder_to_bf16():
  enc, _ = _train('fp32', steps=20)
  scorer = tfrbert.TFRBertScorer(enc, 0.0)
  wid, mask, tid, y = T._separable(4, 6, 10, seed=3)
  tr = tfrbert.TFRBertRankingTrainer(scorer, T._loss())
  s32 = tr.predict(wid.cuda(), mask.cuda(), tid.cuda()).detach().cpu().double()
  enc.set_precision('bf16')
  s16 = tr.predict(wid.cuda(), mask.cuda(), tid.cuda()).detach().cpu().double()
  c = enc.config
  sbar, _ = B.bars(10, c.hidden_size, c.intermediate_size, c.num_layers)
  live = torch.isfinite(s32) & (s32.abs() < 1e30)
  err = float((s16[live] - s32[live]).abs().max() / s32[live].abs().max())
  print('[bert bf16 switch] max |bf16 - fp32| / max |fp32| = %.4f (bar %.4f)' % (err, sbar))
  assert err <= sbar


def test_example_runs_two_steps_in_bf16(tmp_path):
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
  cmd = [sys.executable, os.path.join(T.ROOT, 'examples', 'tfrbert_train.py'), '--train', path,
         '--valid', path, '--label', 'label', '--model_dir', str(tmp_path / 'model'),
         '--train_steps', '2', '--steps_per_loop', '1', '--seq_length', str(seq),
         '--list_size', str(n), '--vocab_size', '2048', '--hidden_size', '64',
         '--num_layers', '1', '--num_heads', '2', '--intermediate_size', '128',
         '--precision', 'bf16']
  out = subprocess.run(cmd, capture_output=True, text=True, cwd=T.ROOT, timeout=600)
  assert out.returncode == 0, out.stdout + out.stderr
  assert 'step 2' in out.stdout
