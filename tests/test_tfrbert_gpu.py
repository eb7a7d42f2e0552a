"""TFR-BERT on the GPU (K15): forward and every parameter gradient of tfr_bert_fwd / _bwd in
both precisions against the fp64 reference (tests/_tfrbert_refs.py), dropout replayed; the
embedding gradients, determinism, argument checks, tfr_adamw_step, the trainer (one step against
the reference chain, ~50 steps of training, checkpoint and resume) and the example script."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _tfrbert_refs as R
from oracle import keras_losses as oracle_losses
from ranking_b200 import _C
from ranking_b200 import data
from ranking_b200 import pipeline
from ranking_b200 import train
from ranking_b200.extension import tfrbert

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

#        S, L,   E,   H,  I,    NL, training   (dh = E / H)
CASES = [(6, 7, 64, 4, 100, 1, True),        # dh 16, I not a multiple of 64
         (4, 65, 64, 2, 132, 2, False),      # dh 32, L past one 64-row tile
         (3, 64, 128, 2, 256, 3, True),      # dh 64, three layers
         (5, 1, 400, 4, 400, 1, True),       # dh 100 (not a power of two), L 1
         (2, 128, 256, 2, 516, 1, False),    # dh 128
         (2, 16, 768, 12, 3072, 1, True),    # BERT-base widths
         (2, 8, 1024, 16, 1028, 1, False),   # E 1024
         (2, 512, 64, 2, 64, 1, True)]       # L 512
V, P, TV = 97, 512, 3
RATES = (0.1, 0.1, 0.1)


def _cfg(E, H, I, NL, training, precision, seed=1234, rates=RATES):
  return _C.BertCfg(vocab_size=V, hidden_size=E, num_heads=H, intermediate_size=I,
                    num_layers=NL, max_position=P, type_vocab_size=TV,
                    hidden_dropout=rates[0], attention_dropout=rates[1], output_dropout=rates[2],
                    training=int(training), seed=seed,
                    precision=_C.PREC_FP32 if precision == 'fp32' else _C.PREC_TF32)


def _inputs(S, L, seed=0):
  g = torch.Generator().manual_seed(seed)
  wid = torch.randint(0, 12, (S, L), generator=g, dtype=torch.int32)   # repeated ids
  tid = torch.randint(0, TV, (S, L), generator=g, dtype=torch.int32)
  mask = (torch.rand(S, L, generator=g) < 0.8).to(torch.uint8)
  mask[:, 0] = 1
  mask[-1] = 0   # an all-padded item
  return wid, mask, tid


def _flat(E, I, NL, seed=0):
  g = torch.Generator().manual_seed(seed)
  parts = []
  for name, shape in R.weight_shapes(V, E, I, NL, P, TV):
    if name.startswith('ln') and '_g' in name:
      parts.append(1.0 + 0.1 * torch.randn(shape, generator=g, dtype=torch.float64))
    else:
      parts.append(0.05 * torch.randn(shape, generator=g, dtype=torch.float64))
  return torch.cat([p.reshape(-1) for p in parts]).float()


def _run(cfg, wid, mask, tid, flat, dscores):
  S, L = wid.shape
  dev = 'cuda'
  w, m, t = wid.to(dev), mask.to(dev), tid.to(dev)
  params = flat.to(dev)
  ws = torch.empty(_C.lib.tfr_bert_workspace_bytes(ctypes.byref(cfg), S, L), dtype=torch.uint8,
                   device=dev)
  scores = torch.empty(S, device=dev)
  grads = torch.full_like(params, float('nan'))
  bad = torch.zeros(1, dtype=torch.int32, device=dev)
  ds = dscores.to(dev)
  st = _C.stream()
  _C.check(_C.lib.tfr_bert_fwd(_C.ptr(w), _C.ptr(m), _C.ptr(t), S, L, ctypes.byref(cfg),
                               _C.ptr(params), _C.ptr(ws), _C.ptr(scores), _C.ptr(bad), st))
  _C.check(_C.lib.tfr_bert_bwd(_C.ptr(w), _C.ptr(m), _C.ptr(t), S, L, ctypes.byref(cfg),
                               _C.ptr(params), _C.ptr(ds), _C.ptr(ws), _C.ptr(grads), st))
  torch.cuda.synchronize()
  return scores.cpu(), grads.cpu(), int(bad.item())


def _reference(cfg, wid, mask, tid, flat, dscores, **kw):
  f = flat.double().clone().requires_grad_()
  s = R.forward(wid, mask, tid, f, V, cfg.hidden_size, cfg.num_heads, cfg.intermediate_size,
                cfg.num_layers, P, TV, training=bool(cfg.training), hdrop=cfg.hidden_dropout,
                adrop=cfg.attention_dropout, sdrop=cfg.output_dropout, seed=cfg.seed, **kw)
  (s * dscores.double()).sum().backward()
  return s.detach(), f.grad


def _errors(cfg, got_s, got_g, ref_s, ref_g):
  """(score error, {block: error}) relative to the largest exact magnitude of each."""
  E, I, NL = cfg.hidden_size, cfg.intermediate_size, cfg.num_layers
  es = float((got_s.double() - ref_s).abs().max() / ref_s.abs().max())
  eg = {}
  gg = R.unflatten(got_g.double(), V, E, I, NL, P, TV)
  rg = R.unflatten(ref_g, V, E, I, NL, P, TV)
  for name in gg:
    den = float(rg[name].abs().max())
    if den == 0.0:
      continue
    eg[name] = float((gg[name] - rg[name]).abs().max()) / den
  return es, eg


@pytest.mark.parametrize('precision', ['fp32', 'tf32'])
@pytest.mark.parametrize('case', CASES, ids=lambda c: 'S%d-L%d-E%d-H%d-I%d-NL%d-%s' % (
    c[0], c[1], c[2], c[3], c[4], c[5], 'train' if c[6] else 'infer'))
def test_forward_and_gradients_against_reference(case, precision):
  S, L, E, H, I, NL, training = case
  cfg = _cfg(E, H, I, NL, training, precision)
  wid, mask, tid = _inputs(S, L)
  flat = _flat(E, I, NL)
  dscores = torch.randn(S, generator=torch.Generator().manual_seed(5))
  got_s, got_g, bad = _run(cfg, wid, mask, tid, flat, dscores)
  assert bad == 0
  assert torch.isfinite(got_s).all() and torch.isfinite(got_g).all()
  ref_s, ref_g = _reference(cfg, wid, mask, tid, flat, dscores)
  es, eg = _errors(cfg, got_s, got_g, ref_s, ref_g)
  sbar, gbar = R.bars(precision, L, E, I, NL)
  worst = max(eg, key=eg.get)
  print('[bert %s %s] score err/bar %.3f, worst grad %s err/bar %.3f' %
        (precision, case, es / sbar, worst, eg[worst] / gbar))
  assert es <= sbar, (es, sbar)
  assert eg[worst] <= gbar, (worst, eg[worst], gbar)
  # table rows no id hit: exactly zero
  g = R.unflatten(got_g, V, E, I, NL, P, TV)
  assert torch.equal(g['word'][12:], torch.zeros_like(g['word'][12:]))
  assert torch.equal(g['pos'][L:], torch.zeros_like(g['pos'][L:]))


@pytest.mark.parametrize('control', ['erf_gelu', 'no_mask'])
def test_negative_control_fails_the_bar(control):
  S, L, E, H, I, NL, _ = CASES[2]
  cfg = _cfg(E, H, I, NL, False, 'fp32')
  wid, mask, tid = _inputs(S, L)
  flat = _flat(E, I, NL)
  dscores = torch.randn(S, generator=torch.Generator().manual_seed(5))
  got_s, got_g, _ = _run(cfg, wid, mask, tid, flat, dscores)
  kw = {'gelu': R.gelu_erf} if control == 'erf_gelu' else {'mask_logits': False}
  ref_s, ref_g = _reference(cfg, wid, mask, tid, flat, dscores, **kw)
  es, eg = _errors(cfg, got_s, got_g, ref_s, ref_g)
  sbar, gbar = R.bars('fp32', L, E, I, NL)
  assert es > sbar or max(eg.values()) > gbar


def test_embedding_gradient_repeated_ids_and_determinism():
  S, L, E, H, I, NL = 4, 9, 64, 4, 64, 1
  cfg = _cfg(E, H, I, NL, True, 'fp32')
  wid = torch.full((S, L), 5, dtype=torch.int32)
  wid[:, ::2] = 7
  tid = torch.zeros(S, L, dtype=torch.int32)
  mask = torch.ones(S, L, dtype=torch.uint8)
  flat = _flat(E, I, NL)
  dscores = torch.randn(S, generator=torch.Generator().manual_seed(6))
  s1, g1, _ = _run(cfg, wid, mask, tid, flat, dscores)
  s2, g2, _ = _run(cfg, wid, mask, tid, flat, dscores)
  assert torch.equal(s1, s2) and torch.equal(g1, g2)
  ref_s, ref_g = _reference(cfg, wid, mask, tid, flat, dscores)
  g = R.unflatten(g1, V, E, I, NL, P, TV)
  r = R.unflatten(ref_g, V, E, I, NL, P, TV)
  hit = [5, 7]
  others = [v for v in range(V) if v not in hit]
  assert torch.equal(g['word'][others], torch.zeros(len(others), E))
  assert torch.equal(g['type'][1:], torch.zeros(TV - 1, E))
  err = (g['word'][hit].double() - r['word'][hit]).abs().max() / r['word'][hit].abs().max()
  assert float(err) < 2e-3


def test_out_of_range_ids_are_skipped_and_counted():
  S, L, E, H, I, NL = 2, 5, 32, 2, 32, 1
  cfg = _cfg(E, H, I, NL, False, 'fp32')
  wid, mask, tid = _inputs(S, L)
  wid[0, 1] = V
  wid[1, 2] = -3
  tid[1, 3] = TV
  flat = _flat(E, I, NL)
  dscores = torch.ones(S)
  got_s, got_g, bad = _run(cfg, wid, mask, tid, flat, dscores)
  assert bad == 3
  ref_s, ref_g = _reference(cfg, wid, mask, tid, flat, dscores)
  es, eg = _errors(cfg, got_s, got_g, ref_s, ref_g)
  assert es < 2e-4 and max(eg.values()) < 2e-3


def test_invalid_arguments_before_any_cuda_call():
  S, L = 2, 4
  wid, mask, tid = [t.cuda() for t in _inputs(S, L)]
  good = _cfg(32, 2, 32, 1, False, 'fp32')
  n = _C.lib.tfr_bert_param_count(ctypes.byref(good))
  params = torch.zeros(n, device='cuda')
  ws = torch.empty(_C.lib.tfr_bert_workspace_bytes(ctypes.byref(good), S, L), dtype=torch.uint8,
                   device='cuda')
  out = torch.empty(S, device='cuda')
  grads = torch.empty(n, device='cuda')
  bad_cfgs = [dict(num_heads=3), dict(hidden_size=1028, num_heads=4), dict(num_heads=16),
              dict(hidden_size=264, num_heads=1), dict(intermediate_size=30),
              dict(intermediate_size=4100), dict(num_layers=0), dict(num_layers=25),
              dict(max_position=513), dict(type_vocab_size=0), dict(type_vocab_size=17),
              dict(vocab_size=0), dict(hidden_dropout=1.0), dict(attention_dropout=-0.1),
              dict(output_dropout=1.5), dict(precision=_C.PREC_TF32X3)]
  calls = []
  for change in bad_cfgs:
    c = _cfg(32, 2, 32, 1, False, 'fp32')
    for k, v in change.items():
      setattr(c, k, v)
    calls.append((c, S, L, wid, mask, tid, params, ws, out, grads))
  calls += [(good, S, 0, wid, mask, tid, params, ws, out, grads),
            (good, S, 513, wid, mask, tid, params, ws, out, grads),
            (good, -1, L, wid, mask, tid, params, ws, out, grads),
            (good, 1 << 20, 64, wid, mask, tid, params, ws, out, grads)]
  for i in range(6):
    args = [wid, mask, tid, params, ws, out]
    args[i] = None
    calls.append((good, S, L, *args, grads))
  calls.append((good, S, L, wid, mask, tid, params, ws, out, None))
  n0 = _C.lib.tfr_launch_count()
  for c, s, l, w, m, t, p, wsp, o, g in calls:
    if g is not None:   # the last call differs from a valid forward only in grads
      assert _C.lib.tfr_bert_fwd(_C.ptr(w), _C.ptr(m), _C.ptr(t), s, l, ctypes.byref(c),
                                 _C.ptr(p), _C.ptr(wsp), _C.ptr(o), None, _C.stream()) == 1
    assert _C.lib.tfr_bert_bwd(_C.ptr(w), _C.ptr(m), _C.ptr(t), s, l, ctypes.byref(c),
                               _C.ptr(p), _C.ptr(o), _C.ptr(wsp), _C.ptr(g), _C.stream()) == 1
  assert _C.lib.tfr_launch_count() == n0
  assert _C.lib.tfr_bert_param_count(None) == 0
  assert _C.lib.tfr_bert_workspace_bytes(ctypes.byref(good), S, 0) == 0
  assert _C.lib.tfr_adamw_step(None, None, None, None, None, 4, 0.1, 0.9, 0.999, 1e-6, 0.0, 1,
                               1.0, None) == 1
  assert _C.lib.tfr_adamw_step(_C.ptr(params), _C.ptr(params), _C.ptr(params), _C.ptr(params),
                               None, 4, 0.1, 0.9, 0.999, 1e-6, 0.0, 0, 1.0, None) == 1
  assert _C.lib.tfr_launch_count() == n0


def test_adamw_kernel_against_reference():
  n = 1000
  g = torch.Generator().manual_seed(3)
  p = torch.randn(n, generator=g)
  mask = (torch.rand(n, generator=g) < 0.5).to(torch.uint8)
  pd, md, vd = p.cuda(), torch.zeros(n, device='cuda'), torch.zeros(n, device='cuda')
  rp, rm, rv = p.double(), torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
  mask_d = mask.cuda()
  for t in range(1, 4):
    gr = torch.randn(n, generator=g)
    gr_d = gr.cuda()
    _C.check(_C.lib.tfr_adamw_step(_C.ptr(pd), _C.ptr(gr_d), _C.ptr(md), _C.ptr(vd),
                                   _C.ptr(mask_d), n, 1e-2, 0.9, 0.999, 1e-6, 0.01, t, 0.5,
                                   _C.stream()))
    rp, rm, rv = R.adamw(rp, gr.double(), rm, rv, t, 1e-2, wd=0.01, decay_mask=mask,
                         grad_scale=0.5)
  torch.cuda.synchronize()
  assert float((pd.cpu().double() - rp).abs().max()) < 1e-6
  assert float((md.cpu().double() - rm).abs().max()) < 1e-6


def _small_encoder(precision='fp32', seed=3, dropout=0.0):
  cfg = tfrbert.BertEncoderConfig(vocab_size=V, hidden_size=64, num_layers=2,
                                  num_attention_heads=4, intermediate_size=128,
                                  max_position_embeddings=32, type_vocab_size=2,
                                  hidden_dropout_prob=dropout, attention_dropout_prob=dropout)
  return tfrbert.BertEncoder(cfg, seed=seed, precision=precision)


def _separable(B, N, L, seed=0):
  """Relevant documents carry token 50, others not: a ranking a BERT can learn."""
  g = torch.Generator().manual_seed(seed)
  wid = torch.randint(1, 40, (B, N, L), generator=g, dtype=torch.int32)
  y = torch.randint(0, 2, (B, N), generator=g).float()
  wid[..., 3] = torch.where(y > 0, 50, 41).to(torch.int32)
  mask = torch.ones(B, N, L, dtype=torch.uint8)
  tid = torch.zeros(B, N, L, dtype=torch.int32)
  tid[..., L // 2:] = 1
  y[:, -1] = -1.0   # padded item
  mask[:, -1] = 0
  return wid, mask, tid, y


def test_trainer_step_matches_reference_chain():
  enc = _small_encoder()
  scorer = tfrbert.TFRBertScorer(enc, bert_output_dropout=0.0)
  loss = _loss()
  tr = tfrbert.TFRBertRankingTrainer(scorer, loss, learning_rate=1e-3)
  wid, mask, tid, y = _separable(3, 5, 12)
  flat0 = enc.flat.detach().cpu().double()
  l = float(tr.train_step(wid.cuda(), mask.cuda(), tid.cuda(), y.cuda()))
  torch.cuda.synchronize()
  f = flat0.clone().requires_grad_()
  c = enc.config
  s = R.forward(wid.reshape(-1, 12), mask.reshape(-1, 12), tid.reshape(-1, 12), f, V,
                c.hidden_size, c.num_attention_heads, c.intermediate_size, c.num_layers,
                c.max_position_embeddings, c.type_vocab_size)
  ref_loss = oracle_losses.SoftmaxLoss()(y.double(), s.reshape(3, 5))
  ref_loss.backward()
  assert abs(l - float(ref_loss)) < 1e-4 * max(1.0, abs(float(ref_loss)))
  n = f.numel()
  rp, rm, rv = R.adamw(flat0, f.grad, torch.zeros(n, dtype=torch.float64),
                       torch.zeros(n, dtype=torch.float64), 1, 1e-3, eps=1e-6, wd=0.01,
                       decay_mask=enc.decay_mask.cpu())
  got = enc.flat.detach().cpu().double()
  # one AdamW step moves every element by about lr; the update matches to a fraction of it
  assert float((got - rp).abs().max()) < 1e-4
  assert float((tr.accum[n:].cpu().double() - rv).abs().max() / rv.abs().max()) < 1e-2


def _loss():
  from ranking_b200.keras import losses
  return losses.get('softmax_loss')


def test_training_reduces_loss_and_tracks_reference():
  enc = _small_encoder()
  flat0 = enc.flat.detach().cpu().double()
  tr = tfrbert.TFRBertRankingTrainer(tfrbert.TFRBertScorer(enc, 0.0), _loss(),
                                     learning_rate=train.PolynomialWarmUp(3e-3, 50, 5))
  wid, mask, tid, y = _separable(4, 6, 10, seed=1)
  losses = [float(tr.train_step(wid.cuda(), mask.cuda(), tid.cuda(), y.cuda()))
            for _ in range(50)]
  assert losses[-1] < 0.85 * losses[0], losses
  # the reference trajectory, fp64
  c = enc.config
  p = flat0.clone()
  n = p.numel()
  m = torch.zeros(n, dtype=torch.float64)
  v = torch.zeros(n, dtype=torch.float64)
  sched = train.PolynomialWarmUp(3e-3, 50, 5)
  ref = []
  for t in range(50):
    f = p.clone().requires_grad_()
    s = R.forward(wid.reshape(-1, 10), mask.reshape(-1, 10), tid.reshape(-1, 10), f, V,
                  c.hidden_size, c.num_attention_heads, c.intermediate_size, c.num_layers,
                  c.max_position_embeddings, c.type_vocab_size)
    lo = oracle_losses.SoftmaxLoss()(y.double(), s.reshape(4, 6))
    lo.backward()
    ref.append(float(lo))
    p, m, v = R.adamw(p, f.grad, m, v, t + 1, sched(t), eps=1e-6, wd=0.01,
                      decay_mask=enc.decay_mask.cpu())
  dev = max(abs(a - b) for a, b in zip(losses, ref))
  print('[bert train] loss %.4f -> %.4f, reference %.4f -> %.4f, max |diff| %.2e' %
        (losses[0], losses[-1], ref[0], ref[-1], dev))
  assert dev < 0.05 * ref[0]


def test_checkpoint_resume_is_bit_identical(tmp_path):
  wid, mask, tid, y = _separable(2, 4, 8, seed=2)
  batches = [({'input_word_ids': wid, 'input_mask': mask, 'input_type_ids': tid}, y)] * 6

  def trainer():
    enc = _small_encoder(seed=9, dropout=0.1)
    return enc, tfrbert.TFRBertRankingTrainer(tfrbert.TFRBertScorer(enc, 0.1), _loss(),
                                              learning_rate=train.PolynomialWarmUp(1e-3, 6, 2))

  enc_a, a = trainer()
  pipeline.fit(a, iter(batches), 6, log_fn=lambda *_: None)
  enc_b, b = trainer()
  d = str(tmp_path / 'ck')
  pipeline.fit(b, iter(batches), 3, checkpoint_dir=d, log_fn=lambda *_: None)
  enc_c, c = trainer()
  enc_c._calls = enc_b._calls   # the dropout stream continues where it stopped
  pipeline.fit(c, iter(batches), 6, checkpoint_dir=d, log_fn=lambda *_: None)
  assert c.adam_step == 6
  assert torch.equal(enc_a.flat.detach(), enc_c.flat.detach())
  assert torch.equal(a.accum, c.accum)
  logs = pipeline.evaluate(c, batches[:1])
  assert np.isfinite(logs['metric/map'])


def test_example_runs_two_steps(tmp_path):
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
  cmd = [sys.executable, os.path.join(ROOT, 'examples', 'tfrbert_train.py'), '--train', path,
         '--valid', path, '--label', 'label', '--model_dir', str(tmp_path / 'model'),
         '--train_steps', '2',
         '--steps_per_loop', '1', '--seq_length', str(seq), '--list_size', str(n),
         '--vocab_size', '2048', '--hidden_size', '64', '--num_layers', '1', '--num_heads', '2',
         '--intermediate_size', '128']
  out = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT, timeout=600)
  assert out.returncode == 0, out.stdout + out.stderr
  assert 'step 2' in out.stdout
