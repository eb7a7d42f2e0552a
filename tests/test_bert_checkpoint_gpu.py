"""Pretrained TFR-BERT and global-norm clipping on the GPU: the Hugging Face fixture in
BertEncoder at every precision against the fp64 references, tfr_global_norm against fp64
(sizes around the block boundaries up to BERT-base), tfr_adamw_step_clipped (bits of
tfr_adamw_step within the clip, fp64 AdamW on the scaled gradient beyond it, NaN on an inf /
NaN norm), the clipping trainer (the fp64 composition, bits of the unclipped trainer under a
huge clip, grad_norm, checkpoint resume) and the example with --init_checkpoint."""
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _tfrbert_bf16_refs as B
import _tfrbert_refs as R
from oracle import keras_losses as oracle_losses
from ranking_b200 import _C
from ranking_b200 import data
from ranking_b200 import pipeline
from ranking_b200 import train
from ranking_b200.extension import tfrbert

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HF = os.path.join(ROOT, 'tests', 'golden', 'bert', 'hf_tiny')
LOG = '[bert ckpt]'


def _hf_rows():
  with open(os.path.join(HF, 'outputs.json')) as f:
    out = json.load(f)
  return (torch.tensor(out['input_ids'], dtype=torch.int32),
          torch.tensor(out['attention_mask'], dtype=torch.uint8),
          torch.tensor(out['token_type_ids'], dtype=torch.int32))


def _sizes(c):
  return (c.vocab_size, c.hidden_size, c.num_attention_heads, c.intermediate_size,
          c.num_layers, c.max_position_embeddings, c.type_vocab_size)


@pytest.mark.parametrize('precision', ['fp32', 'tf32', 'bf16'])
def test_hf_fixture_scores_against_fp64(precision):
  enc = tfrbert.BertEncoder.from_pretrained(HF, seed=5, precision=precision)
  assert enc.flat.dtype == torch.float32
  c = enc.config
  with torch.no_grad():   # a score head with weight on every pooled unit
    enc.flat[-c.hidden_size - 1:] = torch.linspace(-1.0, 1.0, c.hidden_size + 1).cuda()
  wid, mask, tid = _hf_rows()
  tr = tfrbert.TFRBertRankingTrainer(tfrbert.TFRBertScorer(enc, 0.0), _loss())
  got = tr.predict(wid[None].cuda(), mask[None].cuda(), tid[None].cuda())[0].cpu().double()
  flat = enc.flat.detach().cpu().double()
  V, E, H, I, NL, P, Tv = _sizes(c)
  L = wid.shape[1]
  if precision == 'bf16':
    ref = B.forward(wid, mask, tid, flat, V, E, H, I, NL, P, Tv)
    bar, _ = B.bars(L, E, I, NL)
  else:
    ref = R.forward(wid, mask, tid, flat, V, E, H, I, NL, P, Tv)
    bar, _ = R.bars(precision, L, E, I, NL)
  err = float((got - ref).abs().max() / ref.abs().max())
  print('%s hf fixture %s: score err %.3g, bar %.3g' % (LOG, precision, err, bar))
  assert err <= bar, (err, bar)


# --- tfr_global_norm ------------------------------------------------------------------


def _norm(x):
  n = x.numel()
  ws = torch.empty(_C.lib.tfr_global_norm_workspace_bytes(n), dtype=torch.uint8,
                   device='cuda')
  out = torch.full((), -1.0, device='cuda')
  _C.check(_C.lib.tfr_global_norm(_C.ptr(x), n, _C.ptr(out), _C.ptr(ws), ws.numel(),
                                  _C.stream()))
  return out


BLOCK = 256 * 16   # elements per norm block before the grid is capped at 2048 blocks


@pytest.mark.parametrize('n', [1, 7, BLOCK - 1, BLOCK, BLOCK + 1, 5 * BLOCK + 3,
                               2048 * BLOCK - 1, 2048 * BLOCK + 1, 3 * 2048 * BLOCK + 17,
                               110_000_000])
def test_global_norm_against_fp64(n):
  g = torch.Generator(device='cuda').manual_seed(n % 1000)
  x = torch.randn(n, generator=g, device='cuda') * 3.0
  got = _norm(x)
  again = _norm(x)
  torch.cuda.synchronize()
  ref = float(x.double().square().sum().sqrt())
  err = abs(float(got) - ref) / ref
  assert err <= 2.0 ** -23, (n, float(got), ref, err)
  assert got.view(torch.int32).item() == again.view(torch.int32).item()


@pytest.mark.parametrize('offset', [1, 2, 3])
@pytest.mark.parametrize('n', [1, 5, BLOCK + 1, 2048 * BLOCK + 3])
def test_global_norm_unaligned_against_fp64(n, offset):
  """x not 16-byte aligned: the scalar-load path, same contract."""
  g = torch.Generator(device='cuda').manual_seed(n % 1000 + offset)
  x = (torch.randn(n + offset, generator=g, device='cuda') * 3.0)[offset:]
  assert x.data_ptr() % 16 != 0
  got = _norm(x)
  again = _norm(x)
  torch.cuda.synchronize()
  ref = float(x.double().square().sum().sqrt())
  assert abs(float(got) - ref) / ref <= 2.0 ** -23, (n, offset, float(got), ref)
  assert got.view(torch.int32).item() == again.view(torch.int32).item()
  # the aligned copy sums in another order, to the same float
  assert abs(float(_norm(x.clone())) - ref) / ref <= 2.0 ** -23


def test_global_norm_above_float_range_is_inf():
  """The norm is stored as float: one above FLT_MAX becomes inf (and clips every gradient
  to NaN), as the header states."""
  x = torch.full((16,), 3e38, device='cuda')
  assert math.isinf(float(_norm(x)))


def test_global_norm_zero_length_inf_nan():
  x = torch.zeros(0, device='cuda')
  assert float(_norm(x)) == 0.0
  x = torch.ones(3 * BLOCK + 5, device='cuda')
  x[BLOCK + 9] = float('inf')
  assert math.isinf(float(_norm(x)))
  x[2 * BLOCK] = float('nan')
  assert math.isnan(float(_norm(x)))
  x = torch.ones(3 * BLOCK + 5, device='cuda')
  x[-1] = float('nan')
  assert math.isnan(float(_norm(x)))
  # squares past fp32's range are summed in double: the norm is finite
  x = torch.full((10,), 3e30, device='cuda')
  assert abs(float(_norm(x)) - 3e30 * math.sqrt(10)) <= 3e30 * math.sqrt(10) * 2 ** -23


# --- tfr_adamw_step_clipped -----------------------------------------------------------


def _state(n, seed):
  g = torch.Generator().manual_seed(seed)
  p = torch.randn(n, generator=g)
  m = torch.randn(n, generator=g) * 0.1
  v = torch.rand(n, generator=g) * 0.01
  mask = (torch.rand(n, generator=g) < 0.5).to(torch.uint8)
  gr = torch.randn(n, generator=g)
  return p, m, v, mask, gr


def _step(clipped, p, m, v, mask, gr, t, clip=None, norm=None, grad_scale=1.0):
  pd, md, vd, gd, kd = p.cuda(), m.cuda(), v.cuda(), gr.cuda(), mask.cuda()
  args = [_C.ptr(pd), _C.ptr(gd), _C.ptr(md), _C.ptr(vd), _C.ptr(kd), p.numel(), 1e-2, 0.9,
          0.999, 1e-6, 0.01, t, grad_scale]
  if clipped:
    nd = torch.tensor(norm, dtype=torch.float32, device='cuda')
    _C.check(_C.lib.tfr_adamw_step_clipped(*args, clip, _C.ptr(nd), _C.stream()))
  else:
    _C.check(_C.lib.tfr_adamw_step(*args, _C.stream()))
  torch.cuda.synchronize()
  return pd.cpu(), md.cpu(), vd.cpu()


def test_clipped_adamw_within_the_clip_gives_unclipped_bits():
  p, m, v, mask, gr = _state(70001, 1)
  want = _step(False, p, m, v, mask, gr, 3, grad_scale=0.5)
  for norm, clip in ((1.0, 2.0), (2.0, 2.0), (0.0, 1e-3), (3.0e38, float(np.float32(3.0e38)))):
    got = _step(True, p, m, v, mask, gr, 3, clip=clip, norm=norm, grad_scale=0.5)
    for a, b in zip(got, want):
      assert torch.equal(a, b), (norm, clip)


@pytest.mark.parametrize('norm,clip', [(10.0, 1.0), (1.0000001, 1.0), (1e6, 0.5)])
def test_clipped_adamw_against_fp64(norm, clip):
  p, m, v, mask, gr = _state(50000, 2)
  gp, gm, gv = _step(True, p, m, v, mask, gr, 2, clip=clip, norm=norm)
  s = clip / float(np.float32(norm))
  rp, rm, rv = R.adamw(p.double(), gr.double() * s, m.double(), v.double(), 2, 1e-2, wd=0.01,
                       decay_mask=mask)
  assert float((gm.double() - rm).abs().max()) <= 1e-6 * float(rm.abs().max())
  assert float((gv.double() - rv).abs().max()) <= 1e-5 * float(rv.abs().max())
  # |m| / sqrt(v) reaches ~100 here, so the fp32 update carries ~1e-6 of rounding
  assert float((gp.double() - rp).abs().max()) < 1e-5
  # the unclipped step moves differently: the scale is applied
  up, _, _ = _step(False, p, m, v, mask, gr, 2)
  assert not torch.equal(up, gp)


@pytest.mark.parametrize('norm', [float('inf'), float('nan')])
def test_clipped_adamw_nan_norm_makes_every_update_nan(norm):
  p, m, v, mask, gr = _state(5000, 3)
  gp, gm, gv = _step(True, p, m, v, mask, gr, 1, clip=1.0, norm=norm)
  assert bool(torch.isnan(gm).all()) and bool(torch.isnan(gv).all())
  assert bool(torch.isnan(gp).all())


# --- the clipping trainer -------------------------------------------------------------

V = 97


def _loss():
  from ranking_b200.keras import losses
  return losses.get('softmax_loss')


def _small_encoder(seed=3, dropout=0.0, precision='fp32'):
  cfg = tfrbert.BertEncoderConfig(vocab_size=V, hidden_size=64, num_layers=2,
                                  num_attention_heads=4, intermediate_size=128,
                                  max_position_embeddings=32, type_vocab_size=2,
                                  hidden_dropout_prob=dropout, attention_dropout_prob=dropout)
  return tfrbert.BertEncoder(cfg, seed=seed, precision=precision)


def _separable(B_, N, L, seed=0):
  g = torch.Generator().manual_seed(seed)
  wid = torch.randint(1, 40, (B_, N, L), generator=g, dtype=torch.int32)
  y = torch.randint(0, 2, (B_, N), generator=g).float()
  wid[..., 3] = torch.where(y > 0, 50, 41).to(torch.int32)
  mask = torch.ones(B_, N, L, dtype=torch.uint8)
  tid = torch.zeros(B_, N, L, dtype=torch.int32)
  tid[..., L // 2:] = 1
  y[:, -1] = -1.0
  mask[:, -1] = 0
  return wid, mask, tid, y


def test_trainer_tiny_clip_matches_fp64_composition():
  enc = _small_encoder()
  clip = 1e-3
  tr = tfrbert.TFRBertRankingTrainer(tfrbert.TFRBertScorer(enc, 0.0), _loss(),
                                     learning_rate=1e-3, gradient_clip_norm=clip)
  wid, mask, tid, y = _separable(3, 5, 12)
  flat0 = enc.flat.detach().cpu().double()
  tr.train_step(wid.cuda(), mask.cuda(), tid.cuda(), y.cuda())
  torch.cuda.synchronize()
  f = flat0.clone().requires_grad_()
  c = enc.config
  s = R.forward(wid.reshape(-1, 12), mask.reshape(-1, 12), tid.reshape(-1, 12), f, V,
                c.hidden_size, c.num_attention_heads, c.intermediate_size, c.num_layers,
                c.max_position_embeddings, c.type_vocab_size)
  oracle_losses.SoftmaxLoss()(y.double(), s.reshape(3, 5)).backward()
  gnorm = float(f.grad.norm())
  assert gnorm > 10 * clip
  # grad_norm: the pre-clip norm of the step's gradient
  got_norm = float(tr.grad_norm)
  assert abs(got_norm - gnorm) <= 1e-4 * gnorm, (got_norm, gnorm)
  exact = float(tr.grads.double().norm())
  assert abs(got_norm - exact) <= 2.0 ** -23 * exact
  n = f.numel()
  rp, rm, rv = R.adamw(flat0, f.grad * (clip / gnorm), torch.zeros(n, dtype=torch.float64),
                       torch.zeros(n, dtype=torch.float64), 1, 1e-3, eps=1e-6, wd=0.01,
                       decay_mask=enc.decay_mask.cpu())
  assert float((enc.flat.detach().cpu().double() - rp).abs().max()) < 1e-4
  # m = 0.1 g s: the clipped moments, to the precision of the 3xTF32 gradient
  gm = tr.accum[:n].cpu().double()
  assert float((gm - rm).abs().max() / rm.abs().max()) < 1e-3
  assert float(gm.norm()) == pytest.approx(0.1 * clip, rel=1e-4)


def test_trainer_huge_clip_gives_unclipped_bits():
  wid, mask, tid, y = _separable(2, 4, 10, seed=4)
  out = []
  for clip in (None, 1e30):
    enc = _small_encoder(seed=7, dropout=0.1)
    tr = tfrbert.TFRBertRankingTrainer(tfrbert.TFRBertScorer(enc, 0.1), _loss(),
                                       learning_rate=train.PolynomialWarmUp(1e-3, 6, 1),
                                       gradient_clip_norm=clip)
    for _ in range(3):
      tr.train_step(wid.cuda(), mask.cuda(), tid.cuda(), y.cuda())
    torch.cuda.synchronize()
    out.append((enc.flat.detach().clone(), tr.accum.clone()))
  assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])


def test_trainer_clip_checkpoint_resume_is_bit_identical(tmp_path):
  wid, mask, tid, y = _separable(2, 4, 8, seed=2)
  batches = [({'input_word_ids': wid, 'input_mask': mask, 'input_type_ids': tid}, y)] * 6

  def trainer():
    enc = _small_encoder(seed=9, dropout=0.1)
    return enc, tfrbert.TFRBertRankingTrainer(tfrbert.TFRBertScorer(enc, 0.1), _loss(),
                                              learning_rate=train.PolynomialWarmUp(1e-3, 6, 2),
                                              gradient_clip_norm=0.05)

  enc_a, a = trainer()
  pipeline.fit(a, iter(batches), 6, log_fn=lambda *_: None)
  enc_b, b = trainer()
  d = str(tmp_path / 'ck')
  pipeline.fit(b, iter(batches), 3, checkpoint_dir=d, log_fn=lambda *_: None)
  enc_c, c = trainer()
  enc_c._calls = enc_b._calls
  pipeline.fit(c, iter(batches), 6, checkpoint_dir=d, log_fn=lambda *_: None)
  assert c.adam_step == 6
  assert float(c.grad_norm) > 0.05   # the clip was active
  assert torch.equal(enc_a.flat.detach(), enc_c.flat.detach())
  assert torch.equal(a.accum, c.accum)
  assert torch.equal(a.grad_norm, c.grad_norm)


def test_pretrained_encoder_trains_in_every_precision():
  wid, mask, tid = _hf_rows()
  y = torch.tensor([[1.0, 0.0, 2.0, -1.0]])
  for precision in ('fp32', 'tf32', 'bf16'):
    enc = tfrbert.BertEncoder.from_pretrained(HF, seed=1, precision=precision)
    tr = tfrbert.TFRBertRankingTrainer(tfrbert.TFRBertScorer(enc, 0.1), _loss(),
                                       learning_rate=1e-3, gradient_clip_norm=1.0)
    for _ in range(3):
      loss = tr.train_step(wid[None].cuda(), mask[None].cuda(), tid[None].cuda(), y.cuda())
    assert math.isfinite(float(loss)) and math.isfinite(float(tr.grad_norm))
    tr.check_ids()


def test_example_with_init_checkpoint(tmp_path):
  seq, n = 12, 4
  g = np.random.RandomState(0)
  recs = []
  for _ in range(4):
    exs = []
    for j in range(n - 1):
      ln = int(g.randint(3, seq + 1))
      ids = [2] + list(g.randint(1, 64, ln - 1)) + [0] * (seq - ln)
      exs.append({'input_ids': [int(i) for i in ids], 'input_mask': [1] * ln + [0] * (seq - ln),
                  'segment_ids': [0] * (ln // 2) + [1] * (seq - ln // 2),
                  'label': [int(j == 0)]})
    recs.append(data.encode_elwc(None, exs))
  path = str(tmp_path / 'train.tfrecord')
  data.write_tfrecords(path, recs)
  model_dir = tmp_path / 'model'
  # warmup over the one step: its learning rate is 0, so the checkpoint it writes holds the
  # imported weights and the initial score head exactly
  cmd = [sys.executable, os.path.join(ROOT, 'examples', 'tfrbert_train.py'), '--train', path,
         '--label', 'label', '--model_dir', str(model_dir), '--train_steps', '1',
         '--warmup_steps', '1', '--steps_per_loop', '1', '--seq_length', str(seq),
         '--list_size', str(n), '--batch_size', '2', '--init_checkpoint', HF,
         '--gradient_clip_norm', '1.0', '--seed', '77']
  out = subprocess.run(cmd, capture_output=True, text=True, cwd=ROOT, timeout=600)
  assert out.returncode == 0, out.stdout + out.stderr
  assert 'step 1' in out.stdout
  ckpt = torch.load(str(model_dir / 'ckpt' / 'ckpt.pt'), map_location='cpu', weights_only=True)
  ref = tfrbert.BertEncoder.from_pretrained(HF, seed=77)
  assert torch.equal(ckpt['flat'], ref.flat.detach().cpu())
  feats, _ = next(tfrbert.tfrbert_batches(path, 2, n, seq))
  tr = tfrbert.TFRBertRankingTrainer(tfrbert.TFRBertScorer(ref, 0.1), _loss())
  want = tr.predict(**{k: v.cuda() for k, v in feats.items()}).clone()
  enc = tfrbert.BertEncoder(ref.config, seed=1)
  tr2 = tfrbert.TFRBertRankingTrainer(tfrbert.TFRBertScorer(enc, 0.1), _loss())
  pipeline.load_checkpoint(tr2, str(model_dir / 'ckpt' / 'ckpt.pt'))
  got = tr2.predict(**{k: v.cuda() for k, v in feats.items()})
  assert torch.equal(got, want)
  # a size flag that disagrees with the config is an error
  bad = cmd + ['--hidden_size', '64']
  out = subprocess.run(bad, capture_output=True, text=True, cwd=ROOT, timeout=600)
  assert out.returncode != 0 and 'disagrees' in out.stderr
