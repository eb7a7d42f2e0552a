"""DocumentInteractionAttention in precision 'tf32' (TFR_PREC_TF32: TF32 projections and the
wgmma attention core of csrc/din_tc.cu) against oracle/din.py in fp64, with the input ReLU
gated by the kernel's own decisions and each gate checked to be admissible, and dropout and
noise replayed from their counter hashes (tests/test_din_limits_gpu.py's harness).  The bars
come from TF32 operand truncation; their derivation is in tests/_din_tf32_refs.py.

The case table puts the kernels' 64-row query / key blocks and 64-item tiles on both sides of
their boundaries up to N = 1024, every head-size bucket of tc_bucket on both sides of its edge,
num_heads * head_size = 512 at N = 1024, num_layers = 8, training with dropout and noise and
inference, over the mask helper's full, all-padded, single-item and ragged lists.
"""
import ctypes
import itertools
import os
import subprocess
import sys

import pytest
import torch

from oracle import din as odin
import _dasalc_refs
import _din_tf32_refs as R
import test_din_limits_gpu as LIM

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID_ARGUMENT = 1   # TFR_INVALID_ARGUMENT

# (B, N, D, head_size, heads, layers, training)
CASES = [
    (3, 1, 8, 4, 1, 1, True),
    (3, 2, 8, 8, 2, 1, False),
    (3, 63, 136, 16, 2, 1, False),   # input gradient in two column chunks
    (3, 64, 8, 20, 1, 1, True),
    (3, 65, 16, 32, 2, 2, False),
    (3, 127, 8, 36, 2, 1, True),
    (3, 128, 12, 64, 2, 1, False),
    (3, 129, 8, 68, 1, 1, True),
    (3, 257, 16, 128, 1, 1, False),
    (3, 1000, 8, 32, 2, 1, True),
    (3, 40, 8, 16, 2, 8, True),      # TFR_DIN_MAX_LAYERS
    (4, 1024, 16, 128, 4, 1, True),  # TFR_DIN_MAX_LIST with num_heads * head_size = 512
]
LARGEST = CASES[-1]


def _make(case, seed):
  din, x, mask, dout, base = LIM._make(case, seed)
  din.set_precision('tf32')
  return din, x, mask, dout, base


def _errors(got, case):
  """{'out', 'dx', 'acc', blocks...} relative errors of a kernel call against fp64, after
  checking that its ReLU gates are admissible."""
  b, n, d, h, heads, nl, training = case
  din, x, mask, dout, base = got['inputs']
  m = b * n
  dev = 'cuda' if n >= 512 or m >= 4096 else 'cpu'
  gate = LIM.kernel_gate(got['ws'], b, n, d, h, heads, nl).to(dev)
  out, grads, dx = LIM.reference(din, x, mask, dout, got['seed'], training, gate, dev)
  z, band = LIM.input_band(x.to(dev).double(), din.flat.detach().to(dev, torch.float64), d, h,
                           heads, nl, precision='tf32')
  assert _dasalc_refs.gate_ratio(gate, z, band) <= 1
  errs = LIM.block_errors(got['grads'], grads, d, h, heads, nl)
  g_blk = odin.unflatten(got['grads'].double().cpu(), d, h, heads, nl)
  w_blk = odin.unflatten(grads.double().cpu(), d, h, heads, nl)
  for name in errs:   # exact gradient 0 (N = 1): against the layer's W_v gradient
    if float(w_blk[name].norm()) == 0 or name.startswith('bk') and \
        float(w_blk['wk' + name[2:]].norm()) == 0:
      errs[name] = float((g_blk[name] - w_blk[name]).norm() / w_blk['wv' + name[2:]].norm())
  errs['out'] = LIM._rel(got['out'], out.reshape(m, h))
  errs['dx'] = LIM._rel(got['dx'], dx)
  acc = got['acc'].cpu().double()
  errs['acc'] = LIM._rel(acc[:, 2:2 + d - 4] - base[:, 2:2 + d - 4].double(), dx[:, 4:].cpu())
  assert torch.equal(got['acc'][:, :2].cpu(), base[:, :2])
  assert torch.equal(got['acc'][:, d - 2:].cpu(), base[:, d - 2:])
  return errs


def _call(case, seed, precision='tf32'):
  din, x, mask, dout, base = _make(case, seed)
  din.set_precision(precision)
  got = LIM._kernel(din, x, mask, dout, base, case[6])
  got['inputs'] = (din, x, mask, dout, base)
  return got


def _all_bars(case):
  b, n, d, h, heads, nl, _ = case
  bar = R.bars(n, d, h, heads, nl)
  bar['out'] = R.out_bar(n, d, h, heads, nl)
  bar['dx'] = bar['acc'] = R.grad_bar(n, d, h, heads, nl)
  return bar


def _id(case):
  return LIM._id(case)


@gpu
@pytest.mark.parametrize('case', CASES, ids=_id)
def test_forward_and_gradients_against_fp64(case):
  errs = _errors(_call(case, seed=case[1] + case[3] + case[5]), case)
  bar = _all_bars(case)
  bad = {k: (v, bar[k]) for k, v in errs.items() if not v < bar[k]}
  assert not bad, bad
  print(_id(case), 'max err / bar %.3f' % max(errs[k] / bar[k] for k in errs))


@gpu
def test_tensor_cores_really_run():
  """The same inputs in both precisions: the TF32 outputs differ from the fp32 ones, and their
  error against fp64 is far above the fp32 path's and within the TF32 bar."""
  case = (3, 128, 12, 64, 2, 1, False)
  e = {}
  for prec in ('fp32', 'tf32'):
    got = _call(case, seed=11, precision=prec)
    e[prec] = (got, _errors(got, case))
  assert not torch.equal(e['fp32'][0]['out'], e['tf32'][0]['out'])
  assert not torch.equal(e['fp32'][0]['grads'], e['tf32'][0]['grads'])
  bar = _all_bars(case)
  for k in ('out', 'dx', 'wo0', 'wv0'):
    assert e['tf32'][1][k] > 30 * e['fp32'][1][k], (k, e['tf32'][1][k], e['fp32'][1][k])
    assert e['tf32'][1][k] < bar[k]
  assert e['fp32'][1]['out'] < 1e-5


@gpu
def test_identical_calls_give_identical_bits():
  """At the largest shape, with dropout and noise: fwd, bwd and both input-gradient calls."""
  runs = []
  for _ in range(2):
    din, x, mask, dout, base = _make(LARGEST, seed=2)
    runs.append(LIM._kernel(din, x, mask, dout, base, True))
  for k in ('out', 'grads', 'dx', 'acc'):
    assert torch.equal(runs[0][k], runs[1][k]), k


@gpu
def test_permuted_list_permutes_outputs():
  case = (3, 200, 16, 32, 2, 2, False)
  din, x, mask, dout, base = _make(case, seed=5)
  got = LIM._kernel(din, x, mask, dout, base, False)
  perm = torch.randperm(case[1], generator=torch.Generator().manual_seed(1))
  xp, mp = x[:, perm], mask[:, perm]
  dp = dout.reshape(3, case[1], -1)[:, perm].reshape(dout.shape)
  got_p = LIM._kernel(din, xp, mp, dp, base, False)
  h = case[3]
  out = got['out'].reshape(3, case[1], h)[:, perm].reshape(-1, h)
  bar = _all_bars(case)
  assert LIM._rel(got_p['out'], out) < bar['out']
  assert LIM._rel(got_p['grads'], got['grads']) < bar['wo0']


@gpu
def test_all_padded_list_attends_uniformly():
  """List 1 of the mask helper has no valid item: every query row's O is the mean of the
  list's value rows (P = 1 / N exactly in fp32), up to one TF32 product per term."""
  case = (3, 100, 16, 32, 2, 1, False)
  b, n, d, h, heads, _, _ = case
  din, x, mask, dout, base = _make(case, seed=8)
  assert not mask[1].any()
  got = LIM._kernel(din, x, mask, dout, base, False)
  m, hh = b * n, heads * h
  al = lambda v: (v + 63) // 64 * 64
  qkv_off = al(h * 3 * hh + 3 * hh) + 2 * al(m * h)
  o_off = qkv_off + al(m * 3 * hh)
  ws = got['ws']
  off = (-ws.data_ptr()) % 256
  f = ws[off:off + (ws.numel() - off) // 4 * 4].view(torch.float32).double()
  v = f[qkv_off:qkv_off + m * 3 * hh].view(b, n, 3 * hh)[1, :, 2 * hh:]
  o = f[o_off:o_off + m * hh].view(b, n, hh)[1]
  want = v.mean(0, keepdim=True).expand(n, hh)
  tol = 2 * (R.U_P + n * R.U_ACC) * v.abs().mean(0, keepdim=True)
  assert ((o - want).abs() <= tol).all(), float(((o - want).abs() / tol).max())


@gpu
def test_input_grad_accumulate_adds_exactly():
  from ranking_b200 import _C
  case = (3, 65, 40, 16, 2, 1, True)
  b, n, d = case[:3]
  din, x, mask, dout, base = _make(case, seed=3)
  got = LIM._kernel(din, x, mask, dout, base, True)
  cfg = din._run_cfg(training=True)
  cfg.seed = got['seed']
  g = torch.zeros(b * n, d, device='cuda')
  acc = base[:, :d].contiguous().cuda()
  for buf, a in ((g, 0), (acc, 1)):
    _C.check(_C.lib.tfr_din_input_grad(ctypes.byref(cfg), b, n, _C.ptr(din.flat.data),
                                       _C.ptr(got['ws']), 0, d, _C.ptr(buf), d, a, _C.stream()))
  torch.cuda.synchronize()
  assert torch.equal(acc, base[:, :d].cuda() + g)
  assert torch.equal(g, got['dx'])


# ----------------------------------------------------------------- argument errors ---
def _cfg(precision):
  from ranking_b200 import _C
  cfg = _C.DinCfg()
  cfg.input_dim, cfg.head_size, cfg.num_heads, cfg.num_layers = 8, 16, 2, 1
  cfg.precision = precision
  return cfg


@pytest.mark.parametrize('precision', [1, 3, 7, -1])
def test_unknown_precision_is_rejected_before_any_cuda_call(precision):
  """TF32X3 (1), BF16 (3) and unknown values: TFR_INVALID_ARGUMENT from every entry point,
  with a message, on a machine without a GPU too (the pointers are never touched)."""
  from ranking_b200 import _C
  cfg = _cfg(precision)
  lib = _C.lib
  dummy = ctypes.c_void_p(16)
  assert lib.tfr_din_workspace_bytes(ctypes.byref(cfg), 2, 4) == 0
  assert 'precision' in _C.last_error()
  assert lib.tfr_din_fwd(dummy, None, 2, 4, ctypes.byref(cfg), dummy, dummy, dummy, 16,
                         None) == INVALID_ARGUMENT
  assert 'precision' in _C.last_error()
  assert lib.tfr_din_bwd(dummy, None, 2, 4, ctypes.byref(cfg), dummy, dummy, 16, dummy, dummy,
                         None) == INVALID_ARGUMENT
  assert 'precision' in _C.last_error()
  assert lib.tfr_din_input_grad(ctypes.byref(cfg), 2, 4, dummy, dummy, 0, 8, dummy, 8, 0,
                                None) == INVALID_ARGUMENT
  assert 'precision' in _C.last_error()
  for p in (0, 2):   # the two built modes size the same workspace
    assert lib.tfr_din_workspace_bytes(ctypes.byref(_cfg(p)), 2, 4) > 0


def test_layer_precision_argument():
  from ranking_b200.keras import layers
  for bad in ('tf32x3', 'bf16', 'fp16'):
    with pytest.raises(ValueError):
      layers.DocumentInteractionAttention(2, 8, precision=bad)
  din = layers.DocumentInteractionAttention(2, 8, precision='tf32', device='cpu')
  assert din.get_config()['precision'] == 'tf32'
  assert layers.DocumentInteractionAttention(**din.get_config()).precision == 'tf32'
  din.set_precision(None)
  assert din.precision == 'fp32' and 'precision' not in din.get_config()
  with pytest.raises(ValueError):
    din.set_precision('bf16')


# ------------------------------------------------------------ CPU: coverage, controls ---
def test_cases_cover_every_variant():
  """Every head-size bucket of tc_bucket on both sides of each edge, N on both sides of the
  64-row / 64-item boundaries, one and two items, 1000 and 1024 (with H h = 512 and h = 128),
  L = 8, training and inference."""
  pairs, last = R.buckets()
  hs = {c[3] for c in CASES}
  assert {R.bucket(h) for h in hs} == {hp for _, hp in pairs} | {last}
  for edge, _ in pairs:
    assert any(h <= edge and R.bucket(h) == R.bucket(edge) for h in hs)
    assert any(h > edge and R.bucket(h) != R.bucket(edge) for h in hs)
  ns = {c[1] for c in CASES}
  assert ns >= {1, 2, 63, 64, 65, 127, 128, 129, 1000, 1024}
  assert any(n % R.ROWS for n in ns) and any(n % R.ROWS == 0 for n in ns)
  assert any(n == 1024 and h == 128 and h * heads == 512 for _, n, _, h, heads, _, _ in CASES)
  assert any(c[5] == 8 for c in CASES)
  assert {c[6] for c in CASES} == {True, False}
  assert LARGEST[1] == 1024 and LARGEST[6]


def test_negative_controls():
  """The bars reject a reference that gets one thing wrong: one item of every list masked
  wrongly, or the first 64-key tile dropped, moves the outputs and gradients past them."""
  din, x, mask, dout, (b, n, d, h, heads, nl, _) = LIM._cpu_case(False, case=(4, 80, 16, 16, 2, 1))
  seed = (9 << 32) | 1
  out, grads, _ = LIM.reference(din, x, mask, dout, seed, False, None, 'cpu')
  bar = R.bars(n, d, h, heads, nl)
  wrong = mask.clone()
  wrong[:, 3] = ~wrong[:, 3]
  dropped = mask.clone()
  dropped[:, :R.ROWS] = False
  dropped[1] = False   # the all-padded list stays all padded
  for bad_mask in (wrong, dropped):
    o2, g2, _ = LIM.reference(din, x, bad_mask, dout, seed, False, None, 'cpu')
    assert LIM._rel(o2, out) > R.out_bar(n, d, h, heads, nl)
    errs = LIM.block_errors(g2, grads, d, h, heads, nl)
    assert any(errs[k] > bar[k] for k in errs)
  # and the bars sit well above the fp32 path's: TF32 is distinguishable from it
  assert R.out_bar(n, d, h, heads, nl) > 100 * LIM.TOL


# -------------------------------------------------------------------------- trainers ---
@gpu
def test_din_trainer_step_in_tf32():
  import test_din_gpu as DG
  b, n, d, h, heads, nl = 8, 24, 16, 32, 2, 2
  tr, din, tower = DG._trainer(4, b, n, d, h, heads, nl, [64, 32])
  din.set_precision('tf32')
  x, y = DG._batch(torch.Generator().manual_seed(9), b, n, d)
  want_loss, want_grad = DG._oracle_step(tr, din, tower, x, y)
  got = float(tr.train_step(x.cuda(), y.cuda()))
  torch.cuda.synchronize()
  assert abs(got - want_loss) <= R.out_bar(n, d, h, heads, nl) * max(1.0, abs(want_loss))
  err = LIM._rel(tr.grads.cpu().double(), want_grad)
  assert err < R.grad_bar(n, d, h, heads, nl), err
  assert err > 10 * 5e-5   # the fp32 trainer's bar: the tensor cores ran
  # predict: the same DIN in inference, then the tower
  got_p = tr.predict(x.cuda(), y_true=y.cuda()).clone()
  din.set_precision('fp32')
  want_p = tr.predict(x.cuda(), y_true=y.cuda())
  valid = (y >= 0).cuda()
  rel = float((got_p[valid] - want_p[valid]).norm() / want_p[valid].norm())
  assert 0 < rel < R.out_bar(n, d, h, heads, nl), rel


@gpu
def test_dasalc_trainer_step_and_predict_in_tf32():
  import test_dasalc_gpu as DS
  b, n, d, w, h = 6, 30, 16, 64, 16
  tr, din, sc = DS._trainer(21, d, w, h)
  din.set_precision('tf32')
  gen = torch.Generator().manual_seed(4)
  flat = tr.tower.flat.detach().cpu().double()
  state = sc.bn_state.detach().cpu().double()
  x, y = DS._batch(gen, b, n, d)
  _, want_loss, g, state = DS._oracle_step(tr, din, sc, x, y, flat, state)
  got = float(tr.train_step(x.cuda(), y.cuda()))
  torch.cuda.synchronize()
  bar_o, bar_g = R.out_bar(n, d, h, 2, 1), R.grad_bar(n, d, h, 2, 1)
  assert abs(got - want_loss) <= bar_o * max(1.0, abs(want_loss)), (got, want_loss)
  assert LIM._rel(tr.grads.cpu().double(), g) < bar_g
  x, y = DS._batch(gen, b, n, d)
  got = tr.predict(x.cuda(), y_true=y.cuda()).cpu().double()
  want, _, _, _ = DS._oracle_step(tr, din, sc, x, y, tr.tower.flat.detach().cpu().double(),
                                  sc.bn_state.detach().cpu().double(), training=False)
  valid = y >= 0
  assert LIM._rel(got[valid], want[valid]) < bar_o


@gpu
def test_loss_trajectory_tracks_fp32():
  import test_din_gpu as DG
  b, n, d, h = 16, 40, 16, 32
  gen = torch.Generator().manual_seed(2)
  batches = [DG._batch(gen, b, n, d) for _ in range(20)]
  losses = {}
  for prec in ('fp32', 'tf32'):
    tr, din, _ = DG._trainer(7, b, n, d, h, 2, 1, [32])
    din.set_precision(prec)
    losses[prec] = [float(tr.train_step(x.cuda(), y.cuda())) for x, y in batches]
  a, t = torch.tensor(losses['fp32']), torch.tensor(losses['tf32'])
  # 20 Adagrad steps compound the per-step gradient error; allow it 20 steps' worth
  assert ((t - a).abs() <= 20 * R.out_bar(n, d, h, 2, 1) * a.abs()).all(), (a, t)


@gpu
def test_checkpoint_resumes_in_the_other_precision(tmp_path):
  """Two fp32 steps saved, resumed by a new tf32 trainer for two more: the same bits as one
  trainer that switches precision after step 2.  Checkpoints hold no precision."""
  import test_dasalc_gpu as DS
  path = os.path.join(ROOT, 'tests', 'golden', 'numerical', 'train_numerical_elwc.tfrecord')
  batches = lambda: (bt for _ in range(50) for bt in DS._fixture_batches(path))

  def trainer(prec):
    tr, din, _ = DS._trainer(3, 136, 64, 16, rate=0.0, noise=0.0)
    din.set_precision(prec)
    return tr, din
  import ranking_b200 as tfr
  ck = str(tmp_path / 'a')
  tr, _ = trainer('fp32')
  tfr.pipeline.fit(tr, batches(), 2, checkpoint_dir=ck, log_fn=lambda m: None)
  resumed, _ = trainer('tf32')
  tfr.pipeline.fit(resumed, itertools.islice(batches(), 2, None), 4, checkpoint_dir=ck,
                   log_fn=lambda m: None)
  one, din = trainer('fp32')
  ck1 = str(tmp_path / 'b')
  tfr.pipeline.fit(one, batches(), 2, checkpoint_dir=ck1, log_fn=lambda m: None)
  din.set_precision('tf32')
  tfr.pipeline.fit(one, itertools.islice(batches(), 2, None), 4, checkpoint_dir=ck1,
                   log_fn=lambda m: None)
  assert torch.equal(resumed.tower.flat.detach(), one.tower.flat.detach())


# -------------------------------------------------------------------------- examples ---
def _run(args):
  out = subprocess.run([sys.executable] + args, capture_output=True, text=True, timeout=900,
                       cwd=ROOT)
  assert out.returncode == 0, out.stdout + out.stderr
  return out.stdout


@gpu
def test_examples_run_in_tf32(tmp_path):
  num = os.path.join(ROOT, 'tests', 'golden', 'numerical')
  out = _run([os.path.join(ROOT, 'examples', 'dasalc_train.py'),
              '--train_path', os.path.join(num, 'train_numerical_elwc.tfrecord'),
              '--eval_path', os.path.join(num, 'vali_numerical_elwc.tfrecord'),
              '--num_train_steps', '20', '--batch_size', '8', '--din_precision', 'tf32'])
  assert 'step 20 loss' in out and 'ndcg' in out.lower(), out
  ant = os.path.join(ROOT, 'tests', 'golden', 'antique')
  out = _run([os.path.join(ROOT, 'examples', 'antique_train.py'),
              '--train_path', os.path.join(ant, 'train_elwc.tfrecord'),
              '--eval_path', os.path.join(ant, 'train_elwc.tfrecord'),
              '--vocab_file', os.path.join(ant, 'vocab.txt'),
              '--use_document_interaction', '1', '--num_train_steps', '5',
              '--din_precision', 'tf32'])
  assert 'step 5 loss' in out, out
  gen = torch.Generator().manual_seed(0)
  lines = []
  for q in range(24):
    for _ in range(6):
      f = torch.randn(8, generator=gen)
      lines.append('%d qid:%d %s' % (int(torch.randint(0, 5, (1,), generator=gen)), q,
                                     ' '.join('%d:%.4f' % (i + 1, v) for i, v in enumerate(f))))
  svm = tmp_path / 'train.txt'
  svm.write_text('\n'.join(lines) + '\n')
  out = _run([os.path.join(ROOT, 'examples', 'libsvm_train.py'), '--train_path', str(svm),
              '--vali_path', str(svm), '--scorer', 'din', '--num_features', '8',
              '--list_size', '8', '--num_heads', '1', '--head_size', '8', '--num_layers', '1',
              '--hidden_layer_dims', '16', '--train_batch_size', '4', '--num_train_steps', '5',
              '--din_precision', 'tf32'])
  assert 'finished at step 5' in out, out
