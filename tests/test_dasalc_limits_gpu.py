"""DASALC (K13, csrc/dasalc.cu) at its shape limits, against the gated fp64 reference of
_dasalc_refs.py: the three ReLUs take their gates from the kernel call (the hidden layers'
sign words, the sign of t c + t over the kernel's t and c), and every gate is checked to be
admissible, i.e. equal to the reference's own decision except within the forward error bound
of 0.  Dropout and noise draws are replayed from their counter hashes.

The case table reaches every layout of cross_bwd_kernel (cw = 32, 64, 128, 256; one to four
column quads per thread; idle quad lanes; the rl > 1 row-lane reduction at widths that are
not a power of two), context_dim up to kMaxH = 128, hidden_dim up to kMaxW = 4096, D on both
sides of W, M on both sides of one cross block (32 rows) and of one BN reduction block (256
rows), M = 1 (a zero-variance BatchNormalization in training), and make_plan's cap on the dW
split-K partials.  `test_cases_cover_every_variant` recomputes all of that from the tables.

Gates.  Each call is first checked layer by layer (`kernel_checks`): every hidden sign word
must be the sign of its Dense layer recomputed in fp64 from the input the kernel stored for
it, except within that one GEMM's error bound of 0; the stored t and c must equal their layers
recomputed the same way within that bound; and the scores must be what cross_fwd_kernel makes
of the stored t and c, within the bound of that one W-term sum (a dropped quad of o w_o, a
missing b_o or a wrong fill on a live row is orders of magnitude outside it).  The bounds span
one rounding step each, so they judge more than 80 % of the gates at every shape (asserted).

Bars.  With the gates shared, 3xTF32 is fp32-faithful, so the suite's bars apply: the moving
statistics within 1e-5, every parameter block and dE within 1e-4 relative L2 (a block whose
reference is exactly 0 must be 0), and the scores within 1e-5 of the largest |score| up to
W = 512.  Beyond, the end-to-end score error is dominated by t = a_2 W_t + b_t, a GEMM of depth
W whose accumulated rounding grows at most linearly with W (the engine's accumulator is
charged one unit per addition, (3 W + 1) 2^-23 in all), and a score sums W of those t against
w_o.  The bar scales with that depth from the 1e-5 that holds at W = 512: 1e-5 W / 512, 8e-5
at W = 4096 (on an H100 SXM at 700 W, W = 2048 to 4096 land at 2e-5 to 7e-5).  Plain
TF32 is held to test_dasalc_gpu.py's 2e-2 of the largest |score|.  dE is written with a row
pitch larger than context_dim into a buffer of sentinels, which the pad columns must keep.
"""
import ctypes
import math

import pytest
import torch

import _dasalc_refs as ref

gpu = pytest.mark.gpu
SMS = 132            # H100 SXM; the GPU tests take the device's own count
SENTINEL = 1234.5
PAD = 4              # extra columns in the row pitch of E and dE
LOG_EPS = math.log(1e-10)

# (D, W, h, M).  Every M = 1, 31, 32, 33, 255, 256, 257; W from 4 to kMaxW.
CASES = [
    (8, 4, 4, 33),          # W / 4 = 1: cw 32, 31 idle quad lanes, rl = 8
    (136, 100, 36, 31),     # 25 quads: rl = 8 over a width that is not a power of two
    (1024, 64, 36, 257),    # D far above W
    (4, 128, 128, 32),      # context_dim = kMaxH; exactly one cross block
    (36, 132, 4, 255),      # cw 64 (33 quads, rl = 4)
    (136, 256, 36, 256),    # cw 64, every lane busy
    (16, 260, 128, 1),      # cw 128 (65 quads, rl = 2); one row
    (136, 512, 4, 257),     # cw 128, every lane busy
    (64, 516, 36, 33),      # cw 256, one quad per thread, 127 idle
    (136, 2048, 128, 31),   # two quads per thread; M below one cross block
    (36, 4092, 36, 255),    # four quads per thread, the last one idle on one lane
    (128, 4096, 4, 256),    # kMaxW: four quads per thread, D below W
]
# make_plan's cap on the dW split-K partials (64 M floats) is active: W = 4096 allows 4 splits,
# W = 3072 allows 7.  M = 5000 leaves a short last split.
SPLIT_CAP = [(136, 4096, 36, 1100), (136, 4096, 36, 5000), (136, 3072, 36, 2000)]
TF32_CASES = [(136, 100, 36, 31), (36, 132, 4, 255), (136, 512, 4, 257), (64, 516, 36, 33)]


# --------------------------------------------------------------------------- harness ---
def _make(d, w, h, m, seed, precision='tf32x3', mask_all=False):
  from ranking_b200.research import dasalc
  gen = torch.Generator().manual_seed(seed)
  sc = dasalc.DASALCScorer(d, w, h, dropout=0.3, input_noise_stddev=0.5, batch_norm_moment=0.9,
                           precision=precision, seed=seed)
  with torch.no_grad():
    for name in sc.KERNELS:
      b = sc.bias(name)
      b.copy_(torch.randn(b.shape, generator=gen) * 0.1)
    for name in sc.NORMS:
      gm, be = sc.batch_norm(name)
      gm.copy_(1.0 + torch.randn(gm.shape, generator=gen) * 0.2)
      be.copy_(torch.randn(be.shape, generator=gen) * 0.2)
      mean, var = sc.moving_stats(name)
      mean.copy_(torch.randn(mean.shape, generator=gen) * 0.3)
      var.copy_(0.5 + torch.rand(var.shape, generator=gen))
  x = ref.transform(torch.randn(m, d, generator=gen) * 3).float()
  e = torch.randn(m, h, generator=gen)
  mask = torch.rand(m, generator=gen) < 0.85
  if m:
    mask[0] = True
  if mask_all:
    mask[:] = False
  ds = torch.randn(m, generator=gen)
  return sc, x, e, mask, ds


def _kernel(sc, x, e, mask, ds, training):
  """One tfr_dasalc_fwd + tfr_dasalc_bwd through the C ABI; E and dE with row pitch h + PAD,
  dE and scores over sentinels, grads over NaN."""
  from ranking_b200 import _C
  m, d, h = x.shape[0], sc.input_dim, sc.context_dim
  r = max(m, 1)   # M = 0 still passes valid pointers
  prec = {'tf32x3': _C.PREC_TF32X3, 'tf32': _C.PREC_TF32}[sc.precision]
  cfg = sc._run_cfg(training=training)
  ws = sc._new_workspace(m)
  xg = torch.zeros(r, d, device='cuda')
  xg[:m] = x.cuda()
  eg = torch.full((r, h + PAD), SENTINEL, device='cuda')
  eg[:m, :h] = e.cuda()
  m8 = mask.to(torch.uint8).cuda() if m else torch.ones(1, dtype=torch.uint8, device='cuda')
  dsg = torch.zeros(r, device='cuda')
  dsg[:m] = ds.cuda()
  scores = torch.full((r,), SENTINEL, device='cuda')
  grads = torch.full_like(sc.flat.data, float('nan'))
  de = torch.full((r, h + PAD), SENTINEL, device='cuda')
  st = _C.stream()
  _C.check(_C.lib.tfr_dasalc_fwd(_C.ptr(xg), _C.ptr(eg), h + PAD, m, ctypes.byref(cfg),
                                 _C.ptr(sc.flat.data), _C.ptr(m8), _C.ptr(ws), _C.ptr(scores),
                                 prec, st))
  _C.check(_C.lib.tfr_dasalc_bwd(_C.ptr(xg), m, ctypes.byref(cfg), _C.ptr(sc.flat.data),
                                 _C.ptr(dsg), _C.ptr(m8), _C.ptr(ws), _C.ptr(grads), _C.ptr(de),
                                 h + PAD, prec, st))
  torch.cuda.synchronize()
  return {'scores': scores, 'grads': grads, 'de': de, 'ws': ws, 'seed': cfg.seed}


def _rel(a, b):
  """Relative L2 error; the absolute one where the reference is exactly 0."""
  a, b = a.double().reshape(-1), b.double().reshape(-1).to(a.device)
  nb = float(b.norm())
  return float((a - b).norm()) / nb if nb > 0 else float((a - b).norm())


def kernel_checks(sc, got, mask, training, dev):
  """The layer-local checks of one call (_dasalc_refs.local_checks, cross_scores): every sign
  word explained by the stored input of its layer, t and c by theirs, the scores by t and c.
  Returns the kernel's gates on `dev`."""
  d, w, h = sc.input_dim, sc.hidden_dim, sc.context_dim
  m = mask.numel()
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  kg = ref.kernel_gates(got['ws'], d, w, h, m, sms)
  kg = {k: [g.to(dev) for g in v] if k == 'hidden' else v.to(dev) for k, v in kg.items()}
  flat = sc.flat.detach().to(dev, torch.float64)
  r = ref.local_checks(kg, flat, d, w, h, sc.precision)
  assert max(r[k] for k in ('relu1', 'relu2', 't', 'c')) <= 1, r
  if sc.precision == 'tf32x3' and m > 1:   # the checks can judge most gates
    assert min(r['judged1'], r['judged2']) > 0.8, r
  keep = None
  if training and sc.dropout > 0:
    keep = ref.draws(got['seed'], m, d, w, sc.dropout, 0.0, dev)[3]
  s, bound = ref.cross_scores(kg['t'], kg['c'], flat, d, w, h, keep, sc.dropout)
  live = mask.reshape(-1).to(dev)
  err = (got['scores'][:m].to(dev).double() - s).abs()
  assert bool((err <= bound)[live].all()), float((err / bound)[live].max())
  return {'hidden': kg['hidden'], 'cross': kg['cross']}


def score_bar(w):
  """The end-to-end score bar (module docstring): 1e-5 of the largest |score| up to W = 512,
  growing with the depth W of the t GEMM beyond."""
  return 1e-5 * max(1.0, w / 512)


def _check(sc, x, e, mask, ds, training, got, state0):
  """Everything one 3xTF32 kernel call returned, against the gated reference."""
  d, w, h, m = sc.input_dim, sc.hidden_dim, sc.context_dim, x.shape[0]
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  lay = ref.workspace_layout(d, w, h, m, sms)
  assert got['ws'].numel() == 4 * lay['total'] + 256, 'the layout no longer mirrors make_plan'
  dev = 'cuda' if m * w * max(w, d) >= 1 << 28 else 'cpu'
  gates = kernel_checks(sc, got, mask, training, dev)
  flat = sc.flat.detach().to(dev, torch.float64).requires_grad_()
  xd = x.to(dev).double()
  ed = e.to(dev).double().requires_grad_()
  kw = dict(state=state0, training=training, rate=sc.dropout, sigma=sc.input_noise_stddev,
            seed=got['seed'])
  want, stats = ref.forward(xd, ed, flat, d, w, h, mask=mask.to(dev), gates=gates, **kw)
  (want * ds.to(dev).double()).sum().backward()
  # scores (the masked ones are the fp32 ln(1e-10))
  s = got['scores'][:m].cpu()
  want = want.detach().cpu()
  live = mask.reshape(-1)
  assert bool((s[~live] == LOG_EPS).all())
  if bool(live.any()):
    err = (s[live].double() - want[live]).abs().max().item()
    top = want[live].abs().max().item()
    assert err <= score_bar(w) * top, (err / top, score_bar(w))
  # moving statistics
  if training:
    new = ref.updated_state(state0, [(a.cpu(), b.cpu()) for a, b in stats], 0.9)
    assert (sc.bn_state.cpu().double() - new).abs().max().item() < 1e-5
  else:
    assert torch.equal(sc.bn_state.cpu().double(), state0)
  errs = ref.block_errors(got['grads'].cpu(), flat.grad.cpu(), d, w, h)
  bad = {k: v for k, v in errs.items() if not v < 1e-4}
  assert not bad, bad
  assert _rel(got['de'][:m, :h].cpu(), ed.grad.cpu()) < 1e-4
  assert bool((got['de'][:, h:] == SENTINEL).all()), 'dE pad columns written'


def _check_tf32(sc, x, e, mask, training, got, state0):
  """TF32: the layer-local checks at TF32's bound, scores within 2e-2 of the largest |score|,
  the pad columns of dE untouched.  (The suite states no TF32 gradient bar.)"""
  d, w, h, m = sc.input_dim, sc.hidden_dim, sc.context_dim, x.shape[0]
  gates = kernel_checks(sc, got, mask, training, 'cpu')
  flat = sc.flat.detach().cpu().double()
  kw = dict(state=state0, training=training, rate=sc.dropout, sigma=sc.input_noise_stddev,
            seed=got['seed'])
  want, _ = ref.forward(x.double(), e.double(), flat, d, w, h, mask=mask, gates=gates, **kw)
  s = got['scores'][:m].cpu()
  live = mask.reshape(-1)
  assert bool((s[~live] == LOG_EPS).all())
  err = (s[live].double() - want[live]).abs().max().item()
  assert err <= 2e-2 * want[live].abs().max().item(), err
  assert bool((got['de'][:, h:] == SENTINEL).all())


def _run(case, training, precision='tf32x3', mask_all=False):
  d, w, h, m = case
  sc, x, e, mask, ds = _make(d, w, h, m, seed=d + w + h + m, precision=precision,
                             mask_all=mask_all)
  state0 = sc.bn_state.detach().cpu().double().clone()
  got = _kernel(sc, x, e, mask, ds, training)
  if precision == 'tf32':
    _check_tf32(sc, x, e, mask, training, got, state0)
  else:
    _check(sc, x, e, mask, ds, training, got, state0)
  return sc, got


def _id(case):
  return 'D%d-W%d-h%d-M%d' % case


# ------------------------------------------------------------------------ GPU cases ---
@gpu
@pytest.mark.parametrize('case', CASES, ids=_id)
@pytest.mark.parametrize('training', [True, False])
def test_limits(case, training):
  _run(case, training)


@gpu
@pytest.mark.parametrize('case', SPLIT_CAP, ids=_id)
@pytest.mark.parametrize('training', [True, False])
def test_split_cap(case, training):
  d, w, _, m = case
  assert ref.dw_splits(d, w, m, torch.cuda.get_device_properties(0).multi_processor_count)[2]
  _run(case, training)


@gpu
@pytest.mark.parametrize('case', TF32_CASES, ids=_id)
@pytest.mark.parametrize('training', [True, False])
def test_tf32_limits(case, training):
  _run(case, training, precision='tf32')


@gpu
@pytest.mark.parametrize('training', [True, False])
def test_all_masked_batch(training):
  """No live row: every score is ln(1e-10), every gradient and dE exactly 0; the batch
  statistics still move in training."""
  _, got = _run((136, 260, 36, 100), training, mask_all=True)
  assert bool((got['grads'] == 0).all())
  assert bool((got['de'][:, :36] == 0).all())


@gpu
@pytest.mark.parametrize('training', [True, False])
def test_zero_rows(training):
  """M = 0: the forward writes nothing and leaves the moving statistics alone; the backward
  zeroes the whole gradient and writes no dE."""
  sc, x, e, mask, ds = _make(136, 512, 36, 0, seed=1)
  state0 = sc.bn_state.clone()
  got = _kernel(sc, x, e, mask, ds, training)
  assert bool((got['grads'] == 0).all())
  assert float(got['scores'][0]) == SENTINEL
  assert bool((got['de'] == SENTINEL).all())
  assert torch.equal(sc.bn_state, state0)


# --------------------------------------------------------------- CPU: coverage ---
def test_cases_cover_every_variant():
  """The case tables reach every layout of cross_bwd_kernel, the split cap, and the edges of
  M, h, W and D they are there to reach (computed from the kernel's own rules, at 132 SMs)."""
  cws, quads, idle_rl, idle_quad = set(), set(), False, False
  for d, w, h, m in CASES + SPLIT_CAP:
    cw, rl, q, idle = ref.cross_layout(w)
    cws.add(cw)
    quads.add(q)
    w4 = w // 4
    idle_rl |= rl > 1 and w4 & (w4 - 1) != 0
    idle_quad |= cw == 256 and idle
  assert cws == {32, 64, 128, 256}
  assert quads == {1, 2, 3, 4}
  assert idle_rl and idle_quad
  assert {m for *_, m in CASES} >= {1, 31, 32, 33, 255, 256, 257}
  assert any(m < 32 for *_, m in CASES)   # a single, partial cross block
  assert {h for _, _, h, _ in CASES} >= {4, 36, 128} and max(h for _, _, h, _ in CASES) == 128
  assert {w for _, w, _, _ in CASES} >= {4, 100, 128, 132, 256, 260, 512, 516, 2048, 4092,
                                         4096}
  assert any(d > w for d, w, _, _ in CASES) and any(d < w for d, w, _, _ in CASES)
  assert not any(ref.dw_splits(d, w, m, SMS)[2] for d, w, _, m in CASES)
  for d, w, _, m in SPLIT_CAP:
    rows, splits, capped = ref.dw_splits(d, w, m, SMS)
    assert capped, (w, m)
  assert {w for _, w, _, _ in SPLIT_CAP} == {3072, 4096}
  # the largest leaves a short last split
  rows, splits, _ = ref.dw_splits(136, 4096, 5000, SMS)
  assert splits == 4 and 5000 - (splits - 1) * rows < rows


# -------------------------------------------------------- CPU: negative controls ---
NEG = (8, 64, 4, 70)   # D, W, h, M


def _neg_setup(training, seed=3):
  d, w, h, m = NEG
  g = torch.Generator().manual_seed(seed)
  flat = torch.randn(ref.param_count(d, w, h), generator=g, dtype=torch.float64) * 0.3
  p = ref.blocks(flat, d, w, h)
  for name in ('g_in', 'g1', 'g2', 'gc'):
    p[name].copy_(1.0 + 0.2 * torch.randn(p[name].shape, generator=g, dtype=torch.float64))
  state = torch.cat([torch.cat([torch.randn(n, generator=g, dtype=torch.float64) * 0.3,
                                0.5 + torch.rand(n, generator=g, dtype=torch.float64)])
                     for _, n in ref.state_shapes(d, w, h)])
  x = ref.transform(torch.randn(m, d, generator=g, dtype=torch.float64) * 3)
  e = torch.randn(m, h, generator=g, dtype=torch.float64)
  ds = torch.randn(m, generator=g, dtype=torch.float64)
  mask = torch.rand(m, generator=g) < 0.85
  kw = dict(state=state, training=training, rate=0.3 if training else 0.0,
            sigma=0.5 if training else 0.0, seed=(77 << 32) | 5, mask=mask)
  return flat, x, e, ds, kw


def _grads(flat, x, e, ds, kw, gates=None, hook=None):
  d, w, h, _ = NEG
  f = flat.clone().requires_grad_()
  ed = e.clone().requires_grad_()
  pre = []
  s, _ = ref.forward(x, ed, f, d, w, h, gates=gates, pre=pre, **kw)
  if hook is not None:
    pre[0]['t'].register_hook(hook)
  (s * ds).sum().backward()
  return s.detach(), f.grad, ed.grad, pre[0]


def _own_gates(pre):
  return {'hidden': [(pre['z1'] > 0).double().detach(), (pre['z2'] > 0).double().detach()],
          'cross': (pre['v'] > 0).double().detach()}


@pytest.mark.parametrize('training', [True, False])
def test_gated_reference_equals_ungated(training):
  """With the gates the reference decides itself (no pre-activation near 0 here), the gated
  reference is the ungated one."""
  flat, x, e, ds, kw = _neg_setup(training)
  s0, g0, de0, pre = _grads(flat, x, e, ds, kw)
  for v in (pre['z1'], pre['z2'], pre['v']):
    assert v.detach().abs().min().item() > 1e-9
  s1, g1, de1, _ = _grads(flat, x, e, ds, kw, gates=_own_gates(pre))
  for a, b in ((s0, s1), (g0, g1), (de0, de1)):
    assert torch.allclose(a, b, rtol=1e-12, atol=1e-14)


@pytest.mark.parametrize('training', [True, False])
def test_negative_gradient_controls(training):
  """Gradient defects a kernel could have, injected into a stand-in for its result (the exact
  chain under its own gates), each fail the per-block comparison the GPU tests make."""
  d, w, h, m = NEG
  flat, x, e, ds, kw = _neg_setup(training)
  _, want, _, _ = _grads(flat, x, e, ds, kw)
  assert max(ref.block_errors(want, want, d, w, h).values()) == 0
  q = 5   # column quad 5: columns 20..23
  # one column quad of dw_o dropped
  bad = want.clone()
  ref.blocks(bad, d, w, h)['wo'][4 * q:4 * q + 4] = 0
  assert ref.block_errors(bad, want, d, w, h)['wo'] > 1e-4
  # one column quad of dt dropped (every row): W_t's and b_t's gradients, and all upstream
  def drop_quad(g):
    g = g.clone()
    g[:, 4 * q:4 * q + 4] = 0
    return g
  _, bad, _, _ = _grads(flat, x, e, ds, kw, hook=drop_quad)
  errs = ref.block_errors(bad, want, d, w, h)
  assert errs['wt'] > 1e-4 and errs['bt'] > 1e-4, errs


WIDE = [(136, 512, 36, 257), (136, 2048, 128, 64)]   # D, W, h, M


def _glorot_setup(d, w, h, m, training, seed=6):
  """Parameters and inputs drawn as the GPU tests' _make draws them (glorot kernels)."""
  g = torch.Generator().manual_seed(seed)
  parts = []
  for name, shape in ref.param_shapes(d, w, h):
    if name in ('w1', 'w2', 'wt', 'wc', 'wo'):
      fan_in, fan_out = shape if len(shape) == 2 else (shape[0], 1)
      lim = math.sqrt(6.0 / (fan_in + fan_out))
      parts.append((torch.rand(shape, generator=g, dtype=torch.float64) * 2 - 1) * lim)
    elif name.startswith('g'):
      parts.append(1.0 + 0.2 * torch.randn(shape, generator=g, dtype=torch.float64))
    elif name.startswith('be'):
      parts.append(0.2 * torch.randn(shape, generator=g, dtype=torch.float64))
    else:
      parts.append(0.1 * torch.randn(shape, generator=g, dtype=torch.float64))
  flat = torch.cat([t.reshape(-1) for t in parts]).float().double()
  state = torch.cat([torch.cat([torch.randn(n, generator=g, dtype=torch.float64) * 0.3,
                                0.5 + torch.rand(n, generator=g, dtype=torch.float64)])
                     for _, n in ref.state_shapes(d, w, h)])
  x = ref.transform(torch.randn(m, d, generator=g) * 3).float().double()
  e = torch.randn(m, h, generator=g).double()
  kw = dict(state=state, training=training, rate=0.3 if training else 0.0,
            sigma=0.5 if training else 0.0, seed=(91 << 32) | 2)
  return flat, x, e, kw


def _standin(flat, x, e, d, w, h, kw):
  """What a correct kernel stores, up to rounding: the exact chain's Dense inputs and outputs
  rounded to fp32, and its own gates."""
  pre = []
  s, _ = ref.forward(x, e, flat, d, w, h, pre=pre, **kw)
  st = {k: pre[0][k].detach().float().double() for k in ('a0', 'a1', 'a2', 'yc', 't', 'c')}
  st['hidden'] = [(pre[0]['z1'] > 0).double(), (pre[0]['z2'] > 0).double()]
  return st, s.detach().float().double(), pre[0]


@pytest.mark.parametrize('case', WIDE, ids=_id)
@pytest.mark.parametrize('training', [True, False])
def test_negative_controls_at_wide_shapes(case, training):
  """At realistic wide shapes the layer-local checks pass a correct stand-in, judge most of
  its gates, and reject: a gate flipped where the decision is clear, one sign word of the
  second hidden layer cleared, one column quad of t zeroed; and the cross check rejects a score
  with one quad of o w_o dropped, without b_o, or with a live row given the masked fill."""
  d, w, h, m = case
  flat, x, e, kw = _glorot_setup(d, w, h, m, training)
  st, s, pre = _standin(flat, x, e, d, w, h, kw)
  r = ref.local_checks(st, flat, d, w, h)
  assert max(r[k] for k in ('relu1', 'relu2', 't', 'c')) <= 1, r
  assert min(r['judged1'], r['judged2']) > 0.8, r

  def local(**over):
    return ref.local_checks(dict(st, **over), flat, d, w, h)

  z2 = pre['z2'].detach()
  g2 = st['hidden'][1].clone()
  i = int(z2.abs().reshape(-1).argmax())
  g2.view(-1)[i] = 1 - g2.view(-1)[i]
  assert local(hidden=[st['hidden'][0], g2])['relu2'] > 1
  g2 = st['hidden'][1].clone()
  g2[m // 2, 32:64] = 0                       # one sign word of row m / 2
  assert local(hidden=[st['hidden'][0], g2])['relu2'] > 1
  t = st['t'].clone()
  t[:, 20:24] = 0
  assert local(t=t)['t'] > 1

  keep = ref.draws(kw['seed'], m, d, w, kw['rate'], 0.0)[3] if training else None
  want, bound = ref.cross_scores(st['t'], st['c'], flat, d, w, h, keep, kw['rate'])
  assert bool(((s - want).abs() <= bound).all())
  o = torch.relu(st['t'] * st['c'] + st['t'])
  if keep is not None:
    o = o * keep / (1.0 - kw['rate'])
  wo = ref.blocks(flat, d, w, h)['wo']
  bo = float(ref.blocks(flat, d, w, h)['bo'])
  q = int((o[:, :w // 4 * 4].reshape(m, -1, 4) * wo.reshape(-1, 4)).abs().sum(-1)[0].argmax())
  defects = {'dropped quad': want - o[:, 4 * q:4 * q + 4] @ wo[4 * q:4 * q + 4],
             'no b_o': want - bo,
             'masked fill': torch.where(torch.arange(m) == 0, torch.full_like(want, LOG_EPS),
                                        want)}
  for name, bad in defects.items():
    assert not bool(((bad - want).abs() <= bound).all()), name
