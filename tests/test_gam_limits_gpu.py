"""GAMLayer's example-tower kernels (csrc/gam.cu, gam_sweep_kernel<WM, MODE>) at the plans and
limits the shapes of test_gam_gpu.py never reach, against the fp64 oracle (oracle/gam.py):

  * CTAs that walk three or more 32-row tiles with a ragged last tile (the in-CTA Chan merge
    of tile statistics, the cross-tile GAM_RED sums and GAM_GRAD accumulator, the per-lane
    stash reused across tiles), at WM = 16, 32 and 64, with and without BN;
  * WM = 64, where units 32-63 carry BN statistics;
  * hidden widths that are not multiples of 4, feature widths up to 32, F = 512, four hidden
    layers, one warp per CTA, M = 1 and 31, 16 context towers, dropout replay.

Every case restates the plan of make_gam_plan (gam_plan below) and checks, from the kernels
the call launched (torch.profiler), that the sweeps ran with the predicted WM, warps per CTA
and row splits; each case also asserts the plan property it is named for.

Checks: logits and sublogits in max-norm at 1e-5 of the largest entry; the moving BN
statistics after a training step directly against the oracle's at 1e-5 (a momentum of 0.5
keeps the batch statistics' weight in them at one half); parameter gradients in max-norm for
identity towers, and for ReLU towers in L2 plus a bound on the fraction of outlying entries
(gates within rounding of 0 may flip between fp32 and fp64, as in assert_param_grads_close
of test_parity_round2_gpu.py).  With BN, training and inference (moving statistics) both run
forward and backward.

On an H100 SXM (132 SMs, 700 W) this file and tests/test_tower_output_layer_gpu.py ran in
24 s together (125 cases, host-side oracle work included).  Every plan-dependent M is
computed from the device's SM count, so another GPU runs the same variants at other row
counts.
"""
import pytest
import torch

from oracle import gam as OG
from _gam_refs import _flat_grad, _inputs, _keep, _make, _moving
from _tower_refs import kernel_launches

pytestmark = pytest.mark.gpu

MOMENTUM = 0.5
SMEM_BUDGET = 227 * 1024          # kSmemBudget, gam.cu:39


@pytest.fixture(autouse=True)
def _need_cuda():
  if not torch.cuda.is_available():
    pytest.skip('no CUDA device')


def _pad4(x):
  return (x + 3) & ~3


def gam_plan(ex_dims, hidden, bn, m):
  """make_gam_plan restated: the WM bucket (gam.cu:547-553, 562), the padded per-warp
  parameter copy and row stash (582-609), the per-warp shared memory of the GRAD sweep and
  the warps per CTA it allows (610-618), the rows per CTA and row splits (622-629)."""
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  f, L = len(ex_dims), len(hidden)
  bn = bn and L > 0
  dfmax = max(ex_dims)
  h = list(hidden) + [1]
  wmax = max(hidden, default=1)
  wm = 16 if wmax <= 16 else 32 if wmax <= 32 else 64
  o = 0
  for d in range(L + 1):
    o += ((dfmax if d == 0 else h[d - 1]) + 1) * _pad4(h[d])
  o += sum(2 * _pad4(h[d]) for d in range(L))
  pp = _pad4(o)
  s = sum(_pad4((dfmax if d == 0 else h[d - 1]) + 1) for d in range(L + 1))
  nmax = max([1] + h)
  s += sum(_pad4(h[d]) for d in range(L)) if bn else 0
  s += _pad4(nmax) + (_pad4(nmax) if bn else 0)
  if (s // 4) % 2 == 0:
    s += 4
  smem_warp = 4 * (2 * pp + 32 * s)
  nw = 8
  while nw > 1 and nw * smem_warp > SMEM_BUDGET:
    nw -= 1
  assert nw * smem_warp <= SMEM_BUDGET
  chunks = (f + nw - 1) // nw
  target = (8 * sms + chunks - 1) // chunks
  per = (m + target - 1) // target if m > 0 else 32
  per = (per + 31) // 32 * 32
  splits = (m + per - 1) // per if m > 0 else 1
  last = m - (splits - 1) * per
  return {'wm': wm, 'smem_warp': smem_warp, 'nw': nw, 'chunks': chunks, 'rows_per': per,
          'splits': splits, 'tiles': per // 32, 'last_rows': last,
          'last_full_tiles': last // 32}


def multi_tile_m(ex_dims, hidden, bn):
  """The smallest M = 7 (mod 32) at which every CTA walks at least 3 full tiles (the last
  CTA's row range included) before its ragged last tile."""
  for m in range(7, 1 << 24, 32):
    if gam_plan(ex_dims, hidden, bn, m)['last_full_tiles'] >= 3:
      return m
  raise AssertionError('no multi-tile M')


def _rel(a, b):
  a = torch.as_tensor(a).detach().cpu().double()
  b = torch.as_tensor(b).detach().cpu().double()
  return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def _l2(a, b):
  a = torch.as_tensor(a).detach().cpu().double()
  b = torch.as_tensor(b).detach().cpu().double()
  return float((a - b).norm() / (b.norm() + 1e-30))


def _outliers(a, b, tol):
  """Fraction of entries off by more than `tol` of the largest entry."""
  a = torch.as_tensor(a).detach().cpu().double()
  b = torch.as_tensor(b).detach().cpu().double()
  return float(((a - b).abs() > tol * b.abs().max()).double().mean())


def _zero_grads(gam, params):
  gam.flat.grad = None
  for p in params['example'] + params['context']:
    for k in ('dense_w', 'dense_b', 'bn_gamma', 'bn_beta'):
      for t in p[k]:
        t.grad = None


def _check_sweeps(launches, plan, f):
  """Every gam_sweep_kernel launch ran with the plan's WM, warps per CTA and row splits."""
  sweeps = [(n, g, b) for n, g, b in launches if n.startswith('gam_sweep_kernel')]
  assert sweeps, [n for n, _, _ in launches]
  for n, g, b in sweeps:
    assert n.startswith('gam_sweep_kernel<%d,' % plan['wm']), (n, plan)
    assert b == (32 * plan['nw'], 1, 1), (b, plan)
    assert g == ((f + plan['nw'] - 1) // plan['nw'], plan['splits'], 1), (g, plan)


def _run(ex_dims, hidden, m, act=None, bn=False, ctx_dims=(), ctx_hidden=None, dropout=0.0,
         grad_tol=5e-5, relu_l2=1e-4, seed=5):
  """One training step (forward + backward) and, with BN, one inference step, each against
  the oracle; returns the measured errors (printed) after asserting the bounds: logits and
  sublogits 1e-5, moving statistics 1e-5, gradients `grad_tol` (identity) or `relu_l2`
  (ReLU; see the module docstring)."""
  import ranking_b200 as tfr
  plan = gam_plan(ex_dims, hidden, bn, m)
  gam, params = _make(tfr, ex_dims, hidden, ctx_dims, ctx_hidden, act=act, bn=bn,
                      dropout=dropout, seed=seed, momentum=MOMENTUM)
  xs = _inputs(m, ex_dims, seed + 1)
  cs = _inputs(m, list(ctx_dims), seed + 2) if ctx_dims else None
  up = torch.randn(m, 1, generator=torch.Generator().manual_seed(seed + 3))
  moving = _moving(gam, params)
  f = len(ex_dims)
  errs = {}

  def step():
    # repeatable (kernel_launches may run it again): same BN state and dropout draw
    gam.bn_state.copy_(state)
    gam._dropout_calls = 0
    gam.flat.grad = None
    y, sub, _ = gam(([x.cuda() for x in xs], [c.cuda() for c in cs] if cs else None))
    (y * up.cuda()).sum().backward()
    return y, sub

  def compare(tag, y, sub, ref, rsub):
    errs[tag + 'logits'] = _rel(y, ref)
    errs[tag + 'sub'] = _rel(torch.cat(sub, 1), torch.cat(rsub, 1))
    got, want = gam.flat.grad, _flat_grad(gam, params)
    errs[tag + 'grad'] = _rel(got, want)
    errs[tag + 'grad_l2'] = _l2(got, want)
    errs[tag + 'grad_out'] = _outliers(got, want, 4 * relu_l2)
    assert errs[tag + 'logits'] <= 1e-5 and errs[tag + 'sub'] <= 1e-5, errs
    if act is None:
      assert errs[tag + 'grad'] <= grad_tol, errs
    else:
      assert errs[tag + 'grad_l2'] <= relu_l2, errs
      assert errs[tag + 'grad'] <= 2e-2, errs
      assert errs[tag + 'grad_out'] <= 5e-3, errs

  keeps = None
  if dropout > 0:
    seed_call = (gam._dropout_base << 32) | 1
    full = [_keep(seed_call, d, m, f * w, dropout).reshape(m, f, w)
            for d, w in enumerate(hidden)]
    keeps = {'example': [[k[:, i, :].double() / (1 - dropout) for k in full]
                         for i in range(f)], 'context': []}
  gam.train()
  state = gam.bn_state.clone()
  (y, sub), launches = kernel_launches(step)
  _check_sweeps(launches, plan, f)
  ref, rsub, _ = OG.gam_layer([x.double() for x in xs], [c.double() for c in cs] if cs else None,
                              params, activation=act, use_batch_norm=bn, training=True,
                              bn_moving=moving, momentum=MOMENTUM, keep_masks=keeps)
  (ref * up.double()).sum().backward()
  compare('train_', y, sub, ref, rsub)
  if bn:
    got = _moving(gam, params)
    e_mean = e_var = 0.0
    for kind in ('example', 'context'):
      for a, b in zip(got[kind], moving[kind]):
        for d in a:
          e_mean = max(e_mean, _rel(a[d][0], b[d][0]))
          e_var = max(e_var, _rel(a[d][1], b[d][1]))
    errs['moving_mean'], errs['moving_var'] = e_mean, e_var
    assert e_mean <= 1e-5 and e_var <= 1e-5, errs
    # inference: moving statistics normalise, no dropout, no state update
    _zero_grads(gam, params)
    state = gam.bn_state.clone()
    gam.eval()
    (y, sub), launches = kernel_launches(step)
    _check_sweeps(launches, plan, f)
    assert torch.equal(gam.bn_state, state)
    ref, rsub, _ = OG.gam_layer([x.double() for x in xs],
                                [c.double() for c in cs] if cs else None, params,
                                activation=act, use_batch_norm=True, training=False,
                                bn_moving=got)
    (ref * up.double()).sum().backward()
    compare('infer_', y, sub, ref, rsub)
  print('GAM F=%d hidden=%s M=%d act=%s bn=%s plan=%s\n  %s' % (
      f, hidden, m, act, bn, plan, ' '.join('%s=%.2e' % kv for kv in sorted(errs.items()))))
  return plan, errs


# --------------------------------------------------------------------- cases ---
F136 = [1] * 136


@pytest.mark.parametrize('hidden,wm', [([16], 16), ([32], 32), ([64], 64)],
                         ids=['WM16', 'WM32', 'WM64'])
@pytest.mark.parametrize('bn', [False, True], ids=['plain', 'bn'])
def test_multi_tile(hidden, wm, bn):
  """F = 136 features of width 1 (17 chunks of 8 warps; 23 chunks of 6 for [64] with BN),
  M = 7 (mod 32) chosen so that every CTA walks at least 3 full tiles and a ragged one
  (M = 6119 and 4455 on 132 SMs).  BN towers are identity towers: their gradients are held
  in max-norm, and the moving statistics check the in-CTA Chan merge of the tile statistics
  directly.  The plain towers use ReLU.
  Measured (H100): logits / sublogits <= 3.1e-7; BN moving statistics <= 1.1e-7;
  identity gradients <= 9.1e-7 (max-norm); ReLU gradients <= 3.0e-5 in L2 (WM = 64: one
  gate flip, max-norm 6.6e-4, 0.004 % of the entries beyond 4e-4)."""
  m = multi_tile_m(F136, hidden, bn)
  plan = gam_plan(F136, hidden, bn, m)
  assert plan['wm'] == wm and m % 32 == 7
  assert plan['tiles'] >= 3 and plan['last_full_tiles'] >= 3
  _run(F136, hidden, m, act=None if bn else 'relu', bn=bn)


@pytest.mark.parametrize('hidden', [[64], [40, 64], [64, 33, 10]],
                         ids=['64', '40-64', '64-33-10'])
def test_wm64_bn(hidden):
  """WM = 64 with BN and ReLU: units 32-63 of every layer of width > 32 keep their BN
  statistics in the second lane register and the out[2 lane + 64] slots.  Twelve features,
  two of width 3; 5 or 3 warps per CTA.
  Measured (H100): logits / sublogits <= 9.9e-7; moving statistics <= 3.4e-7; gradients
  <= 1.6e-6 in L2, except inference at [64], where a ReLU gate flip gives 5.3e-4 in L2
  (bound 2e-3)."""
  ex_dims = [1] * 10 + [3, 3]
  m = 1237
  plan = gam_plan(ex_dims, hidden, True, m)
  assert plan['wm'] == 64 and plan['nw'] in (3, 5)
  _run(ex_dims, hidden, m, act='relu', bn=True, relu_l2=2e-3)


@pytest.mark.parametrize('hidden,act,bn', [([10, 10], 'relu', True), ([5], None, False),
                                           ([63, 7], 'relu', True), ([10, 10], None, True)],
                         ids=['10-10-relu-bn', '5-identity', '63-7-relu-bn',
                              '10-10-identity-bn'])
def test_widths_not_multiple_of_4(hidden, act, bn):
  """Hidden widths padded to pad4(h) in the per-warp copy and the stash ([10, 10] is the
  reference's own GAM test shape), at a multi-tile M (25 447 rows; 14 567 for [63, 7]).
  Measured (H100): logits / sublogits <= 1.5e-6; moving statistics <= 3.3e-7; identity
  gradients <= 7.5e-6 (max-norm); ReLU gradients <= 3.7e-5 in L2."""
  ex_dims = [1] * 30 + [2] * 2
  m = multi_tile_m(ex_dims, hidden, bn)
  plan = gam_plan(ex_dims, hidden, bn, m)
  assert plan['tiles'] >= 3 and plan['last_full_tiles'] >= 3
  _run(ex_dims, hidden, m, act=act, bn=bn)


@pytest.mark.parametrize('act,bn', [('relu', True), (None, False)], ids=['relu-bn', 'identity'])
def test_feature_widths(act, bn):
  """Feature widths 4, 17 and 32 (the limit) between width-1 features: Dense 0 reads d_f
  columns of X and the bias row sits at d_fmax = 32.
  Measured (H100): logits / sublogits <= 3.5e-7; moving statistics <= 1.1e-7; gradients
  <= 6.1e-7."""
  ex_dims = [1, 4, 1, 17, 1, 32, 1, 1, 4, 32]
  m = 1237
  plan = gam_plan(ex_dims, [16, 8], bn, m)
  assert plan['wm'] == 16
  _run(ex_dims, [16, 8], m, act=act, bn=bn)


def test_largest_tower_one_warp():
  """Four hidden layers of 64 with BN and d_f = 32: one warp needs about 211 KB of shared
  memory in the GRAD sweep, so a CTA holds one feature (nw = 1).  Identity towers, a few
  hundred rows so that the oracle stays cheap.  No feature of width 1: under identity
  activations its 64 first-layer units are one column times constants, and the next BN
  layer divides by the small spread of their combination, which costs fp32 arithmetic about
  1e-3 of the gradient (PyTorch on the host in fp32 shows the same).
  Measured (H100): logits / sublogits <= 4.4e-7; moving statistics <= 1.1e-7; gradients
  <= 3.6e-7 (max-norm)."""
  ex_dims, hidden, m = [32, 17, 32], [64] * 4, 301
  plan = gam_plan(ex_dims, hidden, True, m)
  assert plan['nw'] == 1 and plan['wm'] == 64
  assert 200 * 1024 < plan['smem_warp'] <= SMEM_BUDGET
  _run(ex_dims, hidden, m, act=None, bn=True)


def test_512_features():
  """F = 512 (the limit), d_f = 1, hidden [16], BN and ReLU: 64 chunks of 8 warps.
  Measured (H100): logits / sublogits <= 1.6e-7; moving statistics <= 1.3e-7; gradients
  <= 4.8e-7 in L2."""
  ex_dims, hidden, m = [1] * 512, [16], 1000
  plan = gam_plan(ex_dims, hidden, True, m)
  assert plan['nw'] == 8 and plan['chunks'] == 64
  _run(ex_dims, hidden, m, act='relu', bn=True)


@pytest.mark.parametrize('m', [1, 31])
def test_tiny_m(m):
  """A single partial tile.  At M = 1 the batch variance is 0, every xhat is 0 and the BN
  backward passes no gradient below the first BN layer.  Identity towers with BN.
  Measured (H100): logits / sublogits <= 6.8e-7; moving statistics <= 1.9e-7; gradients
  <= 9.5e-7 (max-norm)."""
  ex_dims, hidden = [1, 2, 1], [16, 8]
  plan = gam_plan(ex_dims, hidden, True, m)
  assert plan['splits'] == 1 and plan['last_rows'] == m
  _run(ex_dims, hidden, m, act=None, bn=True)


@pytest.mark.parametrize('multi', [False, True], ids=['M777', 'multi-tile'])
def test_sixteen_context_towers(multi):
  """16 context towers (the limit) at F = 8 (the limit with context; their fp32 towers
  [c, 10, 10, 8] end in an 8-output layer), context hidden [10, 10], ReLU.  Once at M = 777
  and once at a multi-tile M (one chunk of 8 features: 101 479 rows on 132 SMs).
  Measured (H100): logits / sublogits <= 1.8e-7; gradients <= 4.8e-7 in L2."""
  ex_dims, hidden = [1, 2, 1, 1, 3, 1, 1, 2], [16]
  ctx_dims = [1 + j % 3 for j in range(16)]
  m = multi_tile_m(ex_dims, hidden, False) if multi else 777
  plan = gam_plan(ex_dims, hidden, False, m)
  assert plan['chunks'] == 1
  assert (plan['last_full_tiles'] >= 3) == multi
  _run(ex_dims, hidden, m, act='relu', bn=False, ctx_dims=ctx_dims, ctx_hidden=[10, 10])


def test_dropout_replay_wm64_multi_tile():
  """Dropout at WM = 64 over a multi-tile plan, replayed through the oracle with the host
  copy of the kernels' keep mask (_keep).  BN with identity activation, so the gradients
  hold in max-norm; d_f = 32 features give 3 warps per CTA and keep M * F small
  (M = 12 775 on 132 SMs).
  Measured (H100): logits / sublogits <= 3.4e-7; moving statistics <= 9.5e-8; gradients
  <= 3.8e-7 (max-norm)."""
  ex_dims, hidden = [32] * 24, [64]
  m = multi_tile_m(ex_dims, hidden, True)
  plan = gam_plan(ex_dims, hidden, True, m)
  assert plan['wm'] == 64 and plan['nw'] == 3 and plan['last_full_tiles'] >= 3
  _run(ex_dims, hidden, m, act=None, bn=True, dropout=0.5)
