"""The scorer tower end to end (tfr_mlp_fwd / tfr_mlp_bwd / tfr_mlp_input_grad) at the edges of
its plan, in fp32, tf32x3 and tf32, against the gated fp64 reference of tests/_tower_fp64.py.

Every case compares elementwise, against the reference's per-element bound: the scores
(masked rows must hold RestoreList's fill exactly), every hidden activation H_d the forward
stored, the whole flat parameter gradient, the BN moving statistics (unchanged in inference)
and, for the TF32 modes, two column windows of the input gradient.  The gates come from the
kernel's own H_d, so a pre-activation next to 0 cannot loosen the bar, and each gate is checked
against the sign of the exact pre-activation and the replayed dropout stream, so a kernel that
writes zeros where it should not cannot hide behind them.

The matrix walks make_mlp_plan's boundaries (csrc/capi.cu): rows_per_split leaving 256 at
M = 256 SMs, the output layer's 16-row minimum, the 256-row BN reduction blocks, col_width's
256-column limit (BN widths 260 and 513), the fp32 SGEMM's 128 x 128 x 8 tiles (widths 1..7,
127..129, 255, 257), 1024 inputs to the output layer, 8 Dense layers, 1..8 output units, M = 0
and M = 1; the fused 3xTF32 forward's width limits (launch counter), and each output-layer and
reduction kernel mlp_out_layer_bwd2 / mlp_reduce2 select (torch.profiler).

Each case prints its err / bound ratios, one line per case, and the largest ratio of each
precision is printed when the module ends (pytest -s).
"""
import ctypes
import itertools
import zlib

import pytest
import torch

import _tower_fp64 as R
from _tower_refs import kernel_launches

pytestmark = pytest.mark.gpu

WORST = {}


@pytest.fixture(autouse=True, scope='module')
def _report():
  yield
  for p in sorted(WORST):
    print('\nworst err / bound, %s: %.3g (%s)' % (p, *WORST[p]))


@pytest.fixture(autouse=True)
def _need_cuda():
  if not torch.cuda.is_available():
    pytest.skip('no CUDA device')


def _sms():
  return torch.cuda.get_device_properties(0).multi_processor_count


def _lib():
  import __graft_entry__ as entry
  entry.build()
  from ranking_b200 import _C
  return _C


def _tower(precision, d, hidden, out, act, bn, input_bn, dropout, training, seed):
  import ranking_b200 as tfr
  t = tfr.keras.layers.create_tower(hidden, out, activation=act, input_batch_norm=input_bn,
                                    use_batch_norm=bn, batch_norm_moment=0.9, dropout=dropout,
                                    input_dim=d, precision=precision, seed=seed)
  g = torch.Generator().manual_seed(seed)
  with torch.no_grad():
    for i in range(len(t.dims) - 1):
      t.bias(i).copy_(torch.rand(t.dims[i + 1], generator=g) * 0.4 - 0.2)
    for key, (a, b, w) in t.bn_offsets.items():
      t.flat[a:a + w].copy_(torch.rand(w, generator=g) + 0.5)
      t.flat[b:b + w].copy_(torch.rand(w, generator=g) * 0.4 - 0.2)
      mean, var = t.bn_moving(key)
      mean.copy_(torch.randn(w, generator=g) * 0.1)
      var.copy_(torch.rand(w, generator=g) + 0.5)
  return t.train(training)


def run(precision, d, hidden, out, m, act='relu', masked=False, bn=False, input_bn=False,
        dropout=0.0, training=True, x_offset=0, profile=False, seed=0):
  """One forward + backward (+ input gradient windows) through the C ABI, checked against
  the reference.  Returns (the number of launches tfr_mlp_fwd made, the profiled launches)."""
  _C = _lib()
  prec = {'fp32': _C.PREC_FP32, 'tf32x3': _C.PREC_TF32X3, 'tf32': _C.PREC_TF32}[precision]
  seed = seed or zlib.crc32(repr((precision, d, hidden, out, m, act, bn, input_bn)).encode()) & 0xFFFF
  tower = _tower(precision, d, hidden, out, act, bn, input_bn, dropout, training, seed)
  L = len(hidden)
  g = torch.Generator().manual_seed(seed + 1)
  store = torch.empty(m * d + 4, device='cuda')
  x = store[x_offset:x_offset + m * d].view(m, d)
  x.copy_(torch.randn(m, d, generator=g))
  ds = torch.randn(m, out, generator=g).cuda()
  mask = (torch.rand(m, generator=g) > 0.25).cuda() if masked else None
  m8 = None if mask is None else mask.to(torch.uint8)
  cfg = tower._run_cfg()
  state0 = tower.bn_state.clone()
  ws = tower._new_workspace(m)
  scores = torch.empty(m, out, device='cuda')
  grads = torch.full_like(tower.flat.data, float('nan'))
  windows = []
  if precision != 'fp32' and L > 0 and not input_bn:
    windows = [(0, d)] + ([(4, min(8, d - 4))] if d >= 12 else [])
  dxs = [torch.full((m, d), float('nan'), device='cuda') for _ in windows]
  launches = {}

  def step():
    tower.bn_state.copy_(state0)
    n0 = _C.lib.tfr_launch_count()
    _C.check(_C.lib.tfr_mlp_fwd(_C.ptr(x), m, ctypes.byref(cfg), _C.ptr(tower.flat.data),
                                _C.ptr(m8), _C.ptr(ws), _C.ptr(scores), prec, _C.stream()))
    launches['fwd'] = _C.lib.tfr_launch_count() - n0
    _C.check(_C.lib.tfr_mlp_bwd(_C.ptr(x), m, ctypes.byref(cfg), _C.ptr(tower.flat.data),
                                _C.ptr(ds), _C.ptr(m8), _C.ptr(ws), _C.ptr(grads), prec,
                                _C.stream()))
    for (c0, nc), dx in zip(windows, dxs):
      _C.check(_C.lib.tfr_mlp_input_grad(ctypes.byref(cfg), m, _C.ptr(tower.flat.data),
                                         _C.ptr(ws), c0, nc, _C.ptr(dx), d, prec, _C.stream()))

  profiled = None
  if profile:
    _, profiled = kernel_launches(step)
  else:
    step()
  torch.cuda.synchronize()

  rcfg = R.Cfg(tower.dims, relu=act == 'relu', use_bn=bn, input_bn=input_bn, training=training,
               dropout=dropout, momentum=0.9)
  params = {'w': [tower.kernel(i) for i in range(L + 1)],
            'b': [tower.bias(i) for i in range(L + 1)]}
  if rcfg.use_bn:
    params['gamma'] = [tower.bn_gamma(i) for i in range(L)]
    params['beta'] = [tower.bn_beta(i) for i in range(L)]
  if input_bn:
    params['in_gamma'], params['in_beta'] = tower.bn_gamma('input'), tower.bn_beta('input')
  moving, moved = {}, {}
  state = tower.bn_state
  for key, (a, b, w) in tower.bn_state_offsets.items():
    moving[key] = (state0[a:a + w], state0[b:b + w])
    moved[key] = (state[a:a + w], state[b:b + w])
  if not training:
    assert torch.equal(state, state0)
  got = {'hidden': R.hidden_activations(ws, rcfg, m), 'scores': scores, 'grads': grads,
         'moving': moved if training else {},
         'dx': [(c0, nc, dx[:, :nc]) for (c0, nc), dx in zip(windows, dxs)]}
  for (c0, nc), dx in zip(windows, dxs):
    assert torch.isnan(dx[:, nc:]).all(), 'input gradient wrote past its window'
  if mask is not None and out == 1:
    assert (scores[~mask] == R.LOG_EPSILON).all()   # RestoreList's float32 fill, exactly
  ratios = R.check(rcfg, precision, R.Plan(rcfg, m, _sms()), x, params, ds, got, mask, moving,
                   cfg.dropout_seed)
  name = '%s d=%d %s o=%d m=%d' % (precision, d, hidden, out, m)
  print('%s: %s' % (name, ', '.join('%s %.3g' % r for r in ratios)))
  for what, ratio in ratios:
    if ratio > WORST.get(precision, (-1.0, ''))[0]:
      WORST[precision] = (ratio, name + ' ' + what)
  bad = [(what, ratio) for what, ratio in ratios if not ratio <= 1]
  assert not bad, (name, bad)
  return launches['fwd'], profiled


PRECISIONS = ('fp32', 'tf32x3', 'tf32')
# fp32 runs its odd widths on the CUDA-core path; the tensor-core modes need multiples of 4
ROW_TOWER = {'fp32': (13, [37, 24], 1), 'tf32x3': (36, [128, 64], 1),
             'tf32': (36, [132, 64], 1)}


def _rows(spec):
  s = 256 * _sms()
  return {'S-1': s - 1, 'S': s, 'S+1': s + 1, 'big': 100003}.get(spec, spec)


# ------------------------------------------------------------------------------- rows ---
@pytest.mark.parametrize('m', [1, 15, 16, 17, 255, 256, 257, 'S-1', 'S', 'S+1'])
@pytest.mark.parametrize('precision', PRECISIONS)
def test_rows(precision, m):
  """rows_per_split leaves 256 past M = 256 SMs; the output layer's row blocks bottom out at
  16 rows; M = 1 is one partial row tile everywhere."""
  d, hidden, out = ROW_TOWER[precision]
  run(precision, d, hidden, out, _rows(m), masked=True)


@pytest.mark.parametrize('precision', PRECISIONS)
def test_rows_large_odd(precision):
  """About 10^5 rows: many row splits, the last one short."""
  d, hidden, out = ROW_TOWER[precision]
  m = _rows('big')
  plan = R.Plan(R.Cfg([d] + hidden + [out]), m, _sms())
  assert plan.rows_per_split > 256 and m % plan.rows_per_split != 0
  run(precision, d, hidden, out, m, masked=True)


@pytest.mark.parametrize('bn', [False, True])
@pytest.mark.parametrize('precision', PRECISIONS)
def test_zero_rows(precision, bn):
  """M = 0: the forward launches nothing, the backward overwrites the gradient with zeros."""
  _C = _lib()
  prec = {'fp32': _C.PREC_FP32, 'tf32x3': _C.PREC_TF32X3, 'tf32': _C.PREC_TF32}[precision]
  tower = _tower(precision, 12, [24], 1, 'relu', bn, bn, 0.0, True, seed=5)
  cfg = tower._run_cfg()
  x = torch.ones(1, 12, device='cuda')
  ds = torch.ones(1, 1, device='cuda')
  scores = torch.full((1, 1), 7.0, device='cuda')
  ws = tower._new_workspace(0)
  state0 = tower.bn_state.clone()
  torch.cuda.synchronize()
  n0 = _C.lib.tfr_launch_count()
  _C.check(_C.lib.tfr_mlp_fwd(_C.ptr(x), 0, ctypes.byref(cfg), _C.ptr(tower.flat.data), None,
                              _C.ptr(ws), _C.ptr(scores), prec, _C.stream()))
  assert _C.lib.tfr_launch_count() == n0
  grads = torch.full_like(tower.flat.data, float('nan'))
  _C.check(_C.lib.tfr_mlp_bwd(_C.ptr(x), 0, ctypes.byref(cfg), _C.ptr(tower.flat.data),
                              _C.ptr(ds), None, _C.ptr(ws), _C.ptr(grads), prec, _C.stream()))
  torch.cuda.synchronize()
  assert (grads == 0).all()
  assert scores.item() == 7.0 and torch.equal(tower.bn_state, state0)


# ---------------------------------------------------------------------- fp32 widths ---
FP32_WIDTHS = [1, 3, 5, 7, 127, 128, 129, 255, 257]


@pytest.mark.parametrize('role', ['input', 'hidden', 'feeding'])
@pytest.mark.parametrize('w', FP32_WIDTHS)
def test_fp32_widths(w, role):
  """The SGEMM's K tails (1..7 of a k block of 8) and both 128-wide tile edges, as the tower's
  input width, a hidden width and the width feeding the output layer."""
  d, hidden, out = {'input': (w, [24], 1), 'hidden': (12, [w, 20], 2),
                    'feeding': (12, [20, w], 3)}[role]
  run('fp32', d, hidden, out, 300, masked=out == 1)


# ---------------------------------------------------------------------- TF32 widths ---
TF32_WIDTHS = [124, 128, 132, 252, 256, 260]


@pytest.mark.parametrize('role', ['input', 'hidden', 'feeding'])
@pytest.mark.parametrize('w', TF32_WIDTHS)
@pytest.mark.parametrize('precision', ['tf32x3', 'tf32'])
def test_tf32_widths(precision, w, role):
  d, hidden, out = {'input': (w, [64], 1), 'hidden': (20, [w, 36], 1),
                    'feeding': (20, [36, w], 2)}[role]
  run(precision, d, hidden, out, 600, masked=out == 1)


@pytest.mark.parametrize('hidden,out', [([1024], 1), ([64, 1024], 4), ([1024], 5)])
@pytest.mark.parametrize('precision', PRECISIONS)
def test_1024_feeds_output_layer(precision, hidden, out):
  """The plan's limit on the width feeding the output layer."""
  run(precision, 20, hidden, out, 700)


# (hidden widths, fused?): first width <= 256, later ones <= 128 (mlp_tc_fused_fwd_ok)
FUSED_LIMITS = {
    'first256': ([256, 128], True), 'first260': ([260, 128], False),
    'later128': ([256, 128, 128], True), 'later132': ([256, 132, 64], False),
    'last128': ([128], True), 'last132': ([132], False),
    'out8': ([128, 64], True),
}


@pytest.mark.parametrize('name', sorted(FUSED_LIMITS))
def test_fused_forward_limits(name):
  hidden, fused = FUSED_LIMITS[name]
  out = 8 if name == 'out8' else 1
  n, _ = run('tf32x3', 24, hidden, out, 1000, masked=out == 1)
  # split + fused kernel, or split + one GEMM per hidden layer + the output layer
  assert n == (2 if fused else len(hidden) + 2), (name, n)


# ---------------------------------------------------------------------------- depth ---
DEPTH = {'fp32': ([], [33], [33, 31, 29, 27, 25, 23, 21]),
         'tf32x3': ([], [64], [64, 48, 40, 36, 32, 28, 24]),
         'tf32': ([], [64], [64, 48, 40, 36, 32, 28, 24])}


@pytest.mark.parametrize('depth', [0, 1, 7])
@pytest.mark.parametrize('precision', PRECISIONS)
def test_depth(precision, depth):
  """No hidden layer, one, and the plan's maximum of 8 Dense layers."""
  hidden = DEPTH[precision][{0: 0, 1: 1, 7: 2}[depth]]
  assert len(hidden) == depth
  run(precision, 20, hidden, 2, 700)


# ------------------------------------------------------------------- output units ---
D_OUT, K_OUT = 20, 64
OUT_CASES = [(1, True, 6000), (1, False, 1000), (2, False, 6000), (3, False, 1000),
             (4, False, 6000), (5, False, 6000), (8, False, 1000)]


def _out_kernel(o):
  """mlp_out_layer_bwd2 (mlp_simt.cu) at K = 64 with 16-byte aligned H, W and dH."""
  if o == 1:
    return 'out_layer_bwd2_o1_kernel'
  if o <= 4:
    return 'out_layer_bwd2_vec_kernel<%d>' % o
  return 'out_layer_bwd2_kernel'


def _reduce_kernel(o, m):
  """mlp_reduce2 over the output layer's [K O + O] block slots; its gradient slice starts at
  w_off[1] = (D + 1) K floats."""
  n = K_OUT * o + o
  if n % 4 == 0 and (D_OUT + 1) * K_OUT % 4 == 0:
    return 'reduce2_vec_kernel'
  if R.Plan(R.Cfg([D_OUT, K_OUT, o]), m, _sms()).out_slots >= 128 and n <= 4096:
    return 'reduce_tall_kernel'
  return 'reduce2_kernel'


def test_out_cases_cover_every_variant():
  kernels = {_out_kernel(o) for o, _, _ in OUT_CASES}
  assert kernels == {'out_layer_bwd2_o1_kernel', 'out_layer_bwd2_kernel'} | {
      'out_layer_bwd2_vec_kernel<%d>' % o for o in (2, 3, 4)}


@pytest.mark.parametrize('o,masked,m', OUT_CASES)
@pytest.mark.parametrize('precision', ['tf32x3', 'tf32'])
def test_output_units_tc(precision, o, masked, m):
  _, launches = run(precision, D_OUT, [K_OUT], o, m, masked=masked, profile=True)
  names = [n for n, _, _ in launches]
  kern = _out_kernel(o)
  assert kern in names, (kern, names)
  assert names[names.index(kern) + 1] == _reduce_kernel(o, m), names


def test_output_units_tc_cover_every_reduction():
  sms = _sms()
  assert {_reduce_kernel(o, m) for o, _, m in OUT_CASES} == {
      'reduce2_vec_kernel', 'reduce_tall_kernel', 'reduce2_kernel'}, sms


@pytest.mark.parametrize('o,masked', [(1, True), (1, False), (2, False), (3, False),
                                      (4, False), (5, False), (8, False)])
def test_output_units_fp32(o, masked):
  _, launches = run('fp32', 13, [37], o, 1000, masked=masked, profile=True)
  assert 'out_layer_bwd_kernel' in [n for n, _, _ in launches]


# ----------------------------------------------------------------- BN and dropout ---
BN_TOWER = {'fp32': (13, [513, 37], 1), 'tf32x3': (20, [260, 36], 1),
            'tf32': (20, [260, 36], 1)}
BN_CASES = list(itertools.product([True, False], ['relu', None], [False, True]))


@pytest.mark.parametrize('training,act,input_bn', BN_CASES)
@pytest.mark.parametrize('precision', PRECISIONS)
def test_batch_norm_dropout(precision, training, act, input_bn):
  """BN widths over 256 columns (col_reduce_kernel walks several column blocks) at
  M = 256 k +- 1 rows (a partial last reduction block, or one row in it)."""
  d, hidden, out = BN_TOWER[precision]
  m = [511, 513, 767, 769][BN_CASES.index((training, act, input_bn)) % 4]
  run(precision, d, hidden, out, m, act=act, bn=True, input_bn=input_bn, dropout=0.2,
      training=training, masked=True)


@pytest.mark.parametrize('act', ['relu', None])
@pytest.mark.parametrize('precision', PRECISIONS)
def test_dropout_without_bn(precision, act):
  d, hidden, out = BN_TOWER[precision]
  run(precision, d, hidden, 2, 257, act=act, dropout=0.3)


# ----------------------------------------------------------------- input alignment ---
ALIGN = {'hidden': ([24], False), 'no_hidden': ([], False), 'input_bn': ([24], True)}


@pytest.mark.parametrize('name', sorted(ALIGN))
@pytest.mark.parametrize('precision', PRECISIONS)
def test_input_at_4_byte_offset(precision, name):
  """X as a contiguous view 4 bytes into its storage.  fp32 must be right; the TF32 modes
  must be right or refuse with ValueError (the fused forward declines an unaligned X, the
  per-layer GEMM needs 16-byte operands), never fault."""
  hidden, input_bn = ALIGN[name]
  try:
    run(precision, 12, hidden, 1, 300, input_bn=input_bn, x_offset=1, masked=True)
  except ValueError as e:
    assert precision != 'fp32', e
    assert '16-byte' in str(e), e
  torch.cuda.synchronize()
