"""The scorer tower's CUDA-core output layer (Dense(K -> O), O <= 8) on every variant its
dispatch selects, against the fp64 oracle (fp32, tf32x3, tf32) or the fp64 emulation of the
bf16 roundings (bf16).

Every tower has one hidden layer of width K (identity activation; bf16: ReLU over exact
activations), so the check covers the output layer's own gradient, the dH it hands to the
hidden layer and the column sums that become that layer's bias gradient, without ReLU gate
flips loosening the bar.  Each case restates the dispatch rule it is named for and checks,
from the kernels the call launched (torch.profiler), that the rule's variant ran:

  fp32            out_layer_bwd_kernel, one thread per k (mlp_simt.cu:152, 667-679)
  tf32x3 / tf32   mlp_out_layer_bwd2 (mlp_simt.cu:546-599): o1, vec<O>, generic
  bf16            mlp_bf16.cu:394-415 (forward), 434-469 (backward): fast<C, O>, generic
  reduction       mlp_reduce2 (mlp_simt.cu:522-544) of the per-block output-layer slots
                  (tf32x3 / tf32 / bf16): reduce2_vec, reduce_tall, reduce2

M = 1000 keeps the output-layer backward below 128 block slots, M = 6000 above it (the slot
count is make_mlp_plan's out_slots, capi.cu:176-179).

On an H100 SXM (132 SMs, 700 W) this file and tests/test_gam_limits_gpu.py ran in 24 s
together (125 cases, host-side oracle work included).
"""
import math

import pytest
import torch

from oracle import scorer as OS
from _tower_refs import _emulated_bf16_tower, kernel_launches

pytestmark = pytest.mark.gpu

M_SMALL, M_LARGE = 1000, 6000
D = 16            # tower input width


@pytest.fixture(autouse=True)
def _need_cuda():
  if not torch.cuda.is_available():
    pytest.skip('no CUDA device')


def _rel(a, b):
  a = torch.as_tensor(a).detach().cpu().double()
  b = torch.as_tensor(b).detach().cpu().double()
  return float((a - b).abs().max() / (b.abs().max() + 1e-30))


# ------------------------------------------------------------ dispatch mirrors ---
def tc_out_kernel(k, o, masked):
  """mlp_out_layer_bwd2 (mlp_simt.cu:549, 564, 587): the tower's H, W and dH are 16-byte
  aligned at these shapes (K % 4 == 0, one hidden layer over D = 16 inputs)."""
  if o == 1 and k % 4 == 0 and k <= 1024:
    return 'out_layer_bwd2_o1_kernel'
  if 2 <= o <= 4 and not masked and k % 4 == 0 and k <= 1024:
    return 'out_layer_bwd2_vec_kernel<%d>' % o
  return 'out_layer_bwd2_kernel'


def bf16_out_kernels(k, o):
  """(forward, backward) output-layer kernels of mlp_bf16.cu:394-415 / 434-469
  (kFastK = 128, kFastO = 2)."""
  if k <= 128 and o <= 2:
    t = '<%d,%d>' % (1 if k <= 64 else 2, 1 if o == 1 else 2)
    return 'out_fwd_bf16_fast_kernel' + t, 'out_bwd_bf16_fast_kernel' + t
  return 'out_fwd_bf16_kernel', 'out_bwd_bf16_kernel'


def out_slots(m):
  """make_mlp_plan (capi.cu:177-179): about 4 blocks per SM, at least 16 rows each."""
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  rows = ((m + 4 * sms - 1) // (4 * sms) + 3) // 4 * 4
  rows = max(rows, 16)
  return (m + rows - 1) // rows


def reduce_kernel(k, o, m):
  """mlp_reduce2 (mlp_simt.cu:526-540) over the output layer's [K * O + O] slots: the slot
  stride is a multiple of 64 floats and the gradient slice starts at w_off[1] = (D + 1) K,
  16-byte aligned when K % 4 == 0."""
  n = k * o + o
  if n % 4 == 0 and (D + 1) * k % 4 == 0:
    return 'reduce2_vec_kernel'
  if out_slots(m) >= 128 and n <= 4096:
    return 'reduce_tall_kernel'
  return 'reduce2_kernel'


def _after(launches, name):
  """The launch that follows the first launch of `name`."""
  names = [n for n, _, _ in launches]
  assert name in names, (name, names)
  return launches[names.index(name) + 1]


# ---------------------------------------------------------------- fp32 / tf32 ---
def _tower(tfr, k, o, precision, seed):
  tower = tfr.keras.layers.create_tower([k], o, activation=None, use_batch_norm=False,
                                        dropout=0, input_dim=D, seed=seed, precision=precision)
  g = torch.Generator().manual_seed(seed + 1)
  with torch.no_grad():
    for i in range(2):
      tower.bias(i).copy_(torch.rand(tower.dims[i + 1], generator=g) * 0.4 - 0.2)
  params = {'dense_w': [tower.kernel(i).detach().cpu().double().clone().requires_grad_()
                        for i in range(2)],
            'dense_b': [tower.bias(i).detach().cpu().double().clone().requires_grad_()
                        for i in range(2)]}
  return tower, params


def _run_vs_oracle(precision, m, k, o):
  """Forward and backward of a [D, K, O] identity tower against the fp64 oracle; a
  RestoreList mask on O = 1.  Returns (scores error, gradient error, launches), errors in
  max-norm relative to the largest entry."""
  import ranking_b200 as tfr
  seed = 1000 * o + k + m
  tower, params = _tower(tfr, k, o, precision, seed)
  assert tower.precision == precision
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(m, D, generator=g)
  up = torch.randn(m, o, generator=g)
  mask = torch.rand(m, generator=g) > 0.15 if o == 1 else None

  def step():
    tower.flat.grad = None
    y = tower(x.cuda(), mask=None if mask is None else mask.cuda())
    (y * up.cuda()).sum().backward()
    return y

  y, launches = kernel_launches(step)
  ref = OS.tower_forward(x.double(), params, activation=None)
  ups = up.double()
  got, ref_s = y.detach().cpu().double(), ref.detach()
  if mask is not None:
    fill = got[~mask]
    assert float(fill.max()) == float(fill.min()) == pytest.approx(math.log(1e-10), rel=1e-6)
    ups = ups * mask.double().reshape(-1, 1)
    got, ref_s = got[mask], ref_s[mask]
  (ref * ups).sum().backward()
  want = torch.cat([torch.cat([w.grad.reshape(-1), b.grad.reshape(-1)])
                    for w, b in zip(params['dense_w'], params['dense_b'])])
  e_s, e_g = _rel(got, ref_s), _rel(tower.flat.grad, want)
  print('%s K=%d O=%d M=%d: scores %.2e grads %.2e' % (precision, k, o, m, e_s, e_g))
  return e_s, e_g, launches


FP32_CASES = [(k, o, m) for k in (12, 37, 260, 1024) for o in (1, 3, 4, 5, 8)
              for m in (M_SMALL, M_LARGE)]


@pytest.mark.parametrize('k,o,m', FP32_CASES, ids=['K%d-O%d-M%d' % c for c in FP32_CASES])
def test_fp32_out_layer(k, o, m):
  """fp32 (FFMA) path: out_layer_fwd_kernel, then out_layer_bwd_kernel with round32(K)
  threads (up to 1024) and O of its 8 output registers live, its partials summed by
  reduce_partials_kernel.  Tolerances of test_tower_forward_backward: 1e-5 (scores) and
  5e-5 (gradients).  Measured (H100, largest over the cases): 2.1e-7 / 8.2e-7."""
  e_s, e_g, launches = _run_vs_oracle('fp32', m, k, o)
  names = [n for n, _, _ in launches]
  assert 'out_layer_fwd_kernel' in names, names
  bwd = [b for n, _, b in launches if n == 'out_layer_bwd_kernel']
  assert bwd == [((k + 31) // 32 * 32, 1, 1)], (bwd, names)
  assert e_s <= 1e-5, e_s
  assert e_g <= 5e-5, e_g


TC_CASES = [(k, o, m) for k in (12, 260, 1024) for o in (1, 3, 4, 5, 8)
            for m in (M_SMALL, M_LARGE)]
TC_VARIANT = {1: 'o1', 3: 'vec3', 4: 'vec4'}


@pytest.mark.parametrize('k,o,m', TC_CASES, ids=['%s-K%d-O%d-M%d' % (
    TC_VARIANT.get(c[1], 'generic'), *c) for c in TC_CASES])
def test_tf32x3_out_layer(k, o, m):
  """3xTF32 path: the output layer runs mlp_out_layer_bwd2's o1 (O = 1, masked here), vec<3>,
  vec<4> or generic (O = 5, 8) kernel; K = 1024 leaves o1 and vec one row lane (RL = 1) and
  K = 260 a partly idle lane group.  The slots are reduced by reduce2_vec (O = 4, 8),
  reduce_tall (at least 128 slots) or reduce2.  Tolerances of test_tower_tensor_core_path:
  1e-5 / 5e-5.  Measured (H100, largest over the cases): 3.4e-7 / 2.2e-6."""
  kern = tc_out_kernel(k, o, o == 1)
  assert kern == {1: 'out_layer_bwd2_o1_kernel', 3: 'out_layer_bwd2_vec_kernel<3>',
                  4: 'out_layer_bwd2_vec_kernel<4>'}.get(o, 'out_layer_bwd2_kernel')
  red = reduce_kernel(k, o, m)
  if o in (4, 8):
    assert red == 'reduce2_vec_kernel'
  elif m == M_LARGE and k * o + o <= 4096:
    assert red == 'reduce_tall_kernel' and out_slots(m) >= 128
  else:
    assert red == 'reduce2_kernel'
  e_s, e_g, launches = _run_vs_oracle('tf32x3', m, k, o)
  assert _after(launches, kern)[0] == red, launches
  assert e_s <= 1e-5, e_s
  assert e_g <= 5e-5, e_g


def test_tf32_out_layer_generic():
  """Single-pass TF32 through the generic output-layer kernel (O = 5) above the tall-slot
  threshold, at the tolerances of test_tower_tensor_core_path: 5e-3 / 0.15.
  Measured (H100): 8.6e-4 / 7.2e-4."""
  k, o, m = 260, 5, M_LARGE
  assert tc_out_kernel(k, o, False) == 'out_layer_bwd2_kernel'
  assert reduce_kernel(k, o, m) == 'reduce_tall_kernel'
  e_s, e_g, launches = _run_vs_oracle('tf32', m, k, o)
  assert _after(launches, 'out_layer_bwd2_kernel')[0] == 'reduce_tall_kernel', launches
  assert e_s <= 5e-3, e_s
  assert e_g <= 0.15, e_g


# ----------------------------------------------------------------------- bf16 ---
BF16_CASES = [(k, o, m) for k in (64, 128, 136, 512) for o in (1, 2, 3, 8)
              for m in (M_SMALL, M_LARGE)]


def _bf16_id(k, o, m):
  v = 'fast%d%d' % (1 if k <= 64 else 2, o) if k <= 128 and o <= 2 else 'generic'
  return '%s-K%d-O%d-M%d' % (v, k, o, m)


@pytest.mark.parametrize('k,o,m', BF16_CASES, ids=[_bf16_id(*c) for c in BF16_CASES])
def test_bf16_out_layer(k, o, m):
  """bf16 path against the fp64 emulation of its roundings.  X, W_0 and b_0 lie on a
  dyadic grid (multiples of 1/2, 1/8 and 1/16) so that every hidden activation is exact in
  fp32 and in bf16: the stored H is the emulation's H bit for bit, and the output layer's
  own gradient (W_L, b_L) and the hidden bias gradient (column sums of dH before its bf16
  rounding) differ from the emulation only by fp32 accumulation order.  They and the scores
  are held at 2e-6 of the largest entry, the whole gradient (its dW_0 sees the bf16
  rounding of dH) at 2e-4 (test_tower_bf16_matches_emulation allows 5e-3 for random
  activations).
  Measured (H100, largest over the cases): scores 1.8e-7, W_L / b_L 2.7e-7, hidden bias
  3.3e-7, whole gradient 2.4e-5."""
  import ranking_b200 as tfr
  fwd_k, bwd_k = bf16_out_kernels(k, o)
  assert bwd_k == ('out_bwd_bf16_kernel' if k > 128 or o > 2 else
                   'out_bwd_bf16_fast_kernel<%d,%d>' % (1 if k <= 64 else 2, o))
  red = reduce_kernel(k, o, m)
  assert red == ('reduce2_vec_kernel' if o == 8 else
                 'reduce_tall_kernel' if m == M_LARGE and k * o + o <= 4096 else
                 'reduce2_kernel')
  seed = 7 * k + o + m
  g = torch.Generator().manual_seed(seed)
  tower = tfr.keras.layers.create_tower([k], o, activation='relu', use_batch_norm=False,
                                        dropout=0, input_dim=D, precision='bf16', seed=seed)
  with torch.no_grad():
    tower.kernel(0).copy_(torch.randint(-4, 5, (D, k), generator=g).float() / 8)
    tower.bias(0).copy_(torch.randint(-4, 5, (k,), generator=g).float() / 16)
    tower.bias(1).copy_(torch.rand(o, generator=g) * 0.4 - 0.2)
  x = torch.randint(-2, 3, (m, D), generator=g).float() / 2
  dscores = torch.randn(m, o, generator=g)
  mask = torch.rand(m, generator=g) > 0.1 if o == 1 else None
  ws = [tower.kernel(i).detach().cpu() for i in range(2)]
  bs = [tower.bias(i).detach().cpu() for i in range(2)]

  def step():
    tower.flat.grad = None
    y = tower(x.cuda(), mask=None if mask is None else mask.cuda())
    y.backward(dscores.cuda())
    return y

  y, launches = kernel_launches(step)
  names = [n for n, _, _ in launches]
  assert fwd_k in names, names
  assert _after(launches, bwd_k)[0] == red, names
  ds_eff = dscores * mask.reshape(-1, 1).float() if mask is not None else dscores
  ref_s, ref_g = _emulated_bf16_tower(x, ws, bs, ds_eff, relu=True)
  got = y.detach().double().cpu()
  if mask is not None:
    fill = got[~mask]
    assert float(fill.max()) == float(fill.min()) == pytest.approx(math.log(1e-10), rel=1e-6)
    got, ref_s = got[mask], ref_s[mask]
  grad = tower.flat.grad.detach().double().cpu()
  b0 = slice(D * k, D * k + k)                        # hidden bias: column sums of dH
  out = slice(D * k + k, D * k + k + k * o + o)       # W_L, b_L
  e_s, e_out, e_b0, e_all = (_rel(got, ref_s), _rel(grad[out], ref_g[out]),
                             _rel(grad[b0], ref_g[b0]), _rel(grad, ref_g))
  print('bf16 K=%d O=%d M=%d: scores %.2e out-layer grads %.2e hidden bias %.2e all %.2e'
        % (k, o, m, e_s, e_out, e_b0, e_all))
  assert e_s <= 2e-6, e_s
  assert e_out <= 2e-6, e_out
  assert e_b0 <= 2e-6, e_b0
  assert e_all <= 2e-4, e_all
