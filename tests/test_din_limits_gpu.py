"""DocumentInteractionAttention (K11, csrc/din.cu) backward and input gradient at its shape
limits, against oracle/din.py in fp64 with the input projection's ReLU gated by the kernel's
own decisions (a0 > 0 in its workspace) and every such gate checked to be admissible: equal to
the reference's own decision except where the pre-activation lies within the forward error
bound of 0.  Dropout and noise draws are replayed from their counter hashes.

The case table puts the backward's query / key row passes (kRows = 64) and key tiles
(kKT = 32) on both sides of their boundaries up to TFR_DIN_MAX_LIST = 1024, each KD template
of the attention kernels on both sides of its head_size boundary, num_heads * head_size = 512
at N = 1024, num_layers = TFR_DIN_MAX_LAYERS = 8, and the dW row split with two or more
32-row k blocks per split (M > 32 SMs) and a short last split.
`test_cases_cover_every_variant` recomputes that from the table.

Bars.  Every parameter block separately within 5e-5 relative L2 (the bar of test_din_gpu.py's
whole-vector comparison), every input-gradient window within 5e-5 (test_din_embedding_gpu.py).
The key bias is the one exception: softmax is invariant to a per-query shift of its logits,
which is all the key bias adds, so its exact gradient is 0 and what the kernel returns is the
rounding left in sum_j dK_j; it is held to 5e-5 of the norm of its kernel's gradient dW_k,
whose entries sum the same dK rows weighted by O(1) activations.

The query projection's blocks (W_q, b_q) are the other exception, for the same reason.  Their
gradient comes from dQ_i = scale sum_j dS_ij k_j, and sum_j dS_ij = 0, so the component that
every key row shares (the key bias, and the mean of x_j W_k) cancels out of the exact dQ_i.
attn_bwd_dq_kernel sums the N terms in order in fp32, so its rounding scales with
sum_j |dS_ij| |k_j|, shared component included, while the value that survives the
cancellation is ~ sqrt(N) times smaller than that sum (P_ij ~ 1 / N, with dS_ij of either
sign): the relative error grows with N, like N for a sum whose roundings have random signs.
dK_j = scale sum_i dS_ij q_i and dV_j = sum_i P~_ij dO_i are summed the same way over N
queries, but nothing cancels there (sum_i dS_ij is not 0, P~ >= 0), so their relative error
does not grow with N.  This file's own N <= 257 cases hold W_q and b_q to 5e-5; linear growth
beyond gives 5e-5 N / 256, 2e-4 at N = 1024 (an H100 SXM at 700 W gives 7e-5 there).
"""
import ctypes

import pytest
import torch

from oracle import din as odin
import _dasalc_refs
import _tower_fp64 as T

gpu = pytest.mark.gpu
SMS = 132            # H100 SXM; the GPU tests take the device's own count
K_ROWS, K_KT = 64, 32
SENTINEL = 1234.5
TOL = 5e-5

# (B, N, D, head_size, heads, layers, training)
CASES = [
    (3, 63, 136, 16, 2, 1, False),   # input gradient in two column chunks (3 HH = 96 < D)
    (3, 64, 8, 20, 1, 1, True),
    (3, 65, 16, 32, 2, 2, False),
    (3, 127, 8, 36, 2, 1, True),
    (3, 128, 12, 64, 2, 1, False),
    (3, 129, 8, 68, 1, 1, True),
    (3, 257, 16, 128, 1, 1, False),
    (3, 1000, 8, 32, 2, 1, True),
    (3, 40, 8, 16, 2, 8, True),      # TFR_DIN_MAX_LAYERS
    (5, 1000, 8, 16, 1, 1, True),    # M = 5000: two k blocks per dW split, a short last one
    (4, 1024, 16, 128, 4, 1, True),  # TFR_DIN_MAX_LIST with num_heads * head_size = 512
]
LARGEST = CASES[-1]


def kd(h):
  """TFR_DIN_DISPATCH: the KD template (head dimensions per thread) for head_size h."""
  return 4 if h <= 16 else 8 if h <= 32 else 16 if h <= 64 else 32


def dw_split(m, sms):
  """make_din_plan's dW row splits: (k blocks per split, splits, rows in the last split)."""
  kb = (m + 31) // 32
  per = (kb + sms - 1) // sms if kb else 1
  splits = (kb + per - 1) // per if kb else 1
  return per, splits, m - (splits - 1) * per * 32


# --------------------------------------------------------------------------- harness ---
def _mask(b, n, gen):
  """A full list, an all-padded list, a single-item list, then ragged ones."""
  m = torch.rand(b, n, generator=gen) < 0.6
  m[0] = True
  m[1] = False
  m[2] = False
  m[2, n // 2] = True
  return m


def _make(case, seed):
  from ranking_b200.keras import layers
  b, n, d, h, heads, nl, training = case
  gen = torch.Generator().manual_seed(seed)
  x = torch.randn(b, n, d, generator=gen)
  din = layers.DocumentInteractionAttention(heads, h, nl, dropout=0.2 if training else 0.0,
                                            input_noise_stddev=0.1 if training else None,
                                            seed=seed)
  din.build(d)
  with torch.no_grad():
    for name, t in odin.unflatten(din.flat.data, d, h, heads, nl).items():
      if name.startswith('b'):
        t.copy_(torch.randn(t.shape, generator=gen) * 0.2)
      if name.startswith('gamma'):
        t.copy_(1.0 + torch.randn(t.shape, generator=gen) * 0.2)
  dout = torch.randn(b * n, h, generator=gen)
  base = torch.randn(b * n, d + 8, generator=gen)
  return din, x, _mask(b, n, gen), dout, base


def _kernel(din, x, mask, dout, base, training):
  """tfr_din_fwd + tfr_din_bwd on one workspace (dout with row pitch h + 4), then the input
  gradient twice: all D columns written into a [M, D] buffer, and columns [4, D) accumulated
  onto `base` at row pitch D + 8, offset 2 columns."""
  from ranking_b200 import _C
  b, n, d = x.shape
  h, m = din.head_size, b * n
  cfg = din._run_cfg(training=training)
  ws = din._new_workspace(b, n)
  xg, m8 = x.cuda().contiguous(), mask.to(torch.uint8).cuda().contiguous()
  out = torch.empty(m, h, device='cuda')
  dg = torch.full((m, h + 4), SENTINEL, device='cuda')
  dg[:, :h] = dout.cuda()
  grads = torch.full_like(din.flat.data, float('nan'))
  st = _C.stream()
  _C.check(_C.lib.tfr_din_fwd(_C.ptr(xg), _C.ptr(m8), b, n, ctypes.byref(cfg),
                              _C.ptr(din.flat.data), _C.ptr(ws), _C.ptr(out), h, st))
  _C.check(_C.lib.tfr_din_bwd(_C.ptr(xg), _C.ptr(m8), b, n, ctypes.byref(cfg),
                              _C.ptr(din.flat.data), _C.ptr(dg), h + 4, _C.ptr(ws),
                              _C.ptr(grads), st))
  dx = torch.full((m, d), float('nan'), device='cuda')
  _C.check(_C.lib.tfr_din_input_grad(ctypes.byref(cfg), b, n, _C.ptr(din.flat.data), _C.ptr(ws),
                                     0, d, _C.ptr(dx), d, 0, st))
  acc = base.cuda()
  _C.check(_C.lib.tfr_din_input_grad(ctypes.byref(cfg), b, n, _C.ptr(din.flat.data), _C.ptr(ws),
                                     4, d - 4, ctypes.c_void_p(acc.data_ptr() + 4 * 2), d + 8, 1,
                                     st))
  torch.cuda.synchronize()
  return {'out': out, 'grads': grads, 'dx': dx, 'acc': acc, 'ws': ws, 'seed': cfg.seed}


def kernel_gate(ws, b, n, d, h, heads, nl):
  """[a0 > 0] of the input projection from a kernel call's workspace (make_din_plan: a0
  follows the packed q / k / v weights of every layer, from the first 256-byte boundary)."""
  hh = heads * h
  a0_off = nl * ((h * 3 * hh + 3 * hh + 63) // 64 * 64)
  base = (-ws.data_ptr()) % 256
  f = ws[base:base + (ws.numel() - base) // 4 * 4].view(torch.float32)
  return (f[a0_off:a0_off + b * n * h].view(b, n, h) > 0).double()


def input_band(x, flat, d, h, heads, nl, precision='tf32x3'):
  """Z_in = X W_in + b_in and its forward error bound C u (|X| |W_in| + |b_in|), u of one
  GEMM of depth D in the engine's accounting (tests/_tower_fp64.py)."""
  p = odin.unflatten(flat.detach(), d, h, heads, nl)
  u_p, u_acc, per_k = T.PRECISIONS[precision]
  z = x @ p['w_in'] + p['b_in']
  mag = x.abs() @ p['w_in'].abs() + p['b_in'].abs()
  return z, T.C * (u_p + (per_k * d + 1) * u_acc) * mag


def reference(din, x, mask, dout, seed, training, gate, dev):
  """fp64 outputs, flat gradient and dX of sum(dout * din(x)), the ReLU gated by `gate`."""
  b, n, d = x.shape
  keeps = noise = None
  if training and din.dropout > 0:
    keeps = [(a.to(dev), o.to(dev)) for a, o in odin.keep_masks(
        seed, b, n, din.num_heads, din.head_size, din.num_layers, din.dropout)]
  if training and din.input_noise_stddev:
    noise = odin.noise(seed, b, n, din.head_size, din.input_noise_stddev).to(dev)
  flat = din.flat.detach().to(dev, torch.float64).requires_grad_()
  xd = x.detach().to(dev, torch.float64, copy=True).requires_grad_()
  out = odin.forward(xd, mask.to(dev), flat, din.num_heads, din.head_size, din.num_layers,
                     rate=din.dropout, keeps=keeps, noise_add=noise,
                     relu_gate=None if gate is None else gate.to(dev))
  (out * dout.to(dev).double().reshape(out.shape)).sum().backward()
  return out.detach(), flat.grad, xd.grad.reshape(b * n, d)


def _rel(a, b):
  a, b = a.double().reshape(-1), b.double().reshape(-1).to(a.device)
  return float((a - b).norm() / b.norm().clamp_min(1e-300))


def bars(n, d, h, heads, nl):
  """{block: bar} (see the module docstring)."""
  q = TOL * max(1.0, n / 256)
  return {name: q if name[:2] in ('wq', 'bq') else TOL
          for name, _ in odin.param_shapes(d, h, heads, nl)}


def block_errors(got, want, d, h, heads, nl):
  """{block: error} for every parameter block: relative L2, except the key biases (see the
  module docstring), whose error is taken relative to their kernel's gradient norm."""
  out, off, wnorm = {}, 0, {}
  got, want = got.double().reshape(-1), want.double().reshape(-1).to(got.device)
  for name, shape in odin.param_shapes(d, h, heads, nl):
    k = 1
    for s in shape:
      k *= s
    a, b = got[off:off + k], want[off:off + k]
    if name.startswith('wk'):
      wnorm[name[2:]] = float(b.norm())
    if name.startswith('bk'):
      out[name] = float((a - b).norm()) / max(wnorm[name[2:]], 1e-300)
    else:
      out[name] = _rel(a, b)
    off += k
  return out


# ------------------------------------------------------------------------ GPU cases ---
def _id(case):
  return 'B%d-N%d-D%d-h%d-H%d-L%d-%s' % (case[:6] + ('train' if case[6] else 'infer',))


@gpu
@pytest.mark.parametrize('case', CASES, ids=_id)
def test_gradients_at_limits(case):
  b, n, d, h, heads, nl, training = case
  din, x, mask, dout, base = _make(case, seed=n + h + nl)
  got = _kernel(din, x, mask, dout, base, training)
  m = b * n
  dev = 'cuda' if n >= 512 or m >= 4096 else 'cpu'
  gate = kernel_gate(got['ws'], b, n, d, h, heads, nl).to(dev)
  out, grads, dx = reference(din, x, mask, dout, got['seed'], training, gate, dev)
  # the gates are admissible
  z, band = input_band(x.to(dev).double(), din.flat.detach().to(dev, torch.float64), d, h,
                       heads, nl)
  assert _dasalc_refs.gate_ratio(gate, z, band) <= 1
  if m > 32 * SMS:   # the case meant for two or more k blocks per dW split reaches them here
    per, _, last = dw_split(m, torch.cuda.get_device_properties(0).multi_processor_count)
    assert per >= 2 and last < per * 32, (per, last)
  assert _rel(got['out'], out.reshape(m, h)) < 1e-5
  errs = block_errors(got['grads'], grads, d, h, heads, nl)
  bar = bars(n, d, h, heads, nl)
  bad = {k: (v, bar[k]) for k, v in errs.items() if not v < bar[k]}
  assert not bad, bad
  assert _rel(got['dx'], dx) < TOL
  acc = got['acc'].cpu().double()
  assert _rel(acc[:, 2:2 + d - 4] - base[:, 2:2 + d - 4].double(), dx[:, 4:].cpu()) < TOL
  assert torch.equal(got['acc'][:, :2].cpu(), base[:, :2])
  assert torch.equal(got['acc'][:, d - 2:].cpu(), base[:, d - 2:])


@gpu
def test_two_backward_calls_give_identical_bits():
  """At the largest shape, with dropout and noise: two identical calls, on fresh workspaces,
  return the same bits (no atomics anywhere in the backward)."""
  din, x, mask, dout, base = _make(LARGEST, seed=2)
  runs = []
  for _ in range(2):
    din._calls = 0   # the same seed both times
    runs.append(_kernel(din, x, mask, dout, base, True))
  for k in ('out', 'grads', 'dx', 'acc'):
    assert torch.equal(runs[0][k], runs[1][k]), k


# --------------------------------------------------------------- CPU: coverage ---
def test_cases_cover_every_variant():
  """The case table reaches every KD template on both sides of its boundary, two or more row
  passes of the attention backward, partial key tiles, the list-size limit at the widest
  heads, the layer limit, and two or more k blocks per dW split (at 132 SMs)."""
  hs = {c[3] for c in CASES}
  assert {kd(h) for h in hs} == {4, 8, 16, 32}
  for edge in (16, 32, 64):
    assert any(h <= edge and kd(h) == kd(edge) for h in hs)
    assert any(h > edge and kd(h) != kd(edge) for h in hs)
  ns = {c[1] for c in CASES}
  assert ns >= {63, 64, 65, 127, 128, 129, 257, 1000, 1024}
  assert any((n + K_ROWS - 1) // K_ROWS >= 2 for n in ns)
  assert any(n % K_KT for n in ns) and any(n % K_ROWS == 0 for n in ns)
  assert any(n == 1024 and h * heads == 512 for _, n, _, h, heads, _, _ in CASES)
  assert any(nl == 8 for *_, nl, _ in CASES)
  assert LARGEST[1] == 1024 and LARGEST[6]
  split = [dw_split(c[0] * c[1], SMS) for c in CASES]
  assert any(per >= 2 and last < per * 32 for per, _, last in split)
  assert any(c[0] * c[1] > 32 * SMS for c in CASES)


# -------------------------------------------------------- CPU: reference checks ---
def _cpu_case(training, seed=4, case=(4, 9, 12, 8, 2, 2)):
  case = case + (training,)
  from types import SimpleNamespace
  b, n, d, h, heads, nl, _ = case
  gen = torch.Generator().manual_seed(seed)
  n_params = sum(int(torch.tensor(s).prod()) for _, s in odin.param_shapes(d, h, heads, nl))
  flat = torch.randn(n_params, generator=gen, dtype=torch.float64) * 0.4
  for name, t in odin.unflatten(flat, d, h, heads, nl).items():
    if name.startswith('gamma'):
      t.add_(1.0)
  din = SimpleNamespace(flat=flat, num_heads=heads, head_size=h, num_layers=nl,
                        dropout=0.2 if training else 0.0,
                        input_noise_stddev=0.1 if training else None)
  x = torch.randn(b, n, d, generator=gen, dtype=torch.float64)
  dout = torch.randn(b * n, h, generator=gen, dtype=torch.float64)
  return din, x, _mask(b, n, gen), dout, case


@pytest.mark.parametrize('training', [True, False])
def test_gated_reference_equals_ungated(training):
  din, x, mask, dout, (b, n, d, h, heads, nl, _) = _cpu_case(training)
  seed = (9 << 32) | 1
  z, band = input_band(x, din.flat, d, h, heads, nl)
  assert z.abs().min().item() > 1e-9
  out0, g0, dx0 = reference(din, x, mask, dout, seed, training, None, 'cpu')
  out1, g1, dx1 = reference(din, x, mask, dout, seed, training, (z > 0).double(), 'cpu')
  for a, b_ in ((out0, out1), (g0, g1), (dx0, dx1)):
    assert torch.allclose(a, b_, rtol=1e-12, atol=1e-14)
  assert _dasalc_refs.gate_ratio((z > 0).double(), z, band) == 0


def test_negative_controls():
  """One small block off by 1e-3 passes a whole-vector comparison at the same bar but not
  the per-block one; a gate flipped outside its band is inadmissible."""
  din, x, mask, dout, (b, n, d, h, heads, nl, _) = _cpu_case(True, case=(4, 24, 16, 64, 4, 2))
  _, want, _ = reference(din, x, mask, dout, (9 << 32) | 1, True, None, 'cpu')
  assert max(block_errors(want, want, d, h, heads, nl).values()) == 0
  shapes = odin.param_shapes(d, h, heads, nl)
  for target in ('bo%d' % (nl - 1), 'beta0'):
    bad = want.clone()
    blk = odin.unflatten(bad, d, h, heads, nl)[target]
    blk.mul_(1 + 1e-3)
    assert _rel(bad, want) < TOL, target               # lost in the whole vector
    assert block_errors(bad, want, d, h, heads, nl)[target] > TOL, target
  assert len(shapes) == 2 + 10 * nl
  z, band = input_band(x, din.flat, d, h, heads, nl)
  gate = (z > 0).double()
  i = int((z.abs() / band).argmax())
  gate.view(-1)[i] = 1 - gate.view(-1)[i]
  assert _dasalc_refs.gate_ratio(gate, z, band) > 1
