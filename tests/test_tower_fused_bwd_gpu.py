"""GPU tests of the fused 3xTF32 dW_0 backward (csrc/mlp_tc_fused_bwd.cu).

For towers within mlp_tc_fused_bwd_ok, tfr_mlp_bwd computes dZ_0 = (dZ_1 W_1^T) * relu'(H_0)
and dW_0's split-K partials in one kernel and does not store dZ_0.  The per-layer path is
replayed through tfr_tc_gemm from the dZ_1 the backward leaves in the workspace: the dZ GEMM
(W_1 pre-split as the workspace holds it, sign-word mask), then the swapped dW GEMM with the
plan's splits.  dW_0's partial slots in the workspace must equal that GEMM's split outputs bit
for bit, db_0 must meet an fp64 bound (its column sums are taken in another order), and
tfr_mlp_input_grad, which recomputes dZ_0, must give the per-layer dX bits.  Towers just past a
limit must take the per-layer path: the workspace then holds dZ_0 with the replayed bits.
"""
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import pytest
import torch

pytestmark = pytest.mark.gpu

CONFIG2_M = 204800   # 124 splits of 1664 rows; the last holds one 128-row tile
ROWS = (1, 127, 128, 129, 1663, 1665, 128 * 1024 + 5)
# (dims[0], dims[1], dims[2], activation).  dims[0] of 65..128, or dims[1] <= 128 with dims[0]
# past 64, puts dW_0 in the direct orientation: those towers keep the per-layer path.
SHAPES = [(136, 256, 128, 'relu'), (4, 256, 64, 'relu'), (20, 200, 8, 'relu'),
          (132, 256, 256, None), (136, 160, 128, 'relu'), (64, 256, 32, 'relu'),
          (12, 200, 256, 'relu'), (4, 32, 64, 'relu'), (128, 128, 256, 'relu'),
          (132, 64, 128, None), (136, 64, 8, 'relu')]


def _folded(gn):
  return gn % 128 if gn > 128 and gn % 128 <= 8 else 0


def _tile_units(gm, gn):
  return (gm + 127) // 128 * ((gn - _folded(gn) + 63) // 64)


def _fused(d0, d1, d2):
  """mlp_tc_fused_bwd_ok for a 3xTF32 tower without BN / dropout / input BN."""
  return (d0 <= 136 and d1 <= 256 and d2 <= 256 and
          _tile_units(d1, d0) < _tile_units(d0, d1))


def _lib():
  import __graft_entry__ as entry
  entry.build()
  from ranking_b200 import _C
  return _C


def _tower(d0, hidden, out, act, seed, precision='tf32x3'):
  import ranking_b200 as tfr
  t = tfr.keras.layers.create_tower(hidden, out, activation=act, use_batch_norm=False,
                                    dropout=0, input_dim=d0, seed=seed, precision=precision)
  with torch.no_grad():
    for i in range(len(t.dims) - 1):
      t.bias(i).uniform_(-0.2, 0.2)
  return t


def _layout(dims, m, sms):
  """Float offsets of make_mlp_plan's workspace regions (no BN / dropout)."""
  up = lambda n: (n + 63) // 64 * 64
  L = len(dims) - 2
  w, act, bits = 0, [], []
  for d in range(L):
    act.append(w)
    w += up(m * dims[d + 1])
    bits.append(w)
    w += up(m * ((dims[d + 1] + 31) // 32))
  max_hidden = max([1] + dims[1:L + 1])
  dz = []
  for _ in range(2):
    dz.append(w)
    w += up(m * max_hidden)
  per = (m + sms - 1) // sms
  rows = 256 if per < 256 else (per + 127) // 128 * 128
  splits = (m + rows - 1) // rows
  max_wb = max((dims[d] + 127) // 128 * 128 * dims[d + 1] + dims[d + 1] for d in range(L + 1))
  pstride = up(max_wb)
  partial = w
  w += splits * pstride
  n_params = sum(dims[d] * dims[d + 1] + dims[d + 1] for d in range(L + 1))
  whi = w
  wlo = w + up(n_params)
  w += 4 * up(n_params)
  w_off, off = [], 0
  for d in range(L + 1):
    w_off.append(off)
    off += dims[d] * dims[d + 1] + dims[d + 1]
  return dict(act=act, bits=bits, dz=dz, splits=splits, pstride=pstride, partial=partial,
              whi=whi, wlo=wlo, tile=w, tstride=up(max_hidden), w_off=w_off)


def _floats(ws):
  base = (-ws.data_ptr()) % 256
  return ws[base:base + (ws.numel() - base) // 4 * 4].view(torch.float32)


def _run(_C, tower, x, mask, prec, tasks=False, seed=0):
  """Forward, then a backward on a workspace whose dZ_0 region is NaN: (ws, flat, grads)."""
  m = x.shape[0]
  cfg = tower._run_cfg()
  ws = tower._new_workspace(m)
  flat = _floats(ws)
  O = tower.output_units
  m8 = None if mask is None else mask.to(torch.uint8).contiguous()
  out = torch.empty(m * O, device='cuda')
  fwd = _C.lib.tfr_mlp_fwd_tasks if tasks else _C.lib.tfr_mlp_fwd
  _C.check(fwd(_C.ptr(x), m, ctypes.byref(cfg), _C.ptr(tower.flat.data), _C.ptr(m8), _C.ptr(ws),
               _C.ptr(out), prec, _C.stream()))
  lay = _layout(tower.dims, m, torch.cuda.get_device_properties(0).multi_processor_count)
  L = len(tower.dims) - 2
  flat[lay['dz'][(L - 1) & 1]:][:m * tower.dims[1]].fill_(float('nan'))
  g = torch.Generator().manual_seed(seed)
  ds = torch.randn(m * O, generator=g).cuda()
  grads = torch.empty_like(tower.flat.data)
  if tasks:
    tw = (ctypes.c_float * O)(*[0.5 + 0.25 * o for o in range(O)])
    _C.check(_C.lib.tfr_mlp_bwd_tasks(_C.ptr(x), m, ctypes.byref(cfg), _C.ptr(tower.flat.data),
                                      _C.ptr(ds), tw, _C.ptr(m8), _C.ptr(ws), _C.ptr(grads),
                                      prec, _C.stream()))
  else:
    _C.check(_C.lib.tfr_mlp_bwd(_C.ptr(x), m, ctypes.byref(cfg), _C.ptr(tower.flat.data),
                                _C.ptr(ds), _C.ptr(m8), _C.ptr(ws), _C.ptr(grads), prec,
                                _C.stream()))
  torch.cuda.synchronize()
  return ws, flat, grads, lay


def _dz0_ref(_C, tower, flat, lay, m, act, passes):
  """dZ_0 by the per-layer dZ GEMM from the workspace's dZ_1."""
  d0, d1, d2 = tower.dims[:3]
  L = len(tower.dims) - 2
  dz1 = flat[lay['dz'][L & 1]:][:m * d2].view(m, d2).clone()
  if passes == 3:
    whi = flat[lay['whi'] + lay['w_off'][1]:][:d1 * d2].clone()
    wlo = flat[lay['wlo'] + lay['w_off'][1]:][:d1 * d2].clone()
  else:
    whi, wlo = tower.kernel(1).detach().contiguous(), None
  bits = flat[lay['bits'][0]:][:m * ((d1 + 31) // 32)].view(torch.int32).clone()
  dz0 = torch.empty(m, d1, device='cuda')
  relu = act == 'relu'
  _C.check(_C.lib.tfr_tc_gemm(
      _C.ptr(dz1), d2, _C.ptr(whi), d2, _C.ptr(wlo), _C.ptr(dz0), d1, m, d1, d2, 0, 0, passes,
      0, 3 if relu else 0, None, None, 0, 0, 1, 0, None, _C.ptr(bits) if relu else None,
      _C.stream()))
  torch.cuda.synchronize()
  return dz0


def _same_bits(got, want, what):
  assert got.shape == want.shape, (what, got.shape, want.shape)
  diff = (got.view(torch.int32) != want.view(torch.int32)).nonzero()
  assert diff.numel() == 0, (what, diff[:8].tolist(), got[tuple(diff[0])].item(),
                             want[tuple(diff[0])].item())


def _check_fused(_C, tower, x, mask, act, tasks=False):
  m = x.shape[0]
  d0, d1 = tower.dims[:2]
  ws, flat, grads, lay = _run(_C, tower, x, mask, _C.PREC_TF32X3, tasks=tasks, seed=m)
  L = len(tower.dims) - 2
  dz0_region = flat[lay['dz'][(L - 1) & 1]:][:m * d1]
  dz0 = _dz0_ref(_C, tower, flat, lay, m, act, 3)
  if _fused(*tower.dims[:3]):
    # with L odd the buffer also holds dZ_{L-1}, the output layer's signal, at its start
    other = m * tower.dims[L] if L % 2 else 0
    assert torch.isnan(dz0_region[other:]).all(), 'the fused backward stores no dZ_0'
  else:
    _same_bits(dz0_region.view(m, d1), dz0, 'dZ_0 of the per-layer path')
  # dW_0's partial slots against the per-layer dW GEMM with the plan's splits, in the
  # orientation mlp_tc_weight_grad picks
  splits, pstride = lay['splits'], lay['pstride']
  part = torch.zeros(splits * pstride, device='cuda')
  if _tile_units(d1, d0) < _tile_units(d0, d1):   # swapped: dW_0^T = dZ_0^T X, stored transposed
    a, lda, b, ldb, gm, gn, tr = dz0, d1, x, d0, d1, d0, 1
  else:
    a, lda, b, ldb, gm, gn, tr = x, d0, dz0, d1, d0, d1, 0
  _C.check(_C.lib.tfr_tc_gemm(
      _C.ptr(a), lda, _C.ptr(b), ldb, None, _C.ptr(part), d1, gm, gn, m, 1, 1, 3, 1, 0, None,
      None, 0, tr, splits, pstride, None, None, _C.stream()))
  torch.cuda.synchronize()
  got = flat[lay['partial']:][:splits * pstride].view(splits, pstride)[:, :d0 * d1]
  _same_bits(got, part.view(splits, pstride)[:, :d0 * d1], 'dW_0 partial slots')
  # db_0: fp64 column sums of dZ_0, within 1e-5 of the sum of magnitudes
  w_off = lay['w_off']
  db0 = grads[w_off[0] + d0 * d1:][:d1].double()
  ref = dz0.double().sum(0)
  bound = 1e-5 * dz0.double().abs().sum(0)
  assert ((db0 - ref).abs() <= bound).all(), ((db0 - ref).abs() - bound).max().item()
  dw0 = grads[w_off[0]:][:d0 * d1].double().view(d0, d1)
  ref_w = x.double().t() @ dz0.double()
  scale = x.double().abs().t() @ dz0.double().abs()
  assert ((dw0 - ref_w).abs() <= 1e-5 * scale + 1e-30).all()
  # the input gradient recomputes dZ_0 and matches the per-layer dX on a column range
  col0, ncols = (d0 // 4) // 4 * 4, max(4, d0 // 2) // 4 * 4
  ncols = min(ncols, d0 - col0)
  cfg = tower._run_cfg()
  dx = torch.full((m, ncols), float('nan'), device='cuda')
  _C.check(_C.lib.tfr_mlp_input_grad(ctypes.byref(cfg), m, _C.ptr(tower.flat.data), _C.ptr(ws),
                                     col0, ncols, _C.ptr(dx), ncols, _C.PREC_TF32X3, _C.stream()))
  torch.cuda.synchronize()
  _same_bits(dz0_region.view(m, d1), dz0, 'dZ_0 recomputed by tfr_mlp_input_grad')
  w0 = w_off[0] + col0 * d1
  whi = flat[lay['whi'] + w0:][:ncols * d1].clone()
  wlo = flat[lay['wlo'] + w0:][:ncols * d1].clone()
  want = torch.empty(m, ncols, device='cuda')
  _C.check(_C.lib.tfr_tc_gemm(
      _C.ptr(dz0), d1, _C.ptr(whi), d1, _C.ptr(wlo), _C.ptr(want), ncols, m, ncols, d1, 0, 0, 3,
      0, 0, None, None, 0, 0, 1, 0, None, None, _C.stream()))
  torch.cuda.synchronize()
  _same_bits(dx, want, 'dX')


def _inputs(m, d0, masked, seed):
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(m, d0, generator=g).cuda()
  mask = (torch.rand(m, generator=g) > 0.3).cuda() if masked else None
  return x, mask


@pytest.mark.parametrize('m', ROWS)
@pytest.mark.parametrize('shape', SHAPES, ids=lambda s: '%d-%d-%d-%s' % s)
def test_fused_dw0_matches_per_layer(shape, m):
  _C = _lib()
  d0, d1, d2, act = shape
  tower = _tower(d0, [d1, d2], 1, act, seed=7)
  x, mask = _inputs(m, d0, True, seed=m + d1)
  _check_fused(_C, tower, x, mask, act)


def test_fused_dw0_config2_rows():
  _C = _lib()
  tower = _tower(136, [256, 128, 64], 1, 'relu', seed=3)
  x, mask = _inputs(CONFIG2_M, 136, True, seed=1)
  _check_fused(_C, tower, x, mask, 'relu')


@pytest.mark.parametrize('m', (129, 4100))
def test_fused_dw0_tasks(m):
  _C = _lib()
  tower = _tower(136, [256, 128], 3, 'relu', seed=9)
  x, mask = _inputs(m, 136, True, seed=m)
  _check_fused(_C, tower, x, mask, 'relu', tasks=True)


# just past a limit: the per-layer path, which leaves dZ_0 in the workspace
PAST = {'d0_140': (140, 256, 64, 'tf32x3'), 'd1_264': (64, 264, 64, 'tf32x3'),
        'tf32': (136, 256, 64, 'tf32')}


@pytest.mark.parametrize('name', sorted(PAST))
def test_past_the_limits_takes_per_layer_path(name):
  _C = _lib()
  d0, d1, d2, prec = PAST[name]
  tower = _tower(d0, [d1, d2], 1, 'relu', seed=4, precision=prec)
  m = 1665
  x, mask = _inputs(m, d0, True, seed=2)
  code = _C.PREC_TF32X3 if prec == 'tf32x3' else _C.PREC_TF32
  ws, flat, grads, lay = _run(_C, tower, x, mask, code, seed=5)
  dz0 = _dz0_ref(_C, tower, flat, lay, m, 'relu', 3 if prec == 'tf32x3' else 1)
  region = flat[lay['dz'][1 & 1]:][:m * d1].view(m, d1)
  _same_bits(region, dz0, 'dZ_0 of the per-layer path')
