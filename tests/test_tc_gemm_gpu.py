"""GPU tests of the wgmma TF32 GEMM engine (csrc/tc_gemm.cu) through the C ABI,
against a torch fp64 matmul of the same fp32 inputs.

Tolerance: 3xTF32 (passes=3) must be fp32-faithful: <= 2e-6 of |A||B| row/col
norms (well inside the 1e-5 north_star bar); single-pass TF32 <= 2e-3.
Run as a script (`python tests/test_tc_gemm_gpu.py`) to get a diagnostic table
that keeps going after failures.
"""
import itertools
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import pytest
import torch

pytestmark = pytest.mark.gpu


def _pack_bits(keep):
  """[gm, gn] bool -> int32 words [(gn + 31) // 32, gm], bit j = column 32 * w + j."""
  gm, gn = keep.shape
  nw = (gn + 31) // 32
  pad = torch.zeros(gm, nw * 32, dtype=torch.int64)
  pad[:, :gn] = keep.long()
  words = (pad.reshape(gm, nw, 32) << torch.arange(32)).sum(2)      # [gm, nw] in [0, 2^32)
  words = torch.where(words >= 2 ** 31, words - 2 ** 32, words)
  return words.t().contiguous().to(torch.int32)


def C_ptr(buf, offset):
  import ctypes
  return ctypes.c_void_p(buf.data_ptr() + 4 * offset)


def run_gemm(gm, gn, gk, a_mn, b_mn, passes, split_b, epi=0, act=0, transposed=0,
             splits=1, seed=0, want_bits=False, c_pad=0):
  """c_pad > 0: C starts c_pad floats into its buffer and split partials lie c_pad floats
  further apart than gm * gn (4-byte aligned C, odd split strides)."""
  import ranking_b200  # noqa: F401
  from ranking_b200 import _C
  g = torch.Generator().manual_seed(seed)
  A = torch.randn(gm, gk, generator=g)
  B = torch.randn(gk, gn, generator=g)
  bias = torch.randn(gn, generator=g)
  aux = torch.randn(gm, gn, generator=g)
  ref = A.double() @ B.double()
  scale = (A.double().abs() @ B.double().abs())
  if epi == 1:
    ref = ref + bias.double()
    if act == 1:
      ref = torch.relu(ref)
  elif epi in (2, 3) and act == 1:
    ref = torch.where(aux.double() > 0, ref, torch.zeros_like(ref))
  a_store = (A.t().contiguous() if a_mn else A.contiguous()).cuda()
  if passes == 3 and not split_b:
    b_hi = ((B.view(torch.int32) + 4096) & -8192).view(torch.float32)   # RN to TF32
    b_lo = B - b_hi
  else:
    b_hi, b_lo = B, None
  lay = (lambda t: t.contiguous()) if b_mn else (lambda t: t.t().contiguous())
  b_store = lay(b_hi).cuda()
  b_lo_store = None if b_lo is None else lay(b_lo).cuda()
  shape = (gn, gm) if transposed else (gm, gn)
  stride = gm * gn + c_pad if splits > 1 else 0
  buf = torch.full((c_pad + max(splits, 1) * (gm * gn + c_pad),), float('nan'), device='cuda')
  ldc = gm if transposed else gn
  bias_d, aux_d = bias.cuda(), aux.cuda()    # keep alive until the sync below
  bits_out = bits_in = None
  if want_bits:
    bits_out = torch.full(((gn + 31) // 32, gm), -1, dtype=torch.int32, device='cuda')
  if epi == 3:
    bits_in = _pack_bits(aux > 0).cuda()
  rc = _C.lib.tfr_tc_gemm(
      _C.ptr(a_store), a_store.shape[1], _C.ptr(b_store), b_store.shape[1],
      _C.ptr(b_lo_store), C_ptr(buf, c_pad), ldc, gm, gn, gk, a_mn, b_mn, passes, split_b,
      epi, _C.ptr(bias_d), _C.ptr(aux_d), act, transposed, splits, stride,
      _C.ptr(bits_out), _C.ptr(bits_in), _C.stream())
  _C.check(rc)
  torch.cuda.synchronize()
  C = torch.stack([buf[c_pad + z * stride:c_pad + z * stride + gm * gn].view(shape)
                   for z in range(splits)]) if splits > 1 else buf[c_pad:c_pad + gm * gn].view(shape)
  out = C.double().cpu()
  if want_bits:
    assert torch.equal(bits_out.cpu(), _pack_bits(C.cpu() > 0))
  if splits > 1:
    out = out.sum(0)
  if transposed:
    out = out.t()
  err = ((out - ref).abs() / (scale + 1e-30))
  return float(err.max()), out, ref


CASES = []
for a_mn, b_mn in itertools.product([0, 1], [0, 1]):
  for passes, split_b in [(1, 0), (3, 0), (3, 1)]:
    CASES.append((a_mn, b_mn, passes, split_b))


@pytest.mark.parametrize('a_mn,b_mn,passes,split_b', CASES)
@pytest.mark.parametrize('shape', [(128, 64, 32), (300, 136, 136), (256, 256, 264),
                                   (130, 16, 8)])
def test_tc_gemm_variants(a_mn, b_mn, passes, split_b, shape):
  gm, gn, gk = shape
  if a_mn:
    gm = (gm + 3) // 4 * 4    # MN-major storage needs a 16-byte aligned row pitch
  err, _, _ = run_gemm(gm, gn, gk, a_mn, b_mn, passes, split_b, seed=gm + gn)
  tol = 2e-6 if passes == 3 else 2e-3
  assert err <= tol, err


def test_tc_gemm_epilogues_and_splits():
  err, _, _ = run_gemm(384, 256, 136, 0, 1, 3, 0, epi=1, act=1)
  assert err <= 2e-6, err
  err, _, _ = run_gemm(384, 128, 64, 0, 0, 3, 0, epi=2, act=1)
  assert err <= 2e-6, err
  # ReLU sign bits written by the forward epilogue / consumed by the backward one
  for shape in [(384, 256, 136), (1000, 128, 256), (300, 136, 64), (200, 64, 128)]:
    err, _, _ = run_gemm(*shape, 0, 1, 3, 0, epi=1, act=1, want_bits=True)
    assert err <= 2e-6, (shape, err)
    err, _, _ = run_gemm(*shape, 0, 0, 3, 0, epi=3, act=1)
    assert err <= 2e-6, (shape, err)
    err, _, _ = run_gemm(*shape, 0, 0, 1, 0, epi=3, act=1)
    assert err <= 2e-3, (shape, err)
  # dW-shaped: both operands MN-major, long K split over CTAs, transposed store
  err, _, _ = run_gemm(256, 136, 4096, 1, 1, 3, 1, transposed=1, splits=4)
  assert err <= 2e-6, err
  err, _, _ = run_gemm(136, 256, 4096, 1, 1, 3, 1, splits=8)
  assert err <= 2e-6, err


def test_tc_gemm_unaligned_output():
  """C only 4-byte aligned, and split-K partials an odd number of floats apart: the paired
  stores of the epilogue must fall back to single ones."""
  err, _, _ = run_gemm(300, 136, 136, 0, 1, 3, 0, epi=1, act=1, c_pad=1)
  assert err <= 2e-6, err
  err, _, _ = run_gemm(256, 136, 2048, 1, 1, 3, 1, splits=3, c_pad=1)
  assert err <= 2e-6, err


@pytest.mark.parametrize('gm', [512, 600, 657, 1280])
@pytest.mark.parametrize('gn,gk', [(256, 136), (128, 256), (64, 128)])
def test_tc_gemm_cta_pairs_kmajor(gm, gn, gk):
  """Forward / dZ GEMM shapes (K-major pre-split weights, >= 4 row blocks): even and odd
  block counts (600 rows = 5 blocks), ragged last blocks (657), every epilogue (store,
  bias + ReLU + sign bits, mask from sign bits)."""
  for epi, act, bits in ((0, 0, False), (1, 1, True), (3, 1, False)):
    err, _, _ = run_gemm(gm, gn, gk, 0, 0, 3, 0, epi=epi, act=act, want_bits=bits, seed=gm + gn)
    assert err <= 2e-6, (gm, gn, gk, epi, err)


@pytest.mark.parametrize('shape', [(256, 136, 4096, 1, 4), (256, 128, 4096, 0, 8),
                                   (384, 136, 2048, 1, 3), (640, 64, 1536, 0, 5)])
def test_tc_gemm_cta_pairs_dw(shape):
  """dW GEMM shapes (MN-major operands split on the fly): 2, 3 and 5 row blocks, split-K
  partials, transposed and direct stores."""
  gm, gn, gk, transposed, splits = shape
  err, _, _ = run_gemm(gm, gn, gk, 1, 1, 3, 1, transposed=transposed, splits=splits, seed=gm)
  assert err <= 2e-6, (shape, err)


if __name__ == '__main__':
  # Diagnostic mode: print everything, never stop.
  import traceback
  for shape in [(128, 64, 32), (128, 256, 64), (300, 136, 136), (130, 16, 8)]:
    for a_mn, b_mn, passes, split_b in CASES:
      try:
        gm, gn, gk = shape
        if a_mn:
          gm = (gm + 3) // 4 * 4
        err, out, ref = run_gemm(gm, gn, gk, a_mn, b_mn, passes, split_b)
        msg = 'err %.3e' % err
        if not (err <= (2e-6 if passes == 3 else 2e-3)):
          d = (out - ref).abs()
          nan = int(torch.isnan(out).sum())
          rows_bad = (d.max(1).values > 1e-2).nonzero().flatten()[:12].tolist()
          cols_bad = (d.max(0).values > 1e-2).nonzero().flatten()[:12].tolist()
          msg += ' BAD nan=%d rows%s cols%s out00=%.4f ref00=%.4f' % (
              nan, rows_bad, cols_bad, float(out[0, 0]), float(ref[0, 0]))
        print('shape', shape, 'a_mn', a_mn, 'b_mn', b_mn, 'passes', passes,
              'split_b', split_b, msg, flush=True)
      except Exception as e:   # noqa: BLE001
        print('shape', shape, a_mn, b_mn, passes, split_b, 'EXC', repr(e)[:300],
              flush=True)
        traceback.print_exc()
        sys.exit(1)   # a CUDA fault poisons the context; stop here
