"""GPU tests of the wgmma bf16 GEMM engine (csrc/tc_gemm_bf16.cu) through the C ABI,
against a torch fp64 matmul of the SAME bf16-rounded inputs (so only the fp32
accumulation order and the bf16 rounding of the output differ).

Tolerance: bf16 outputs (mn = 0): |err| <= 2^-8 |ref| + 1e-5 |A||B| (one bf16 rounding of
the result + fp32 accumulation); fp32 partial outputs (mn = 1): <= 2e-6 |A||B|.
Run as a script for a diagnostic table that keeps going after failures.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import pytest
import torch

pytestmark = pytest.mark.gpu


def _pack_bits(keep):
  gm, gn = keep.shape
  nw = (gn + 31) // 32
  pad = torch.zeros(gm, nw * 32, dtype=torch.int64)
  pad[:, :gn] = keep.long()
  words = (pad.reshape(gm, nw, 32) << torch.arange(32)).sum(2)
  words = torch.where(words >= 2 ** 31, words - 2 ** 32, words)
  return words.t().contiguous().to(torch.int32)


def run_kmajor(gm, gn, gk, epi=0, act=0, want_bits=False, want_colsum=False, seed=0):
  """mn = 0: C[gm, gn] (bf16) = A[gm, gk] B[gn, gk]^T."""
  import ranking_b200  # noqa: F401
  from ranking_b200 import _C
  g = torch.Generator().manual_seed(seed)
  A = torch.randn(gm, gk, generator=g).bfloat16()
  B = torch.randn(gn, gk, generator=g).bfloat16()
  bias = torch.randn(gn, generator=g)
  keep = torch.rand(gm, gn, generator=g) > 0.4
  ref = A.double() @ B.double().t()
  scale = A.double().abs() @ B.double().abs().t()
  if epi == 1:
    ref = ref + bias.double()
    if act == 1:
      ref = torch.relu(ref)
  elif epi == 3:
    ref = torch.where(keep, ref, torch.zeros_like(ref))
  a_d, b_d, bias_d = A.cuda(), B.cuda(), bias.cuda()
  C = torch.full((gm, gn), float('nan'), dtype=torch.bfloat16, device='cuda')
  bits_out = bits_in = colsum = None
  slots = (torch.zeros(1, dtype=torch.int32))
  import ctypes
  nslots = ctypes.c_int(0)
  if want_bits:
    bits_out = torch.full(((gn + 31) // 32, gm), -1, dtype=torch.int32, device='cuda')
  if epi == 3:
    bits_in = _pack_bits(keep).cuda()
  stride = (gn + 63) // 64 * 64
  if want_colsum:
    colsum = torch.full((148 * 8, stride), float('nan'), device='cuda')
  rc = _C.lib.tfr_tc_gemm_bf16(
      _C.ptr(a_d), gk, _C.ptr(b_d), gk, _C.ptr(C), gn, gm, gn, gk, 0, epi, _C.ptr(bias_d),
      act, _C.ptr(bits_out), _C.ptr(bits_in), _C.ptr(colsum), stride,
      ctypes.cast(ctypes.byref(nslots), ctypes.c_void_p), 1, 0, _C.stream())
  _C.check(rc)
  torch.cuda.synchronize()
  out = C.double().cpu()
  err = float(((out - ref).abs() - 2.0 ** -8 * ref.abs()).clamp(min=0).div(scale + 1e-30).max())
  if want_bits:
    assert torch.equal(bits_out.cpu(), _pack_bits(C.float().cpu() > 0))
  if want_colsum:
    cs = colsum[:nslots.value, :gn].double().sum(0).cpu()
    cref = ref.sum(0)
    cscale = scale.sum(0)
    cerr = float(((cs - cref).abs() / (cscale + 1e-30)).max())
    assert cerr <= 1e-5, ('colsum', cerr)
  return err, out, ref


def run_mnmajor(gm, gn, gk, splits, seed=0):
  """mn = 1: C[gm, gn] (fp32, summed over the split partials) = A[gk, gm]^T B[gk, gn]."""
  import ranking_b200  # noqa: F401
  from ranking_b200 import _C
  g = torch.Generator().manual_seed(seed)
  A = torch.randn(gk, gm, generator=g).bfloat16()
  B = torch.randn(gk, gn, generator=g).bfloat16()
  ref = A.double().t() @ B.double()
  scale = A.double().abs().t() @ B.double().abs()
  a_d, b_d = A.cuda(), B.cuda()
  rows = (gm + 127) // 128 * 128
  C = torch.full((splits, rows, gn), float('nan'), device='cuda')
  rc = _C.lib.tfr_tc_gemm_bf16(
      _C.ptr(a_d), gm, _C.ptr(b_d), gn, _C.ptr(C), gn, gm, gn, gk, 1, 0, None, 0, None, None,
      None, 0, None, splits, rows * gn, _C.stream())
  _C.check(rc)
  torch.cuda.synchronize()
  out = C[:, :gm].double().sum(0).cpu()
  err = float(((out - ref).abs() / (scale + 1e-30)).max())
  return err, out, ref


KM_SHAPES = [(128, 64, 64), (300, 136, 136), (1000, 256, 256), (130, 16, 8), (257, 272, 40),
             (4096, 128, 256), (512, 64, 128)]
MN_SHAPES = [(136, 256, 5000, 7), (256, 256, 4096, 4), (64, 64, 1000, 3), (128, 64, 777 * 8, 5),
             (256, 128, 20000, 148), (384, 144, 3000, 2), (8, 8, 64, 1)]


@pytest.mark.parametrize('shape', KM_SHAPES)
def test_bf16_gemm_kmajor(shape):
  err, _, _ = run_kmajor(*shape, seed=sum(shape))
  assert err <= 1e-5, err


@pytest.mark.parametrize('shape', KM_SHAPES)
def test_bf16_gemm_kmajor_epilogues(shape):
  err, _, _ = run_kmajor(*shape, epi=1, act=1, want_bits=True, seed=1 + sum(shape))
  assert err <= 1e-5, err
  err, _, _ = run_kmajor(*shape, epi=1, act=0, seed=2 + sum(shape))
  assert err <= 1e-5, err
  err, _, _ = run_kmajor(*shape, epi=3, act=1, want_colsum=True, seed=3 + sum(shape))
  assert err <= 1e-5, err


@pytest.mark.parametrize('shape', MN_SHAPES)
def test_bf16_gemm_mnmajor(shape):
  err, _, _ = run_mnmajor(*shape, seed=sum(shape))
  assert err <= 2e-6, err


if __name__ == '__main__':
  import traceback

  def report(tag, shape, fn):
    try:
      err, out, ref = fn()
      msg = 'err %.3e' % err
      if not err <= 1e-5:
        d = (out - ref).abs()
        nan = int(torch.isnan(out).sum())
        rows_bad = (d.max(1).values > 1e-1).nonzero().flatten()[:10].tolist()
        cols_bad = (d.max(0).values > 1e-1).nonzero().flatten()[:10].tolist()
        msg += ' BAD nan=%d rows%s cols%s out00=%.4f ref00=%.4f' % (
            nan, rows_bad, cols_bad, float(out[0, 0]), float(ref[0, 0]))
      print(tag, shape, msg, flush=True)
    except AssertionError as e:
      print(tag, shape, 'ASSERT', repr(e)[:200], flush=True)
    except Exception as e:   # noqa: BLE001
      print(tag, shape, 'EXC', repr(e)[:300], flush=True)
      traceback.print_exc()
      sys.exit(1)   # a CUDA fault poisons the context

  for shape in KM_SHAPES:
    report('kmajor store', shape, lambda: run_kmajor(*shape))
    report('kmajor bias+relu+bits', shape,
           lambda: run_kmajor(*shape, epi=1, act=1, want_bits=True))
    report('kmajor mask+colsum', shape,
           lambda: run_kmajor(*shape, epi=3, act=1, want_colsum=True))
  for shape in MN_SHAPES:
    report('mnmajor', shape, lambda: run_mnmajor(*shape))
