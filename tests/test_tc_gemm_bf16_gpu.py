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
SENTINEL = 7.0


def _pack_bits(keep):
  gm, gn = keep.shape
  nw = (gn + 31) // 32
  pad = torch.zeros(gm, nw * 32, dtype=torch.int64)
  pad[:, :gn] = keep.long()
  words = (pad.reshape(gm, nw, 32) << torch.arange(32)).sum(2)
  words = torch.where(words >= 2 ** 31, words - 2 ** 32, words)
  return words.t().contiguous().to(torch.int32)


def run_kmajor(gm, gn, gk, epi=0, act=0, want_bits=False, want_colsum=False, seed=0, lda=None,
               ldc=None):
  """mn = 0: C[gm, gn] (bf16, row pitch ldc) = A[gm, gk] (row pitch lda) B[gn, gk]^T.  The
  columns [gk, lda) of A hold values that must not be read, the columns [gn, ldc) of C a
  sentinel that must stay."""
  import ranking_b200  # noqa: F401
  from ranking_b200 import _C
  g = torch.Generator().manual_seed(seed)
  lda = lda or gk
  ldc = ldc or gn
  A_full = torch.randn(gm, lda, generator=g).bfloat16()
  A_full[:, gk:] = 1e4
  A = A_full[:, :gk]
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
  a_d, b_d, bias_d = A_full.cuda(), B.cuda(), bias.cuda()
  C = torch.full((gm, ldc), SENTINEL, dtype=torch.bfloat16, device='cuda')
  C[:, :gn] = float('nan')
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
      _C.ptr(a_d), lda, _C.ptr(b_d), gk, _C.ptr(C), ldc, gm, gn, gk, 0, epi, _C.ptr(bias_d),
      act, _C.ptr(bits_out), _C.ptr(bits_in), _C.ptr(colsum), stride,
      ctypes.cast(ctypes.byref(nslots), ctypes.c_void_p), 1, 0, _C.stream())
  _C.check(rc)
  torch.cuda.synchronize()
  assert (C[:, gn:].float() == SENTINEL).all(), 'columns past GN written'
  C = C[:, :gn]
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


def run_mnmajor(gm, gn, gk, splits, seed=0, lda=None, ldc=None):
  """mn = 1: C[gm, gn] (fp32, summed over the split partials; row pitch ldc) = A[gk, gm]^T
  (row pitch lda) B[gk, gn].  Columns [gm, lda) of A must not be read, columns [gn, ldc) of
  every partial keep their sentinel."""
  import ranking_b200  # noqa: F401
  from ranking_b200 import _C
  g = torch.Generator().manual_seed(seed)
  lda = lda or gm
  ldc = ldc or gn
  A_full = torch.randn(gk, lda, generator=g).bfloat16()
  A_full[:, gm:] = 1e4
  A = A_full[:, :gm]
  B = torch.randn(gk, gn, generator=g).bfloat16()
  ref = A.double().t() @ B.double()
  scale = A.double().abs().t() @ B.double().abs()
  a_d, b_d = A_full.cuda(), B.cuda()
  rows = (gm + 127) // 128 * 128
  C = torch.full((splits, rows, ldc), SENTINEL, device='cuda')
  C[:, :gm, :gn] = float('nan')
  rc = _C.lib.tfr_tc_gemm_bf16(
      _C.ptr(a_d), lda, _C.ptr(b_d), gn, _C.ptr(C), ldc, gm, gn, gk, 1, 0, None, 0, None, None,
      None, 0, None, splits, rows * ldc, _C.stream())
  _C.check(rc)
  torch.cuda.synchronize()
  assert (C[:, :, gn:] == SENTINEL).all(), 'columns past GN written'
  out = C[:, :gm, :gn].double().sum(0).cpu()
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


def dw_splits(sms, kin, nout, rows):
  """csrc/bert.cu dw_splits: the split count TFR-BERT's bf16 dW GEMMs launch."""
  tiles = ((kin + 127) // 128) * ((nout + 127) // 128)
  nkb = (rows + 63) // 64
  best, best_t = 1, 0.0
  for s in range(1, min(16, nkb) + 1):
    per = (nkb + s - 1) // s
    if (nkb + per - 1) // per != s:
      continue
    t = ((tiles * s + sms - 1) // sms) * per * 0.46e-6 + s * kin * nout * 8.0 / 3e12
    if s == 1 or t < best_t:
      best, best_t = s, t
  return best


# TFR-BERT's calls (csrc/bert.cu bgemm / dense_grad_bf16), (GM, GN, GK, lda, ldc, bias):
# the pooler on the [CLS] rows (GM = S, lda = L E), GN = 3E or I up to 4096, GK = I up to 4096.
BERT_KM = [(5, 768, 768, 64 * 768, 768, True),       # pooler, BERT-base
           (1, 1024, 1024, 512 * 1024, 1032, True),  # pooler, one sequence, ldc > GN
           (130, 600, 200, 200, 608, True),          # qkv at E 200
           (256, 2304, 768, 768, 2304, True),        # qkv, BERT-base
           (200, 3072, 768, 768, 3072, True),        # u = x' W1
           (136, 4096, 1024, 1024, 4104, False),     # u at I 4096, ldc > GN
           (70, 240, 1032, 1032, 240, True),         # y2 = a W2 at I 1032
           (256, 768, 3072, 3072, 768, True),        # y2, BERT-base
           (130, 1024, 4096, 4096, 1024, False)]     # d x' = du W1^T at I 4096
# dW (mn = 1), (GM = Kin, GN = Nout, GK = rows, lda, ldc, splits): the pooler's dW over S
# [CLS] rows (A strided by L E) and the dW of the layers, split as dw_splits picks.
BERT_MN = [(768, 768, gk, 64 * 768, 768, 1) for gk in (1, 2, 5, 63, 64, 65)] + [
    (64, 64, 5, 7 * 64, 72, 1),                        # ldc > GN
    (4096, 1024, 520, 4096, 1024, None),              # dW2 at I 4096 (Kin = 4096)
    (4096, 64, 1937, 4096, 64, None),
    (64, 192, 1937, 64, 200, None),                   # 16 splits, the last one block short
    (136, 408, 3000, 136, 408, None)]


def _bert_id(c):
  return 'x'.join(str(v) for v in c)


@pytest.mark.parametrize('shape', BERT_KM, ids=_bert_id)
def test_bf16_gemm_kmajor_bert_calls(shape):
  gm, gn, gk, lda, ldc, bias = shape
  err, _, _ = run_kmajor(gm, gn, gk, epi=1 if bias else 0, act=0, seed=gm + gn + gk, lda=lda,
                         ldc=ldc)
  print('[bf16 gemm bert mn=0 %s] err %.2e (bar 1e-5)' % (_bert_id(shape), err))
  assert err <= 1e-5, err


@pytest.mark.parametrize('shape', BERT_MN, ids=_bert_id)
def test_bf16_gemm_mnmajor_bert_calls(shape):
  gm, gn, gk, lda, ldc, splits = shape
  splits = splits or dw_splits(132, gm, gn, gk)
  err, _, _ = run_mnmajor(gm, gn, gk, splits, seed=gm + gn + gk, lda=lda, ldc=ldc)
  print('[bf16 gemm bert mn=1 %s] splits %d, err %.2e (bar 2e-6)' %
        (_bert_id(shape), splits, err))
  assert err <= 2e-6, err


def test_bert_dw_split_counts():
  """The dW shapes above reach dw_splits' 16 with a shorter last split, and more than one."""
  counts = {c[:3]: dw_splits(132, *c[:3]) for c in BERT_MN if c[5] is None}
  assert counts[(64, 192, 1937)] == 16
  nkb = (1937 + 63) // 64
  per = (nkb + 15) // 16
  assert nkb - 15 * per < per   # the last split is shorter
  assert any(1 < s < 16 for s in counts.values()), counts


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
