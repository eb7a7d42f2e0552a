"""The folded remainder of the TF32 GEMM engine's dW kernels (A and B MN-major,
wgmma_gemm.cuh): when GN is 128 q + r with r in 1..8, the last 128-column tile owns the r
columns past it (B stage rows 128..135, m64n136 wgmma) instead of a column tile of its own.

Each output element must see the same k blocks, k order and hi.hi, lo.hi, hi.lo sequence as
before, so the folded GEMM is compared bit for bit with the same GEMM run as two calls: columns
[0, GN - r), which fold nothing, and the narrow tile [GN - r, GN), which runs the unfolded
arithmetic.  The K-major-B layout (b_mn = 0) does not fold and must agree the same way.  Also
checked against fp64, at GN = 137 (r = 9, not folded), and for repeatability."""
import ctypes
import functools

import pytest
import torch

from test_tc_gemm_gpu import CASES

MN_CASES = [c for c in CASES if c[0] == 1]   # (a_mn, b_mn, passes, split_b)


@functools.lru_cache(maxsize=None)
def _lib():
  import __graft_entry__ as g
  g.build()
  from ranking_b200 import _C
  return _C


def _tol(passes):
  return 2e-6 if passes == 3 else 2e-3


def _ld(n):
  return (n + 3) // 4 * 4   # leading dimensions are multiples of 4 floats


class _Gemm:
  """A [GK, GM] (MN-major), B [GK, GN] (b_mn) or [GN, GK] with padded leading dimensions; B
  pre-split into hi / lo for 3xTF32 without split_b.  C holds `splits` slices of
  gm * gn + c_pad floats, starting c_pad floats into its buffer."""

  def __init__(self, gm, gn, gk, b_mn, passes, split_b, transposed, splits, c_pad, seed):
    g = torch.Generator().manual_seed(seed)
    self.gm, self.gn, self.gk = gm, gn, gk
    self.b_mn, self.passes, self.split_b = b_mn, passes, split_b
    self.transposed, self.splits, self.c_pad = transposed, splits, c_pad
    self.A = torch.randn(gk, gm, generator=g)
    self.B = torch.randn(gk, gn, generator=g)
    if passes == 3 and not split_b:
      hi = ((self.B.view(torch.int32) + 4096) & -8192).view(torch.float32)   # RN to TF32
      parts = [hi, self.B - hi]
    else:
      parts = [self.B]
    self.a_d = self.A.cuda()
    self.b_d = []
    for p in parts:
      if b_mn:
        self.ldb = _ld(gn)
        s = torch.zeros(gk, self.ldb)
        s[:, :gn] = p
      else:
        self.ldb = _ld(gk)
        s = torch.zeros(gn, self.ldb)
        s[:, :gk] = p.t()
      self.b_d.append(s.cuda())
    self.ldc = gm if transposed else gn
    self.stride = gm * gn + c_pad if splits > 1 else 0

  def new_c(self):
    return torch.full((self.c_pad + self.splits * (self.gm * self.gn + self.c_pad),),
                      float('nan'), device='cuda')

  def run(self, C, c0=0, nc=None):
    """Columns [c0, c0 + nc) of the product into C (operands and output offset by c0)."""
    _C = _lib()
    nc = self.gn - c0 if nc is None else nc
    boff = c0 if self.b_mn else c0 * self.ldb
    coff = self.c_pad + (c0 * self.ldc if self.transposed else c0)
    ptr = lambda t, off: ctypes.c_void_p(t.data_ptr() + 4 * off)   # noqa: E731
    b_lo = ptr(self.b_d[1], boff) if len(self.b_d) > 1 else None
    _C.check(_C.lib.tfr_tc_gemm(
        _C.ptr(self.a_d), self.gm, ptr(self.b_d[0], boff), self.ldb, b_lo, ptr(C, coff),
        self.ldc, self.gm, nc, self.gk, 1, self.b_mn, self.passes, self.split_b, 0, None, None, 0,
        self.transposed, self.splits, self.stride, None, None, _C.stream()))

  def result(self, C):
    """The product summed over the split-K slices, [GM, GN] in fp64."""
    shape = (self.gn, self.gm) if self.transposed else (self.gm, self.gn)
    n = self.gm * self.gn
    out = sum(C[self.c_pad + z * self.stride:self.c_pad + z * self.stride + n].view(shape)
              .double().cpu() for z in range(self.splits))
    return out.t() if self.transposed else out

  def err(self, C):
    ref = self.A.double().t() @ self.B.double()
    scale = self.A.double().abs().t() @ self.B.double().abs()
    return float(((self.result(C) - ref).abs() / (scale + 1e-30)).max())


# (gm, gk, splits, c_pad): one split; 9 k blocks over 4 splits (3, 3, 3 and an empty one) with
# C 4-byte aligned and an odd split stride; 10 blocks with a ragged last one over 4 splits (a
# short last split); 400 blocks over 200 splits, so every CTA chains several folded tiles.
SPLITS = [(200, 96, 1, 0), (256, 288, 4, 1), (256, 300, 4, 0), (256, 12800, 200, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize('a_mn,b_mn,passes,split_b', MN_CASES)
@pytest.mark.parametrize('transposed', [0, 1])
@pytest.mark.parametrize('gn', [129, 132, 136, 264])
@pytest.mark.parametrize('gm,gk,splits,c_pad', SPLITS)
def test_folded_tail_bit_exact(a_mn, b_mn, passes, split_b, transposed, gn, gm, gk, splits,
                               c_pad):
  """Folded GEMM == columns [0, GN - r) and [GN - r, GN) as two calls, bit for bit; two
  identical calls give identical bits; and the result is within the fp64 tolerance."""
  e = _Gemm(gm, gn, gk, b_mn, passes, split_b, transposed, splits, c_pad, seed=gn + gk)
  r = gn % 128
  folded, again, parts = e.new_c(), e.new_c(), e.new_c()
  e.run(folded)
  e.run(again)
  e.run(parts, 0, gn - r)
  e.run(parts, gn - r, r)
  torch.cuda.synchronize()
  assert torch.equal(folded.view(torch.int32), again.view(torch.int32))
  assert torch.equal(folded.view(torch.int32), parts.view(torch.int32)), float(
      (e.result(folded) - e.result(parts)).abs().max())
  assert e.err(folded) <= _tol(passes)


@pytest.mark.gpu
@pytest.mark.parametrize('a_mn,b_mn,passes,split_b', MN_CASES)
@pytest.mark.parametrize('transposed', [0, 1])
@pytest.mark.parametrize('gn', [129, 136, 137, 264])
@pytest.mark.parametrize('gk,splits', [(180, 1), (1000, 3)])
def test_folded_tail_against_fp64(a_mn, b_mn, passes, split_b, transposed, gn, gk, splits):
  """Ragged k (a 20-wide and an 8-wide last block) and GN = 137, the first width whose
  remainder (9 columns) keeps a column tile of its own."""
  e = _Gemm(300, gn, gk, b_mn, passes, split_b, transposed, splits, 0, seed=gn * gk)
  C = e.new_c()
  e.run(C)
  torch.cuda.synchronize()
  assert e.err(C) <= _tol(passes)


def test_mn_major_pair_takes_plain_store_only():
  """With A and B both MN-major (the dW layout) only the plain store epilogue without column
  sums is accepted: the folded remainder columns have no other epilogue.  No GPU needed."""
  _C = _lib()
  p = ctypes.c_void_p(256)    # never dereferenced: validation fails first
  for epi in (1, 2, 3):
    rc = _C.lib.tfr_tc_gemm(p, 256, p, 136, None, p, 136, 256, 136, 64, 1, 1, 3, 1, epi, p, p,
                            1, 0, 1, 0, None, p, None)
    assert rc == 1, _C.last_error()
