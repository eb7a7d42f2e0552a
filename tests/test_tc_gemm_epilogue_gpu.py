"""GPU tests of the staged epilogue of the GEMM engine (wgmma_gemm.cuh).  For a K-major A the
MMA warpgroups hand each tile's accumulators to an epilogue warpgroup through a staging tile in
shared memory and go on with the next tile.  These shapes give every CTA several tiles, so the
staging tile is reused while the next k loop runs, with ragged GM and GN.  Each epilogue kind is
compared bit for bit with the same GEMM run in row chunks small enough for one tile per CTA
(where no staging tile is ever reused), against fp64, and with a second identical call."""
import ctypes

import pytest
import torch

from test_tc_gemm_gpu import _pack_bits

pytestmark = pytest.mark.gpu

GM = 33357                 # 261 row blocks, the last of 77 rows (no multiple of 16)
CHUNK = 32 * 128           # 32 row blocks x at most 2 column tiles: one tile per CTA
GNS = [136, 8, 64, 200]
GK = 96


def _ptr(t, offset_elems=0):
  return None if t is None else ctypes.c_void_p(t.data_ptr() + t.element_size() * offset_elems)


def _inputs(gn, bf16, seed):
  g = torch.Generator().manual_seed(seed)
  A = torch.randn(GM, GK, generator=g)
  B = torch.randn(gn, GK, generator=g)
  if bf16:
    A, B = A.bfloat16(), B.bfloat16()
  bias = torch.randn(gn, generator=g)
  keep = torch.rand(GM, gn, generator=g) > 0.4
  return A, B, bias, keep


def _reference(A, B, bias, keep, epi):
  ref = A.double() @ B.double().t()
  scale = A.double().abs() @ B.double().abs().t()
  if epi == 1:
    ref = torch.relu(ref + bias.double())
  elif epi == 3:
    ref = torch.where(keep, ref, torch.zeros_like(ref))
  return ref, scale


class _Tf32:
  """3xTF32, both operands K-major, B pre-split: the forward / dZ GEMMs of the tower."""
  out_dtype = torch.float32

  def __init__(self, gn, seed):
    self.gn = gn
    self.A, B, self.bias, self.keep = _inputs(gn, False, seed)
    self.B = B
    b_hi = ((B.view(torch.int32) + 4096) & -8192).view(torch.float32)   # RN to TF32
    self.a_d, self.bhi_d, self.blo_d = self.A.cuda(), b_hi.cuda(), (B - b_hi).cuda()
    self.bias_d = self.bias.cuda()

  def run(self, r0, rows, epi, C, bits_out, bits_in, colsum=None):
    from ranking_b200 import _C
    assert colsum is None
    _C.check(_C.lib.tfr_tc_gemm(
        _ptr(self.a_d, r0 * GK), GK, _ptr(self.bhi_d), GK, _ptr(self.blo_d), _ptr(C), self.gn,
        rows, self.gn, GK, 0, 0, 3, 0, epi, _ptr(self.bias_d), None, 1, 0, 1, 0,
        _ptr(bits_out), _ptr(bits_in), _C.stream()))
    return 0


class _Bf16:
  """bf16 operands and output, K-major: the same epilogue with packed stores and column sums."""
  out_dtype = torch.bfloat16

  def __init__(self, gn, seed):
    self.gn = gn
    self.A, self.B, self.bias, self.keep = _inputs(gn, True, seed)
    self.a_d, self.b_d, self.bias_d = self.A.cuda(), self.B.cuda(), self.bias.cuda()

  def run(self, r0, rows, epi, C, bits_out, bits_in, colsum=None):
    from ranking_b200 import _C
    nslots = ctypes.c_int(0)
    _C.check(_C.lib.tfr_tc_gemm_bf16(
        _ptr(self.a_d, r0 * GK), GK, _ptr(self.b_d), GK, _ptr(C), self.gn, rows, self.gn, GK, 0,
        epi, _ptr(self.bias_d), 1, _ptr(bits_out), _ptr(bits_in), _ptr(colsum),
        0 if colsum is None else colsum.shape[1],
        ctypes.cast(ctypes.byref(nslots), ctypes.c_void_p), 1, 0, _C.stream()))
    return nslots.value


def _call(eng, r0, rows, epi, want_bits, keep_bits, want_colsum=False):
  """Runs rows [r0, r0 + rows) and returns (C, sign words out, column-sum slots)."""
  gn, nw = eng.gn, (eng.gn + 31) // 32
  C = torch.full((rows, gn), float('nan'), dtype=eng.out_dtype, device='cuda')
  bits_out = (torch.full((nw, rows), -1, dtype=torch.int32, device='cuda') if want_bits else None)
  bits_in = keep_bits[:, r0:r0 + rows].contiguous() if epi == 3 else None
  colsum = (torch.full((8 * 256, (gn + 63) // 64 * 64), float('nan'), device='cuda')
            if want_colsum else None)
  nslots = eng.run(r0, rows, epi, C, bits_out, bits_in, colsum)
  torch.cuda.synchronize()
  return C, bits_out, None if colsum is None else colsum[:nslots, :gn]


def _check(eng, epi, want_bits=False, want_colsum=False, tol=2e-6, bf16_ulp=0.0):
  import ranking_b200  # noqa: F401
  keep_bits = _pack_bits(eng.keep).cuda()
  C, bits, colsum = _call(eng, 0, GM, epi, want_bits, keep_bits, want_colsum)
  # a second identical call: same bits
  C2, bits2, colsum2 = _call(eng, 0, GM, epi, want_bits, keep_bits, want_colsum)
  assert torch.equal(C.view(torch.int32 if C.dtype == torch.float32 else torch.int16),
                     C2.view(torch.int32 if C.dtype == torch.float32 else torch.int16))
  # one tile per CTA, chunk by chunk
  for r0 in range(0, GM, CHUNK):
    rows = min(CHUNK, GM - r0)
    Cc, bc, _ = _call(eng, r0, rows, epi, want_bits, keep_bits)
    assert torch.equal(C[r0:r0 + rows], Cc), (r0, float((C[r0:r0 + rows] - Cc).abs().max()))
    if want_bits:
      assert torch.equal(bits[:, r0:r0 + rows], bc), r0
  if want_bits:
    assert torch.equal(bits, bits2)
    assert torch.equal(bits.cpu(), _pack_bits(C.float().cpu() > 0))
  ref, scale = _reference(eng.A, eng.B, eng.bias, eng.keep, epi)
  out = C.double().cpu()
  err = float(((out - ref).abs() - bf16_ulp * ref.abs()).clamp(min=0).div(scale + 1e-30).max())
  assert err <= tol, err
  if want_colsum:
    assert torch.equal(colsum, colsum2)
    cs = colsum.double().sum(0).cpu()
    cerr = float(((cs - ref.sum(0)).abs() / (scale.sum(0) + 1e-30)).max())
    assert cerr <= 1e-5, ('colsum', cerr)


@pytest.mark.parametrize('gn', GNS)
def test_staged_store(gn):
  _check(_Tf32(gn, seed=gn), epi=0)


@pytest.mark.parametrize('gn', GNS)
def test_staged_bias_relu_sign_words(gn):
  _check(_Tf32(gn, seed=gn + 1), epi=1, want_bits=True)


@pytest.mark.parametrize('gn', GNS)
def test_staged_mask_from_sign_words(gn):
  _check(_Tf32(gn, seed=gn + 2), epi=3)


@pytest.mark.parametrize('gn', GNS)
def test_staged_bf16_bias_relu_sign_words(gn):
  _check(_Bf16(gn, seed=gn + 3), epi=1, want_bits=True, tol=1e-5, bf16_ulp=2.0 ** -8)


@pytest.mark.parametrize('gn', GNS)
def test_staged_bf16_mask_and_column_sums(gn):
  _check(_Bf16(gn, seed=gn + 4), epi=3, want_colsum=True, tol=1e-5, bf16_ulp=2.0 ** -8)
