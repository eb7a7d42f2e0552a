"""GPU tests of the epilogue warpgroup's row loop (wgmma_gemm.cuh) on the lane mappings and
store paths it chooses per tile: whole rows per warp step on tiles with more than 64 live
columns, two rows per step on tiles with at most 64; mask words prefetched into registers,
including the rows past GM; sign words stored 8 rows at a time in the fast loop and row by row
in the general one; column sums added onto running sums loaded before the row pass.  GM is no
multiple of 8 (sign-word planes past the first start mid-sector) or a multiple of 8 but not of
128 (ragged last row block).  Every CTA runs several tiles, with one or two column tiles.  Each
case is compared bit for bit with the same GEMM run in row chunks small enough for one tile per
CTA, with a second identical call, and against fp64."""
import ctypes

import pytest
import torch

from test_tc_gemm_gpu import _pack_bits

pytestmark = pytest.mark.gpu

GMS = [33357, 33352]       # 33357: odd; 33352: a multiple of 8 whose last row block has 72 rows
GNS = [8, 60, 64, 128, 136, 200, 256]
GNS_BF16 = [8, 56, 64, 128, 136, 200, 256]   # bf16 C needs a row pitch of a multiple of 8
GK = 72                    # two full k blocks of TF32 and a half one
CHUNK = 32 * 128           # 32 row blocks x at most 2 column tiles: one tile per CTA


def _ptr(t, offset_elems=0):
  return None if t is None else ctypes.c_void_p(t.data_ptr() + t.element_size() * offset_elems)


class _Case:
  def __init__(self, gm, gn, bf16, seed):
    g = torch.Generator().manual_seed(seed)
    self.gm, self.gn, self.bf16 = gm, gn, bf16
    A = torch.randn(gm, GK, generator=g)
    B = torch.randn(gn, GK, generator=g)
    if bf16:
      A, B = A.bfloat16(), B.bfloat16()
    self.A, self.B = A, B
    self.bias = torch.randn(gn, generator=g)
    self.keep = torch.rand(gm, gn, generator=g) > 0.4
    self.out_dtype = torch.bfloat16 if bf16 else torch.float32
    self.a_d, self.bias_d = A.cuda(), self.bias.cuda()
    if bf16:
      self.b_d = B.cuda()
    else:
      b_hi = ((B.view(torch.int32) + 4096) & -8192).view(torch.float32)   # RN to TF32
      self.bhi_d, self.blo_d = b_hi.cuda(), (B - b_hi).cuda()
    self.keep_bits = _pack_bits(self.keep).cuda()

  def run(self, r0, rows, epi, want_colsum=False):
    """Rows [r0, r0 + rows): (C, sign words out or None, column-sum slots or None)."""
    from ranking_b200 import _C
    gn, nw = self.gn, (self.gn + 31) // 32
    C = torch.full((rows, gn), float('nan'), dtype=self.out_dtype, device='cuda')
    bits_out = torch.full((nw, rows), -1, dtype=torch.int32, device='cuda') if epi == 1 else None
    bits_in = self.keep_bits[:, r0:r0 + rows].contiguous() if epi == 3 else None
    colsum = (torch.full((8 * 256, (gn + 63) // 64 * 64), float('nan'), device='cuda')
              if want_colsum else None)
    nslots = ctypes.c_int(0)
    if self.bf16:
      _C.check(_C.lib.tfr_tc_gemm_bf16(
          _ptr(self.a_d, r0 * GK), GK, _ptr(self.b_d), GK, _ptr(C), gn, rows, gn, GK, 0, epi,
          _ptr(self.bias_d), 1, _ptr(bits_out), _ptr(bits_in), _ptr(colsum),
          0 if colsum is None else colsum.shape[1],
          ctypes.cast(ctypes.byref(nslots), ctypes.c_void_p), 1, 0, _C.stream()))
    else:
      assert colsum is None
      _C.check(_C.lib.tfr_tc_gemm(
          _ptr(self.a_d, r0 * GK), GK, _ptr(self.bhi_d), GK, _ptr(self.blo_d), _ptr(C), gn,
          rows, gn, GK, 0, 0, 3, 0, epi, _ptr(self.bias_d), None, 1, 0, 1, 0,
          _ptr(bits_out), _ptr(bits_in), _C.stream()))
    torch.cuda.synchronize()
    return C, bits_out, None if colsum is None else colsum[:nslots.value, :gn]


def _bits_eq(a, b):
  return torch.equal(a.view(torch.int32 if a.dtype == torch.float32 else torch.int16),
                     b.view(torch.int32 if b.dtype == torch.float32 else torch.int16))


def _check(case, epi, want_colsum=False):
  import ranking_b200  # noqa: F401
  C, bits, colsum = case.run(0, case.gm, epi, want_colsum)
  C2, bits2, colsum2 = case.run(0, case.gm, epi, want_colsum)
  assert _bits_eq(C, C2)
  if bits is not None:
    assert torch.equal(bits, bits2)
  if want_colsum:
    assert torch.equal(colsum, colsum2)
  for r0 in range(0, case.gm, CHUNK):
    rows = min(CHUNK, case.gm - r0)
    Cc, bc, _ = case.run(r0, rows, epi)
    assert _bits_eq(C[r0:r0 + rows], Cc), r0
    if bits is not None:
      assert torch.equal(bits[:, r0:r0 + rows], bc), r0
  ref = case.A.double() @ case.B.double().t()
  scale = case.A.double().abs() @ case.B.double().abs().t()
  if epi == 1:
    ref = torch.relu(ref + case.bias.double())
    assert torch.equal(bits.cpu(), _pack_bits(C.float().cpu() > 0))
  else:
    ref = torch.where(case.keep, ref, torch.zeros_like(ref))
  tol, ulp = (1e-5, 2.0 ** -8) if case.bf16 else (2e-6, 0.0)
  err = float(((C.double().cpu() - ref).abs() - ulp * ref.abs()).clamp(min=0).div(scale + 1e-30).max())
  assert err <= tol, err
  if want_colsum:
    cs = colsum.double().sum(0).cpu()
    cerr = float(((cs - ref.sum(0)).abs() / (scale.sum(0) + 1e-30)).max())
    assert cerr <= 1e-5, ('colsum', cerr)


@pytest.mark.parametrize('gm', GMS)
@pytest.mark.parametrize('gn', GNS)
def test_rows_tf32_bias_relu_sign_words(gm, gn):
  _check(_Case(gm, gn, False, seed=gm + gn), epi=1)


@pytest.mark.parametrize('gm', GMS)
@pytest.mark.parametrize('gn', GNS)
def test_rows_tf32_mask_from_sign_words(gm, gn):
  _check(_Case(gm, gn, False, seed=gm + gn + 1), epi=3)


@pytest.mark.parametrize('gm', GMS)
@pytest.mark.parametrize('gn', GNS_BF16)
def test_rows_bf16_bias_relu_sign_words(gm, gn):
  _check(_Case(gm, gn, True, seed=gm + gn + 2), epi=1)


# 520 columns: five column tiles, so a CTA's tiles change column tile (132 CTAs)
@pytest.mark.parametrize('gm', GMS)
@pytest.mark.parametrize('gn', GNS_BF16 + [520])
def test_rows_bf16_mask_and_column_sums(gm, gn):
  _check(_Case(gm, gn, True, seed=gm + gn + 3), epi=3, want_colsum=True)
