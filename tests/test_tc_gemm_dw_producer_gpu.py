"""The dW kernels' producer warpgroup (wgmma_gemm.cuh, producer_ring): A and B MN-major, TF32.
The producer copies each k block's raw MN-major B slab into the stage by cp.async, transposes it
in place into the swizzled K-major tile (split into hi / lo for 3xTF32) and hands the stage to
the MMA warpgroups on an mbarrier ring that runs on across tiles.

The reference is the same GEMM with B given K-major (b_mn = 0, Bᵀ made by torch), whose B is
copied into the K-major tile and split there: every k block, k order, skipped zero k step and
hi.hi, lo.hi, hi.lo order is the same, so the two must agree bit for bit.  (GN past 128 with a
remainder of 1..8 columns folds it on the MN-major side only; the fold runs the same sums.)
Each case is also checked against fp64 at the engine's tolerances."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _tol(passes):
  return 2e-6 if passes == 3 else 2e-3


def _gemm(A, B, gm, gn, gk, b_mn, passes, split_b, transposed, splits):
  """C = A^T B (A [gk, gm]); B is [gk, gn] when b_mn else [gn, gk].  Returns [splits, ...]."""
  from ranking_b200 import _C

  def padded(t):   # leading dimensions are multiples of 4 floats
    out = torch.zeros(t.shape[0], (t.shape[1] + 3) // 4 * 4, device=t.device)
    out[:, :t.shape[1]] = t
    return out
  if passes == 3 and not split_b:
    hi = ((B.view(torch.int32) + 4096) & -8192).view(torch.float32)   # RN to TF32
    b, b_lo = padded(hi), padded(B - hi)
  else:
    b, b_lo = padded(B), None
  shape = (gn, gm) if transposed else (gm, gn)
  C = torch.full((splits,) + shape, float('nan'), device='cuda')
  _C.check(_C.lib.tfr_tc_gemm(
      _C.ptr(A), gm, _C.ptr(b), b.shape[1], _C.ptr(b_lo), _C.ptr(C), gm if transposed else gn,
      gm, gn, gk, 1, b_mn, passes, split_b, 0, None, None, 0, transposed, splits,
      C[0].numel() if splits > 1 else 0, None, None, _C.stream()))
  torch.cuda.synchronize()
  return C


def _check(gm, gn, gk, splits, passes=3, split_b=1, transposed=0, seed=0):
  import ranking_b200  # noqa: F401
  g = torch.Generator().manual_seed(seed)
  A = torch.randn(gk, gm, generator=g)
  B = torch.randn(gk, gn, generator=g)
  Ad, Bd = A.cuda(), B.cuda()
  mn = _gemm(Ad, Bd, gm, gn, gk, 1, passes, split_b, transposed, splits)
  again = _gemm(Ad, Bd, gm, gn, gk, 1, passes, split_b, transposed, splits)
  km = _gemm(Ad, Bd.t().contiguous(), gm, gn, gk, 0, passes, split_b, transposed, splits)
  assert torch.equal(mn.view(torch.int32), again.view(torch.int32))
  assert torch.equal(mn.view(torch.int32), km.view(torch.int32)), float(
      (mn - km).abs().nan_to_num(float('inf')).max())
  out = mn.double().sum(0).cpu()
  if transposed:
    out = out.t()
  ref = A.double().t() @ B.double()
  scale = A.double().abs().t() @ B.double().abs()
  assert float(((out - ref).abs() / (scale + 1e-30)).max()) <= _tol(passes)
  return mn


VARIANTS = [(3, 1), (3, 0), (1, 0)]   # (passes, split_b): on-the-fly split, pre-split, TF32


@pytest.mark.parametrize('passes,split_b', VARIANTS)
@pytest.mark.parametrize('transposed', [0, 1])
def test_more_tiles_per_cta_than_stages(passes, split_b, transposed):
  """1,000 row blocks of 2-block slices over at most 132 CTAs: every CTA chains 7 or more
  tiles, so its ring wraps many times inside and across tiles."""
  _check(128000, 136, 64, 1, passes, split_b, transposed, seed=1)


@pytest.mark.parametrize('passes,split_b', VARIANTS)
@pytest.mark.parametrize('gk', [1, 7, 31, 33, 95])
def test_k_tail_short_of_a_block(passes, split_b, gk):
  """A last k block of 1..31 rows: zero-filled slab rows and skipped k steps."""
  _check(256, 136, gk, 1, passes, split_b, seed=gk)


@pytest.mark.parametrize('passes,split_b', VARIANTS)
@pytest.mark.parametrize('gk,splits', [(288, 4), (96, 5), (64, 8)])
def test_empty_trailing_slices(passes, split_b, gk, splits):
  """9 blocks over 4 splits (an empty fourth), 3 over 5 and 2 over 8: trailing slices own no
  k block, so their tiles send nothing through the ring, and hold zeros."""
  C = _check(256, 136, gk, splits, passes, split_b, seed=gk + splits)
  per = ((gk + 31) // 32 + splits - 1) // splits
  for z in range(splits):
    if z * per * 32 >= gk:
      assert torch.equal(C[z], torch.zeros_like(C[z])), z


@pytest.mark.parametrize('passes,split_b', VARIANTS)
@pytest.mark.parametrize('gn', [129, 133, 136, 264, 64, 37, 3, 168, 192])
@pytest.mark.parametrize('transposed', [0, 1])
def test_widths(passes, split_b, gn, transposed):
  """GN = 128 q + r with r in 1..8 (folded remainder); GN <= 64 (m64n64); and a wide tile
  followed by an m64n64 one of 40 or 64 columns."""
  _check(200, gn, 1000, 3, passes, split_b, transposed, seed=gn)


def test_dw_shapes_of_the_tower():
  """The config-2 tower's dW GEMMs at a reduced M, with the trainer's split-K layout."""
  for gm, gn, transposed in [(256, 136, 1), (256, 128, 0), (128, 64, 0)]:
    _check(gm, gn, 20800, 25, 3, 1, transposed, seed=gm + gn)
