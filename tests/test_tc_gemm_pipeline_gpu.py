"""GPU tests of the GEMM engine's k-block pipeline (wgmma_gemm.cuh): one wgmma group stays in
flight across k blocks, and the cp.async ring runs stages - 2 blocks ahead.  These shapes walk
every prologue and drain depth of the ring, chain several tiles per CTA, split K into short and
empty slices, and reach the three-stage ring of a 3xTF32 column sum over 1024 columns.  The
split-K property test pins that the pipeline schedule changes no sum: every split-K slice is
bit for bit the unsplit GEMM over the same k range."""
import ctypes

import pytest
import torch

from test_tc_gemm_bf16_gpu import run_kmajor, run_mnmajor
from test_tc_gemm_gpu import CASES, run_gemm

pytestmark = pytest.mark.gpu

# TF32 k blocks are 32 wide: 1 .. 6 full blocks, then 5 blocks and a 20-wide tail (3 k steps)
TF32_GK = [32, 64, 96, 128, 160, 192, 180]
# bf16 k blocks are 64 wide: 1 .. 6 full blocks, then 5 blocks and a 24-wide tail (2 k steps)
BF16_GK = [64, 128, 192, 256, 320, 384, 344]


def _tol(passes):
  return 2e-6 if passes == 3 else 2e-3


@pytest.mark.parametrize('a_mn,b_mn,passes,split_b', CASES)
@pytest.mark.parametrize('gk', TF32_GK)
def test_tc_gemm_k_blocks_per_tile(a_mn, b_mn, passes, split_b, gk):
  """136 columns: one 128-wide and one 8-wide tile per row block."""
  err, _, _ = run_gemm(256, 136, gk, a_mn, b_mn, passes, split_b, seed=gk)
  assert err <= _tol(passes), err


@pytest.mark.parametrize('a_mn,b_mn,passes,split_b', CASES)
@pytest.mark.parametrize('gk', [96, 180])
def test_tc_gemm_tiles_chained_per_cta(a_mn, b_mn, passes, split_b, gk):
  """260 row blocks x 2 column tiles: every CTA runs several tiles back to back."""
  err, _, _ = run_gemm(33280, 136, gk, a_mn, b_mn, passes, split_b, seed=gk + 1)
  assert err <= _tol(passes), err


@pytest.mark.parametrize('a_mn,b_mn,passes,split_b', CASES)
@pytest.mark.parametrize('gk,splits', [(288, 4), (320, 4), (300, 4), (160, 2)])
def test_tc_gemm_short_and_empty_splits(a_mn, b_mn, passes, split_b, gk, splits):
  """9 k blocks over 4 splits: 3, 3, 3 and an empty fourth; 10 (and 9 with a tail): a last
  split of one block; 5 over 2: 3 and 2."""
  err, _, _ = run_gemm(256, 136, gk, a_mn, b_mn, passes, split_b, splits=splits, seed=gk)
  assert err <= _tol(passes), err


def _tf32_gemm(A, B, C, gm, gn, gk, passes, transposed, k0=0):
  """dW layout: A [GK, GM] and B [GK, GN] MN-major, split on the fly, from row k0 on."""
  from ranking_b200 import _C
  a = ctypes.c_void_p(A.data_ptr() + 4 * k0 * gm)
  b = ctypes.c_void_p(B.data_ptr() + 4 * k0 * gn)
  _C.check(_C.lib.tfr_tc_gemm(
      a, gm, b, gn, None, _C.ptr(C), gm if transposed else gn, gm, gn, gk, 1, 1, passes, 1,
      0, None, None, 0, transposed, C.shape[0], C[0].numel() if C.shape[0] > 1 else 0,
      None, None, _C.stream()))


@pytest.mark.parametrize('passes', [1, 3])
@pytest.mark.parametrize('transposed', [0, 1])
@pytest.mark.parametrize('gk,splits', [(428, 4), (288, 4), (2048, 5)])
def test_tc_gemm_split_slices_bit_exact(passes, transposed, gk, splits):
  """Each split-K slice of a dW-shaped GEMM equals, bit for bit, one unsplit GEMM over the
  same k range (operand pointers offset by k0 rows); an empty slice holds zeros."""
  import ranking_b200  # noqa: F401
  gm, gn, bk = 256, 136, 32
  g = torch.Generator().manual_seed(gk + splits)
  A = torch.randn(gk, gm, generator=g).cuda()
  B = torch.randn(gk, gn, generator=g).cuda()
  shape = (gn, gm) if transposed else (gm, gn)
  parts = torch.full((splits,) + shape, float('nan'), device='cuda')
  _tf32_gemm(A, B, parts, gm, gn, gk, passes, transposed)
  nkb = (gk + bk - 1) // bk
  per = (nkb + splits - 1) // splits
  for z in range(splits):
    k0 = z * per * bk
    klen = min(gk, k0 + per * bk) - k0
    if klen <= 0:
      assert torch.equal(parts[z], torch.zeros_like(parts[z])), z
      continue
    one = torch.full((1,) + shape, float('nan'), device='cuda')
    _tf32_gemm(A, B, one, gm, gn, klen, passes, transposed, k0=k0)
    torch.cuda.synchronize()
    assert torch.equal(parts[z], one[0]), (z, float((parts[z] - one[0]).abs().max()))


@pytest.mark.parametrize('gk,splits', [(576, 4), (640, 4), (600, 3)])
def test_bf16_split_slices_bit_exact(gk, splits):
  """The bf16 dW layout (both operands MN-major, read through the transpose bit)."""
  import ranking_b200  # noqa: F401
  from ranking_b200 import _C
  gm, gn, bk = 256, 136, 64
  g = torch.Generator().manual_seed(gk)
  A = torch.randn(gk, gm, generator=g).bfloat16().cuda()
  B = torch.randn(gk, gn, generator=g).bfloat16().cuda()
  rows = (gm + 127) // 128 * 128

  def run(C, k0, klen):
    a = ctypes.c_void_p(A.data_ptr() + 2 * k0 * gm)
    b = ctypes.c_void_p(B.data_ptr() + 2 * k0 * gn)
    _C.check(_C.lib.tfr_tc_gemm_bf16(
        a, gm, b, gn, _C.ptr(C), gn, gm, gn, klen, 1, 0, None, 0, None, None, None, 0, None,
        C.shape[0], rows * gn, _C.stream()))

  parts = torch.full((splits, rows, gn), float('nan'), device='cuda')
  run(parts, 0, gk)
  nkb = (gk + bk - 1) // bk
  per = (nkb + splits - 1) // splits
  for z in range(splits):
    k0 = z * per * bk
    klen = min(gk, k0 + per * bk) - k0
    if klen <= 0:
      assert torch.equal(parts[z, :gm], torch.zeros_like(parts[z, :gm])), z
      continue
    one = torch.full((1, rows, gn), float('nan'), device='cuda')
    run(one, k0, klen)
    torch.cuda.synchronize()
    assert torch.equal(parts[z, :gm], one[0, :gm]), z


@pytest.mark.parametrize('gk', BF16_GK)
def test_bf16_k_blocks_per_tile(gk):
  err, _, _ = run_kmajor(300, 136, gk, epi=1, act=1, want_bits=True, seed=gk)
  assert err <= 1e-5, err
  err, _, _ = run_kmajor(300, 136, gk, epi=3, act=1, want_colsum=True, seed=gk + 1)
  assert err <= 1e-5, err
  err, _, _ = run_mnmajor(136, 136, gk, 1, seed=gk + 2)
  assert err <= 2e-6, err


def test_bf16_tiles_chained_per_cta():
  err, _, _ = run_kmajor(33280, 136, 344, seed=5)
  assert err <= 1e-5, err


@pytest.mark.parametrize('gk,splits', [(576, 4), (640, 4), (600, 3)])
def test_bf16_short_and_empty_splits(gk, splits):
  err, _, _ = run_mnmajor(256, 136, gk, splits, seed=gk)
  assert err <= 2e-6, err


def _rel_err(got, ref):
  got = got.detach().double().cpu()
  ref = ref.detach().double().cpu()
  return float((got - ref).abs().max() / (ref.abs().max() + 1e-30))


@pytest.mark.parametrize('h2', TF32_GK)
def test_tower_colsum_1024_three_stage_ring(oracle_api, h2):
  """A 1024-wide hidden layer: its dZ GEMM (GN = 1024, GK = h2) takes bias column sums over
  1024 columns, which leaves room for three 3xTF32 stages, so the copies run one block ahead."""
  import ranking_b200 as tfr
  m, d = 600, 32
  tower = tfr.keras.layers.create_tower([1024, h2], 1, activation=None, use_batch_norm=False,
                                        dropout=0, input_dim=d, seed=h2, precision='tf32x3')
  with torch.no_grad():
    for i in range(len(tower.dims) - 1):
      tower.bias(i).uniform_(-0.2, 0.2)
  nl = len(tower.dims) - 1
  params = {'dense_w': [tower.kernel(i).detach().cpu().double().clone().requires_grad_()
                        for i in range(nl)],
            'dense_b': [tower.bias(i).detach().cpu().double().clone().requires_grad_()
                        for i in range(nl)]}
  g = torch.Generator().manual_seed(h2)
  x = torch.randn(m, d, generator=g)
  up = torch.randn(m, 1, generator=g)
  y = tower(x.cuda())
  (y * up.cuda()).sum().backward()
  ref = oracle_api.scorer.tower_forward(x.double(), params, activation=None)
  (ref * up.double()).sum().backward()
  assert _rel_err(y, ref) <= 1e-5, _rel_err(y, ref)
  want = torch.cat([torch.cat([w.grad.reshape(-1), b.grad.reshape(-1)])
                    for w, b in zip(params['dense_w'], params['dense_b'])])
  err = _rel_err(tower.flat.grad, want)
  assert err <= 5e-5, err
