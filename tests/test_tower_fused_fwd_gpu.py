"""GPU tests of the fused 3xTF32 tower forward (csrc/mlp_tc_fused.cu).

Towers inside the fused kernel's limits must give exactly the bits of the per-layer path:
each Dense layer through the wgmma engine (`tfr_tc_gemm`, W^T split into hi / lo the way
split_params_kernel does it), then the same last hidden activation through a tower with no
hidden layer on the CUDA-core path, which runs the same output-layer kernel.  The hidden
activations and ReLU sign words the fused kernel stores in the workspace (the backward reads
them) must equal the per-layer GEMMs' outputs bit for bit as well.  Towers just
past a width limit take the per-layer path (one launch per layer, seen in the launch counter)
and must still match an fp64 forward to 1e-5.  (More than 8 output units is refused by the
tower plan itself.)
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import pytest
import torch

pytestmark = pytest.mark.gpu

ROWS = (1, 127, 129, 300, 4100)
MANY_TILES = 40000   # 313 row tiles: every CTA of the persistent grid walks several

# (input dim, hidden widths, output units, activation, masked)
FUSED = {
    'config2': (136, [256, 128, 64], 1, 'relu', True),
    'ktails_n64': (20, [132, 100, 4], 2, 'relu', False),   # 4-wide second chunk, K tails
    'identity': (36, [64, 32], 1, None, True),
    'one_hidden': (16, [128], 8, 'relu', False),
    'long_k': (1024, [256, 128, 64], 2, 'relu', False),   # 32 k blocks per chunk
}
PAST_LIMIT = {
    'first_260': (24, [260, 64], 1, 'relu', True),
    'later_132': (24, [128, 132], 1, 'relu', False),
}


def _lib():
  import __graft_entry__ as entry
  entry.build()
  from ranking_b200 import _C
  return _C


def _tower(d, hidden, out, act, seed):
  import ranking_b200 as tfr
  t = tfr.keras.layers.create_tower(hidden, out, activation=act, use_batch_norm=False,
                                    dropout=0, input_dim=d, seed=seed, precision='tf32x3')
  with torch.no_grad():
    for i in range(len(t.dims) - 1):
      t.bias(i).uniform_(-0.2, 0.2)
  return t.eval()


def _inputs(m, d, masked, seed):
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(m, d, generator=g).cuda()
  mask = (torch.rand(m, generator=g) > 0.3).cuda() if masked else None
  return x, mask


def _fwd_launches(_C, tower, x, mask):
  n0 = _C.lib.tfr_launch_count()
  with torch.no_grad():
    s = tower(x, mask)
  torch.cuda.synchronize()
  return s, _C.lib.tfr_launch_count() - n0


def _fwd_workspace(_C, tower, x, mask):
  """tfr_mlp_fwd on an explicit workspace: (scores, [(H_d, sign words_d) per hidden layer]).
  The workspace starts at the next 256-byte boundary with, per hidden layer d, H_d [M, n_d]
  then its sign words [ceil(n_d / 32), M], each region padded to 64 floats."""
  import ctypes
  m = x.shape[0]
  ws = tower._new_workspace(m)
  out = torch.empty(m, tower.output_units, device='cuda')
  cfg = tower._run_cfg()
  m8 = None if mask is None else mask.to(torch.uint8).contiguous()
  _C.check(_C.lib.tfr_mlp_fwd(_C.ptr(x), m, ctypes.byref(cfg), _C.ptr(tower.flat.data),
                              _C.ptr(m8), _C.ptr(ws), _C.ptr(out), _C.PREC_TF32X3,
                              _C.stream()))
  torch.cuda.synchronize()
  base = (-ws.data_ptr()) % 256
  flat = ws[base:base + (ws.numel() - base) // 4 * 4].view(torch.float32)
  up = lambda n: (n + 63) // 64 * 64
  layers, w = [], 0
  for n in tower.dims[1:-1]:
    h = flat[w:w + m * n].view(m, n)
    w += up(m * n)
    nw = (n + 31) // 32
    bits = flat[w:w + nw * m].view(torch.int32).view(nw, m)
    w += up(nw * m)
    layers.append((h, bits))
  return out, layers


def _per_layer(_C, tower, x, mask, act):
  """Dense layers one by one through tfr_tc_gemm (3xTF32, W^T pre-split), then the output
  layer of a zero-hidden-layer fp32 tower on the last activation.  Returns the scores and
  [(H_d, sign words_d)] (sign words None without ReLU)."""
  import ranking_b200 as tfr
  h = x
  layers = []
  L = len(tower.dims) - 2
  for i in range(L):
    w_t = tower.kernel(i).detach().t().contiguous()
    hi = ((w_t.view(torch.int32) + 4096) & -8192).view(torch.float32)   # RN to TF32
    lo = w_t - hi
    k, n = tower.dims[i], tower.dims[i + 1]
    out = torch.empty(h.shape[0], n, device='cuda')
    bits = torch.empty((n + 31) // 32, h.shape[0], dtype=torch.int32, device='cuda')
    _C.check(_C.lib.tfr_tc_gemm(
        _C.ptr(h), k, _C.ptr(hi), k, _C.ptr(lo), _C.ptr(out), n, h.shape[0], n, k, 0, 0, 3,
        0, 1, _C.ptr(tower.bias(i).detach()), None, 1 if act == 'relu' else 0, 0, 1, 0,
        _C.ptr(bits) if act == 'relu' else None, None, _C.stream()))
    h = out
    layers.append((out, bits if act == 'relu' else None))
  head = tfr.keras.layers.create_tower([], tower.output_units, input_dim=tower.dims[L],
                                       precision='fp32')
  head.load_keras_weights([tower.kernel(L).detach().cpu()], [tower.bias(L).detach().cpu()])
  with torch.no_grad():
    s = head(h, mask)
  torch.cuda.synchronize()
  return s, layers


def _assert_same_bits(got, want, what):
  assert got.shape == want.shape, (what, got.shape, want.shape)
  diff = (got != want).nonzero()
  assert diff.numel() == 0, (what, diff[:8].tolist(), got[tuple(diff[0])].item(),
                             want[tuple(diff[0])].item())


def _fp64(tower, x, mask, act):
  h = x.double()
  L = len(tower.dims) - 2
  for i in range(L + 1):
    h = h @ tower.kernel(i).detach().double() + tower.bias(i).detach().double()
    if i < L and act == 'relu':
      h = torch.relu(h)
  if mask is not None and tower.output_units == 1:
    h = torch.where(mask.reshape(-1, 1), h, torch.full_like(h, -23.025850929940457))
  return h


@pytest.mark.parametrize('name,m', [(n, m) for n in sorted(FUSED) for m in ROWS] +
                         [('config2', MANY_TILES), ('ktails_n64', MANY_TILES)])
def test_fused_forward_matches_per_layer_bits(name, m):
  _C = _lib()
  d, hidden, out, act, masked = FUSED[name]
  tower = _tower(d, hidden, out, act, seed=11)
  x, mask = _inputs(m, d, masked, seed=m)
  got, launches = _fwd_launches(_C, tower, x, mask)
  assert launches == 2, launches   # parameter split + the fused kernel
  want, want_layers = _per_layer(_C, tower, x, mask, act)
  _assert_same_bits(got, want, 'scores')
  got_ws, got_layers = _fwd_workspace(_C, tower, x, mask)
  _assert_same_bits(got_ws, want, 'scores (explicit workspace)')
  for i, ((h, bits), (want_h, want_bits)) in enumerate(zip(got_layers, want_layers)):
    _assert_same_bits(h, want_h, 'H%d' % (i + 1))
    if want_bits is not None:
      _assert_same_bits(bits, want_bits, 'sign words of H%d' % (i + 1))


@pytest.mark.parametrize('m', (129, 4100))
@pytest.mark.parametrize('name', sorted(PAST_LIMIT))
def test_past_the_limits_takes_per_layer_path(name, m):
  _C = _lib()
  d, hidden, out, act, masked = PAST_LIMIT[name]
  tower = _tower(d, hidden, out, act, seed=5)
  x, mask = _inputs(m, d, masked, seed=m + 1)
  got, launches = _fwd_launches(_C, tower, x, mask)
  assert launches == len(hidden) + 2, launches   # split + one GEMM per layer + output layer
  ref = _fp64(tower, x, mask, act)
  err = (got.double() - ref).abs().max().item() / max(1.0, ref.abs().max().item())
  assert err <= 1e-5, err
