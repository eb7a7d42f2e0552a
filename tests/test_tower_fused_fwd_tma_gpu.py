"""GPU tests of the fused tower forward's TMA operand ring and TMA activation stores
(csrc/mlp_tc_fused.cu).

The kernel loads W^T hi / lo and X tiles as TMA boxes of 32 columns x 128 rows, zero-filled
past K, N and M, and stores each hidden activation from shared memory as the same boxes,
clipped to M and N.  These towers put every edge of that under test: row counts of one row,
one short of and one past a tile, and 128 k + 5; input widths of 4 and 20 (a box wider than
the tensor), 136 (a K tail) and 256; 64-, 128- and 256-wide layers; and enough rows that every
CTA walks many tiles, so the stage ring wraps across layers and tiles.  Scores, hidden
activations and ReLU sign words must equal the per-layer path bit for bit, and two identical
calls must give identical bits.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import pytest

import test_tower_fused_fwd_gpu as F

pytestmark = pytest.mark.gpu

ROWS = (1, 127, 129, 128 * 7 + 5, 128 * 700 + 5)

# (input dim, hidden widths, output units)
TOWERS = {
    'd4_w64': (4, [64, 64], 8),
    'd20_w128': (20, [128, 64], 3),
    'd136_w256': (136, [256, 128, 64], 1),
    'd256_w256_w64': (256, [256, 64], 8),
    'd136_w64_w128': (136, [64, 128, 128], 2),
}


def _check(name, m, act, seed):
  _C = F._lib()
  d, hidden, out = TOWERS[name]
  tower = F._tower(d, hidden, out, act, seed=seed)
  x, mask = F._inputs(m, d, out == 1, seed=m + seed)
  got, launches = F._fwd_launches(_C, tower, x, mask)
  assert launches == 2, launches   # parameter split + the fused kernel
  want, want_layers = F._per_layer(_C, tower, x, mask, act)
  F._assert_same_bits(got, want, 'scores')
  got_ws, got_layers = F._fwd_workspace(_C, tower, x, mask)
  F._assert_same_bits(got_ws, want, 'scores (explicit workspace)')
  for i, ((h, bits), (want_h, want_bits)) in enumerate(zip(got_layers, want_layers)):
    F._assert_same_bits(h, want_h, 'H%d' % (i + 1))
    if want_bits is not None:
      F._assert_same_bits(bits, want_bits, 'sign words of H%d' % (i + 1))
  return tower, x, mask, got_layers


@pytest.mark.parametrize('m', ROWS)
@pytest.mark.parametrize('name', sorted(TOWERS))
def test_tma_forward_matches_per_layer_bits(name, m):
  _check(name, m, 'relu', seed=17)


@pytest.mark.parametrize('name', sorted(TOWERS))
def test_tma_forward_without_activation(name):
  _check(name, 128 * 7 + 5, None, seed=23)


@pytest.mark.parametrize('name', sorted(TOWERS))
def test_tma_forward_is_deterministic(name):
  _C = F._lib()
  tower, x, mask, first_layers = _check(name, 128 * 700 + 5, 'relu', seed=29)
  first, _ = F._fwd_workspace(_C, tower, x, mask)
  second, second_layers = F._fwd_workspace(_C, tower, x, mask)
  F._assert_same_bits(second, first, 'scores')
  for i, ((h, bits), (h0, bits0)) in enumerate(zip(second_layers, first_layers)):
    F._assert_same_bits(h, h0, 'H%d' % (i + 1))
    F._assert_same_bits(bits, bits0, 'sign words of H%d' % (i + 1))
