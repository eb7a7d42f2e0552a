"""GPU tests of the fused tower forward's hand-off between its MMA warps and its epilogue
warpgroup (csrc/mlp_tc_fused.cu).

The MMA warps write each layer's activations into a shared-memory tile and wait for the
epilogue warpgroup to have stored the previous one before they overwrite it.  These towers
keep that wait on the critical path: with layers of one k block each the MMA warps reach
every epilogue before the epilogue warpgroup has finished the last one, and a 256-wide first
layer of one k block per chunk hands over its two chunks back to back.  Scores, hidden
activations and ReLU sign words must equal the per-layer path bit for bit, over many row
tiles per CTA and over a single partial tile, and two identical calls must give identical
bits.
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import pytest
import torch

import test_tower_fused_fwd_gpu as F

pytestmark = pytest.mark.gpu

# (input dim, hidden widths)
TOWERS = {
    'one_kblock_layers': (8, [32, 32, 32]),
    'one_kblock_chunks': (32, [256, 32]),
}


@pytest.mark.parametrize('out', (1, 8))
@pytest.mark.parametrize('act', ('relu', None))
@pytest.mark.parametrize('m', (129, 40000))
@pytest.mark.parametrize('name', sorted(TOWERS))
def test_handoff_matches_per_layer_bits(name, m, act, out):
  _C = F._lib()
  d, hidden = TOWERS[name]
  tower = F._tower(d, hidden, out, act, seed=3)
  x, mask = F._inputs(m, d, out == 1, seed=m + 7)
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


@pytest.mark.parametrize('name', sorted(TOWERS) + ['config2'])
def test_handoff_is_deterministic(name):
  _C = F._lib()
  if name == 'config2':
    d, hidden, out, act, _ = F.FUSED['config2']
  else:
    (d, hidden), out, act = TOWERS[name], 8, 'relu'
  tower = F._tower(d, hidden, out, act, seed=9)
  x, mask = F._inputs(40000, d, out == 1, seed=2)
  first, first_layers = F._fwd_workspace(_C, tower, x, mask)
  second, second_layers = F._fwd_workspace(_C, tower, x, mask)
  F._assert_same_bits(second, first, 'scores')
  for i, ((h, bits), (h0, bits0)) in enumerate(zip(second_layers, first_layers)):
    F._assert_same_bits(h, h0, 'H%d' % (i + 1))
    F._assert_same_bits(bits, bits0, 'sign words of H%d' % (i + 1))
