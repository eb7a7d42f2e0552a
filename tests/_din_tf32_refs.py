"""CPU-side pieces of tests/test_din_tf32_gpu.py: the error bars of DocumentInteractionAttention
in precision 'tf32' and the head-size buckets of its tensor-core attention kernels, read from
csrc/din_tc.cu (tc_bucket) so that the case table's coverage is recomputed from the dispatch
itself.

Bars.  In 'tf32' every contraction of the DIN is one TF32 product: the projection GEMMs, their
dW and input-gradient GEMMs, and the attention core's q.k, P~ v, dO.v, dS k, P~^T dO and dS^T q
(csrc/din_tc.cu).  tests/_tower_fp64.py's accounting charges one such contraction of depth k

    u(k) = u_p + k u_acc,   u_p = 2^-9 + 2^-20 (both operands truncated to TF32),
                            u_acc = 2^-23 (the tensor core's additions, a full ulp each),

relative to the sum of magnitudes it adds.  The elementwise fp32 steps (softmax, LayerNorm,
dropout, residual adds) are ~2^-24 each and are dropped beside u_p ~ 2^-9.  A quantity's
first-order error is the sum of the u of the contractions on its longest path, times
tests/_tower_fp64.py's safety factor C = 2:
  * forward output: the input projection, then per layer the QKV projection, S, P~ V and the
    output projection: 1 + 4 L contractions;
  * every parameter-gradient block and the input gradient: the forward chain, then back through
    every layer (dO = dY Wo^T; S and dP recomputed; dQ / dK / dV; dX = dQKV W^T), then the
    block's own dW GEMM: 2 + 9 L contractions;
with k the deepest contraction of the shape, max(N, D, 3 H h).  The per-block shape is
tests/test_din_limits_gpu.py's: W_q / b_q grow with N / 256 past N = 256 (their gradient is
what survives the cancellation sum_j dS_ij = 0) and the key bias is measured against its
kernel's gradient norm (its exact gradient is 0).  With N = 1 the softmax is constant, so the
exact gradients of W_q, b_q, W_k and b_k are all 0; their errors are then measured against the
norm of the same layer's W_v gradient, whose entries sum the same dO v products.

The kernels round the A operands they form in registers (P~, dS) to nearest TF32; every tile
read from shared memory is truncated by the tensor core.  The bars charge truncation to every
operand, an upper bound for both.
"""
import os
import re

import _tower_fp64 as T
from oracle import din as odin

U_P = 2.0 ** -9 + 2.0 ** -20
U_ACC = 2.0 ** -23
ROWS = 64   # query rows of a CTA, keys of a tile (din_tc.cu kT)

_SRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'ranking_b200',
                    'csrc', 'din_tc.cu')


def buckets():
  """[(edge, HP), ...] of tc_bucket in din_tc.cu: h <= edge -> HP; the last HP takes the rest."""
  src = open(_SRC).read()
  body = re.search(r'constexpr int tc_bucket\(int h\) \{(.*?)\}', src, re.S).group(1)
  pairs = [(int(a), int(b)) for a, b in re.findall(r'h <= (\d+) \? (\d+)', body)]
  last = int(re.search(r': (\d+);', body).group(1))
  return pairs, last


def bucket(h):
  pairs, last = buckets()
  for edge, hp in pairs:
    if h <= edge:
      return hp
  return last


def _u(n, d, h, heads):
  return U_P + max(n, d, 3 * heads * h) * U_ACC


def out_bar(n, d, h, heads, nl):
  return T.C * (1 + 4 * nl) * _u(n, d, h, heads)


def grad_bar(n, d, h, heads, nl):
  return T.C * (2 + 9 * nl) * _u(n, d, h, heads)


def bars(n, d, h, heads, nl):
  """{block: bar} for the flat gradient (see the module docstring)."""
  g = grad_bar(n, d, h, heads, nl)
  q = g * max(1.0, n / 256)
  return {name: q if name[:2] in ('wq', 'bq') else g
          for name, _ in odin.param_shapes(d, h, heads, nl)}
