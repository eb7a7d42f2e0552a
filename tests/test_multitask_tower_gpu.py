"""The task-major ("planar") scorer entry points, tfr_mlp_fwd_tasks / tfr_mlp_bwd_tasks.

Forward: plane o of the scores is the transpose of tfr_mlp_fwd's interleaved column o, bit for
bit, on unmasked rows, and RestoreList's ln(1e-10) on masked rows of every plane; the call takes
the same route (launch count) as tfr_mlp_fwd, through the fused 3xTF32 kernel where that fits
and the per-layer walk where it does not.

Backward: the gradients and the input gradient match the fp64 reference of
tests/_tower_fp64.py fed the interleaved signal w_o * dscore_planes[o] with masked rows zeroed;
one task of weight 1 is tfr_mlp_bwd's bits; doubling every weight doubles every gradient
exactly; two identical calls agree bit for bit.  The argument checks need no GPU.
"""
import ctypes
import zlib

import pytest
import torch

import _tower_fp64 as R

PRECISIONS = ('fp32', 'tf32', 'tf32x3', 'tf32x3-layers')
# (input width, hidden widths) per mode; tf32x3-layers' first hidden layer is wider than the
# fused forward takes, so it runs layer by layer
TOWERS = {'fp32': (13, [37, 24]), 'fp32-oddK': (13, [37, 21]), 'tf32': (36, [64, 32]),
          'tf32x3': (36, [128, 64]), 'tf32x3-layers': (36, [260, 32])}


def _lib():
  import __graft_entry__ as entry
  entry.build()
  from ranking_b200 import _C
  return _C


def _prec(_C, mode):
  return {'fp32': _C.PREC_FP32, 'tf32': _C.PREC_TF32, 'tf32x3': _C.PREC_TF32X3,
          'tf32x3-layers': _C.PREC_TF32X3}[mode]


def _tower(mode, d, hidden, out, seed):
  import ranking_b200 as tfr
  precision = 'tf32x3' if mode.startswith('tf32x3') else mode
  t = tfr.keras.layers.create_tower(hidden, out, activation='relu', use_batch_norm=False,
                                    dropout=0, input_dim=d, precision=precision, seed=seed)
  g = torch.Generator().manual_seed(seed)
  with torch.no_grad():
    for i in range(len(t.dims) - 1):
      t.bias(i).copy_(torch.rand(t.dims[i + 1], generator=g) * 0.4 - 0.2)
  return t


class Case(object):
  """A tower, inputs, a mask and the buffers of one task-major call."""

  def __init__(self, mode, shape, out, m, masked, x_offset=0):
    self._C = _C = _lib()
    self.mode, self.prec, self.m, self.out = mode, _prec(_C, mode), m, out
    d, hidden = shape
    self.d, self.hidden = d, hidden
    seed = zlib.crc32(repr((mode, d, hidden, out, m)).encode()) & 0xFFFF
    self.tower = _tower(mode, d, hidden, out, seed)
    g = torch.Generator().manual_seed(seed + 1)
    store = torch.empty(m * d + 4, device='cuda')
    self.x = store[x_offset:x_offset + m * d].view(m, d)
    self.x.copy_(torch.randn(m, d, generator=g))
    self.planes_ds = torch.randn(out, m, generator=g).cuda()
    self.mask = (torch.rand(m, generator=g) > 0.25).cuda() if masked else None
    self.m8 = None if self.mask is None else self.mask.to(torch.uint8)
    self.cfg = self.tower._run_cfg()
    self.ws = self.tower._new_workspace(m)

  def fwd(self, tasks, mask=True):
    _C = self._C
    m8 = self.m8 if mask else None
    shape = (self.out, self.m) if tasks else (self.m, self.out)
    s = torch.full(shape, float('nan'), device='cuda')
    fn = _C.lib.tfr_mlp_fwd_tasks if tasks else _C.lib.tfr_mlp_fwd
    n0 = _C.lib.tfr_launch_count()
    _C.check(fn(_C.ptr(self.x), self.m, ctypes.byref(self.cfg), _C.ptr(self.tower.flat.data),
                _C.ptr(m8), _C.ptr(self.ws), _C.ptr(s), self.prec, _C.stream()))
    return s, _C.lib.tfr_launch_count() - n0

  def bwd_tasks(self, weights, ds=None):
    _C = self._C
    grads = torch.full_like(self.tower.flat.data, float('nan'))
    w = None if weights is None else (ctypes.c_float * self.out)(*weights)
    _C.check(_C.lib.tfr_mlp_bwd_tasks(
        _C.ptr(self.x), self.m, ctypes.byref(self.cfg), _C.ptr(self.tower.flat.data),
        _C.ptr(self.planes_ds if ds is None else ds), w, _C.ptr(self.m8), _C.ptr(self.ws),
        _C.ptr(grads), self.prec, _C.stream()))
    return grads

  def input_grad(self):
    _C = self._C
    dx = torch.full((self.m, self.d), float('nan'), device='cuda')
    _C.check(_C.lib.tfr_mlp_input_grad(ctypes.byref(self.cfg), self.m,
                                       _C.ptr(self.tower.flat.data), _C.ptr(self.ws), 0, self.d,
                                       _C.ptr(dx), self.d, self.prec, _C.stream()))
    return dx


def _need_cuda():
  if not torch.cuda.is_available():
    pytest.skip('no CUDA device')


# ---------------------------------------------------------------------------- forward ---
@pytest.mark.gpu
@pytest.mark.parametrize('m', [1, 129, 40000, 204800])
@pytest.mark.parametrize('out', [1, 2, 3, 5, 8])
@pytest.mark.parametrize('key', ['fp32', 'fp32-oddK', 'tf32', 'tf32x3', 'tf32x3-layers'])
def test_forward_planes(key, out, m):
  _need_cuda()
  mode = 'fp32' if key.startswith('fp32') else key
  c = Case(mode, TOWERS[key], out, m, masked=True)
  ref, n_ref = c.fwd(tasks=False, mask=False)
  planes, n_tasks = c.fwd(tasks=True)
  torch.cuda.synchronize()
  assert n_tasks == n_ref, (n_tasks, n_ref)   # same route as tfr_mlp_fwd
  live = c.mask
  want = ref.t()
  assert torch.equal(planes[:, live], want[:, live])
  assert (planes[:, ~live] == R.LOG_EPSILON).all()
  # without a mask every row is the transpose
  planes_nomask, _ = c.fwd(tasks=True, mask=False)
  assert torch.equal(planes_nomask, want)


# --------------------------------------------------------------------------- backward ---
def _ref_check(c, weights, grads, dx):
  """fp64 reference on the weighted, masked interleaved signal."""
  w = torch.tensor(weights if weights is not None else [1.0] * c.out, device='cuda')
  ds = (c.planes_ds * w[:, None]).t().contiguous()       # fp32, as the kernel forms it
  if c.mask is not None:
    ds[~c.mask] = 0.0
  planes, _ = c.fwd(tasks=True, mask=False)   # hidden activations for the gates
  L = len(c.hidden)
  rcfg = R.Cfg(c.tower.dims, relu=True)
  params = {'w': [c.tower.kernel(i) for i in range(L + 1)],
            'b': [c.tower.bias(i) for i in range(L + 1)]}
  got = {'hidden': R.hidden_activations(c.ws, rcfg, c.m), 'scores': planes.t(), 'grads': grads,
         'dx': [] if dx is None else [(0, c.d, dx)]}
  sms = torch.cuda.get_device_properties(0).multi_processor_count
  precision = 'tf32x3' if c.mode.startswith('tf32x3') else c.mode
  ratios = R.check(rcfg, precision, R.Plan(rcfg, c.m, sms), c.x, params, ds, got)
  print('%s o=%d m=%d w=%s: %s' % (c.mode, c.out, c.m, weights,
                                   ', '.join('%s %.3g' % r for r in ratios)))
  bad = [(what, r) for what, r in ratios if not r <= 1]
  assert not bad, bad


WEIGHTS = [None, (1.0, 0.5, 3.0)]


@pytest.mark.gpu
@pytest.mark.parametrize('masked', [False, True])
@pytest.mark.parametrize('weights', WEIGHTS, ids=['unit', 'mixed'])
@pytest.mark.parametrize('out', [1, 2, 3, 5, 8])
@pytest.mark.parametrize('key', ['fp32', 'fp32-oddK', 'tf32', 'tf32x3', 'tf32x3-layers'])
def test_backward_reference(key, out, weights, masked):
  _need_cuda()
  mode = 'fp32' if key.startswith('fp32') else key
  c = Case(mode, TOWERS[key], out, 3001, masked=masked)
  w = None if weights is None else [weights[i % 3] for i in range(out)]
  c.fwd(tasks=True)
  grads = c.bwd_tasks(w)
  dx = None if mode == 'fp32' else c.input_grad()
  torch.cuda.synchronize()
  _ref_check(c, w, grads, dx)


@pytest.mark.gpu
@pytest.mark.parametrize('mode', ['tf32x3', 'tf32'])
def test_backward_large(mode):
  _need_cuda()
  c = Case(mode, TOWERS[mode], 5, 204800, masked=True)
  w = [3.0, 0.5, 1.0, 3.0, 0.5]
  c.fwd(tasks=True)
  grads = c.bwd_tasks(w)
  dx = c.input_grad()
  torch.cuda.synchronize()
  _ref_check(c, w, grads, dx)


@pytest.mark.gpu
def test_backward_unaligned_input_no_hidden_layer():
  """No hidden layer and X 4 bytes off 16-byte alignment: the output layer reads X itself,
  which the float4 planar backward cannot; the per-split kernel writes the slots instead."""
  _need_cuda()
  c = Case('tf32x3', (36, []), 3, 3001, masked=True, x_offset=1)
  w = [0.5, 3.0, 1.0]
  c.fwd(tasks=True)
  grads = c.bwd_tasks(w)
  torch.cuda.synchronize()
  _ref_check(c, w, grads, None)


@pytest.mark.gpu
@pytest.mark.parametrize('masked', [False, True])
@pytest.mark.parametrize('key', ['fp32', 'tf32', 'tf32x3', 'tf32x3-layers'])
def test_one_task_is_mlp_bwd(key, masked):
  _need_cuda()
  _C = _lib()
  c = Case(key, TOWERS[key], 1, 40000, masked=masked)
  c.fwd(tasks=False)
  ref = torch.empty_like(c.tower.flat.data)
  _C.check(_C.lib.tfr_mlp_bwd(_C.ptr(c.x), c.m, ctypes.byref(c.cfg), _C.ptr(c.tower.flat.data),
                              _C.ptr(c.planes_ds), _C.ptr(c.m8), _C.ptr(c.ws), _C.ptr(ref),
                              c.prec, _C.stream()))
  dx_ref = None if key == 'fp32' else c.input_grad()
  c.fwd(tasks=True)
  got = c.bwd_tasks([1.0])
  got_none = c.bwd_tasks(None)
  dx = None if key == 'fp32' else c.input_grad()
  torch.cuda.synchronize()
  assert torch.equal(got, ref)
  assert torch.equal(got_none, ref)
  if dx is not None:
    assert torch.equal(dx, dx_ref)


@pytest.mark.gpu
@pytest.mark.parametrize('out', [1, 3, 8])
@pytest.mark.parametrize('key', ['fp32', 'tf32', 'tf32x3', 'tf32x3-layers'])
def test_weight_scaling_and_determinism(key, out):
  _need_cuda()
  c = Case(key, TOWERS[key], out, 40000, masked=True)
  w = [(0.5, 3.0, 1.25)[i % 3] for i in range(out)]
  c.fwd(tasks=True)
  g1 = c.bwd_tasks(w)
  g1b = c.bwd_tasks(w)
  g2 = c.bwd_tasks([2.0 * v for v in w])
  torch.cuda.synchronize()
  assert torch.equal(g1, g1b)
  assert torch.equal(g2, 2.0 * g1)


# ---------------------------------------------------------------------- argument errors ---
def test_argument_errors():
  """TFR_INVALID_ARGUMENT (1) before any CUDA call: the pointers below are never touched."""
  _C = _lib()
  lib = _C.lib
  p = ctypes.c_void_p(256)

  def cfg(out):
    c = _C.MlpCfg()
    c.n_dense = 2
    c.dims[0], c.dims[1], c.dims[2] = 8, 16, out
    c.activation = _C.ACT_RELU
    c.bn_epsilon, c.bn_momentum = 1e-3, 0.999
    return c

  def fwd(c, prec=_C.PREC_TF32X3, planes=p):
    return lib.tfr_mlp_fwd_tasks(p, 64, ctypes.byref(c), p, None, p, planes, prec, None)

  def bwd(c, prec=_C.PREC_TF32X3, planes=p, w=None):
    return lib.tfr_mlp_bwd_tasks(p, 64, ctypes.byref(c), p, planes, w, None, p, p, prec, None)

  assert fwd(cfg(9)) == 1 and 'task count' in _C.last_error()
  assert bwd(cfg(9)) == 1 and 'task count' in _C.last_error()
  assert fwd(cfg(2), prec=_C.PREC_BF16) == 1 and 'precision' in _C.last_error()
  assert bwd(cfg(2), prec=_C.PREC_BF16) == 1 and 'precision' in _C.last_error()
  assert fwd(cfg(2), planes=None) == 1 and 'NULL' in _C.last_error()
  assert bwd(cfg(2), planes=None) == 1 and 'NULL' in _C.last_error()
  for bad in (float('nan'), float('inf')):
    w = (ctypes.c_float * 2)(1.0, bad)
    assert bwd(cfg(2), w=w) == 1 and 'not finite' in _C.last_error()
  assert lib.tfr_mlp_fwd_tasks(p, 64, None, p, None, p, p, _C.PREC_FP32, None) == 1
