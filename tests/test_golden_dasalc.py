"""DASALC (K13) without a GPU: the feature transform's closed-form points, the documented
parameter / bn_state layout, every argument error (reported before any CUDA call) and the
numerical ELWC fixtures of the reference's DASALC example."""
import ctypes
import math
import os

import pytest
import torch

import __graft_entry__ as g

g.build()
from ranking_b200 import _C  # noqa: E402
from ranking_b200 import data  # noqa: E402
from ranking_b200.research import dasalc  # noqa: E402
import _dasalc_refs as ref  # noqa: E402

NUMERICAL = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'numerical')


def _cfg(d=136, w=512, h=100, **kw):
  c = _C.DasalcCfg()
  c.input_dim, c.hidden_dim, c.context_dim = d, w, h
  c.dropout = kw.get('dropout', 0.4)
  c.input_noise_stddev = kw.get('noise', 1.5)
  c.bn_epsilon = kw.get('eps', 1e-3)
  c.bn_momentum = kw.get('momentum', 0.9)
  c.training = 1
  c.bn_state = kw.get('bn_state', 16)   # any non-NULL address: never dereferenced here
  return c


def test_log1p_cutoff_closed_form():
  x = torch.tensor([0.0, 1.0, -1.0, -3.0, 1e20, -1e20, math.e - 1.0])
  want = torch.tensor([0.0, math.log(2.0), -math.log(2.0), -math.log(4.0), 30.0, -30.0, 1.0],
                      dtype=torch.float64)
  assert torch.allclose(ref.transform(x), want, rtol=0, atol=1e-7)
  assert torch.equal(ref.transform(torch.tensor([1e20]), cutoff=5.0),
                     torch.tensor([5.0], dtype=torch.float64))


def test_log1p_cutoff_needs_a_device_tensor():
  with pytest.raises(RuntimeError, match='CUDA device'):
    dasalc.log1p_cutoff(torch.zeros(4))


@pytest.mark.parametrize('d,w,h', [(136, 512, 100), (4, 64, 4), (700, 3072, 128)])
def test_counts_follow_documented_layout(d, w, h):
  c = _cfg(d, w, h)
  shapes = ref.param_shapes(d, w, h)
  assert [n for n, _ in shapes] == ['w1', 'b1', 'w2', 'b2', 'wt', 'bt', 'wc', 'bc', 'wo', 'bo',
                                    'g_in', 'be_in', 'g1', 'be1', 'g2', 'be2', 'gc', 'bec']
  want = sum(math.prod(s) for _, s in shapes)
  assert want == d * w + w + 2 * (w * w + w) + h * w + w + w + 1 + 2 * d + 4 * w + 2 * h
  assert _C.lib.tfr_dasalc_param_count(ctypes.byref(c)) == want
  assert _C.lib.tfr_dasalc_bn_state_count(ctypes.byref(c)) == 2 * (d + 2 * w + h)
  assert _C.lib.tfr_dasalc_workspace_bytes(ctypes.byref(c), 1000) > 0


@pytest.mark.parametrize('field,value,msg', [
    ('input_dim', 0, 'input_dim'), ('input_dim', 6, 'input_dim'),
    ('hidden_dim', 10, 'hidden_dim'), ('hidden_dim', 4100, 'hidden_dim'),
    ('context_dim', 132, 'context_dim'), ('context_dim', 2, 'context_dim'),
    ('dropout', 1.0, 'dropout'), ('dropout', -0.1, 'dropout'),
    ('input_noise_stddev', -1.0, 'input_noise_stddev'), ('bn_epsilon', 0.0, 'bn_epsilon'),
    ('bn_momentum', 1.5, 'bn_momentum')])
def test_config_errors(field, value, msg):
  c = _cfg()
  setattr(c, field, value)
  assert _C.lib.tfr_dasalc_param_count(ctypes.byref(c)) == 0
  assert msg in _C.last_error()
  assert _C.lib.tfr_dasalc_bn_state_count(ctypes.byref(c)) == 0
  assert _C.lib.tfr_dasalc_workspace_bytes(ctypes.byref(c), 8) == 0
  p = ctypes.c_void_p(16)
  assert _C.lib.tfr_dasalc_fwd(p, p, 100, 8, ctypes.byref(c), p, None, p, p,
                               _C.PREC_TF32X3, None) == 1
  assert _C.lib.tfr_dasalc_bwd(p, 8, ctypes.byref(c), p, p, None, p, p, p, 100,
                               _C.PREC_TF32X3, None) == 1


def _fwd(c, x=16, e=16, lde=100, m=8, params=16, ws=16, scores=16, prec=_C.PREC_TF32X3):
  v = lambda a: None if a is None else ctypes.c_void_p(a)  # noqa: E731
  return _C.lib.tfr_dasalc_fwd(v(x), v(e), lde, m, c, v(params), None, v(ws), v(scores), prec,
                               None)


def _bwd(c, x=16, m=8, params=16, ds=16, ws=16, grads=16, de=16, ldde=100,
         prec=_C.PREC_TF32X3):
  v = lambda a: None if a is None else ctypes.c_void_p(a)  # noqa: E731
  return _C.lib.tfr_dasalc_bwd(v(x), m, c, v(params), v(ds), None, v(ws), v(grads), v(de),
                               ldde, prec, None)


def test_call_argument_errors():
  c = ctypes.byref(_cfg())
  assert _fwd(None) == 1 and 'NULL' in _C.last_error()
  for kw in ({'x': None}, {'e': None}, {'params': None}, {'ws': None}, {'scores': None}):
    assert _fwd(c, **kw) == 1 and 'NULL' in _C.last_error(), kw
  assert _fwd(c, lde=96) == 1 and 'lde' in _C.last_error()
  assert _fwd(c, m=-1) == 1 and 'M' in _C.last_error()
  assert _fwd(c, m=1 << 24) == 1 and '2^31' in _C.last_error()
  for kw in ({'x': None}, {'params': None}, {'ds': None}, {'ws': None}, {'grads': None},
             {'de': None}):
    assert _bwd(c, **kw) == 1 and 'NULL' in _C.last_error(), kw
  assert _bwd(c, ldde=99) == 1 and 'ldde' in _C.last_error()
  assert _bwd(c, m=-5) == 1
  nostate = ctypes.byref(_cfg(bn_state=None))
  assert _fwd(nostate) == 1 and 'bn_state' in _C.last_error()
  assert _bwd(nostate) == 1 and 'bn_state' in _C.last_error()
  for prec in (_C.PREC_FP32, _C.PREC_BF16, 7):
    assert _fwd(c, prec=prec) == 2 and 'precision' in _C.last_error()
    assert _bwd(c, prec=prec) == 2
  p = ctypes.c_void_p(16)
  assert _C.lib.tfr_symmetric_log1p_clip(None, 4, 30.0, p, None) == 1
  assert _C.lib.tfr_symmetric_log1p_clip(p, 4, 30.0, None, None) == 1
  assert _C.lib.tfr_symmetric_log1p_clip(p, 4, 0.0, p, None) == 1
  assert 'cutoff' in _C.last_error()


def test_scorer_argument_errors():
  with pytest.raises(ValueError, match='precision'):
    dasalc.DASALCScorer(136, precision='bf16', device='cpu')
  with pytest.raises(ValueError, match='hidden_dim'):
    dasalc.DASALCScorer(136, hidden_dim=510, device='cpu')


@pytest.mark.parametrize('name', ['train_numerical_elwc.tfrecord', 'vali_numerical_elwc.tfrecord'])
def test_numerical_fixtures_parse(name):
  spec = {'custom_features_%d' % (i + 1): (1, 0.0) for i in range(136)}
  spec['utility'] = (1, -1.0)
  batches = list(data.elwc_batches(os.path.join(NUMERICAL, name), 4, 200, None, spec, 'utility',
                                   drop_remainder=False, pin_memory=False))
  assert batches
  for x, y in batches:
    assert list(x.shape[1:]) == [200, 136] and list(y.shape) == [x.shape[0], 200]
    assert set(torch.unique(y).tolist()) <= {-1.0, 0.0, 1.0, 2.0, 3.0, 4.0}
    assert bool((y >= 0).any(1).all())   # every list has a labelled item
    assert bool(torch.isfinite(x).all())
  x = torch.cat([b[0] for b in batches])
  assert float(x.abs().max()) > 0
