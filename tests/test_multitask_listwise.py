"""Multi-task DASALC entry points without a GPU: parameter counts, and every argument error
reported before any CUDA call."""
import ctypes
import math

import pytest

ROOT_PTR = ctypes.c_void_p(256)   # never dereferenced: the calls fail their checks first


@pytest.fixture(scope='module')
def C():
  import __graft_entry__ as g
  g.build()
  from ranking_b200 import _C
  return _C


def _cfg(C, d=16, w=64, h=8):
  cfg = C.DasalcCfg()
  cfg.input_dim, cfg.hidden_dim, cfg.context_dim = d, w, h
  cfg.dropout, cfg.bn_epsilon, cfg.bn_momentum, cfg.training = 0.1, 1e-3, 0.9, 1
  cfg.bn_state = ROOT_PTR.value
  return cfg


def test_param_counts(C):
  import _multitask_listwise_refs as mref
  cfg = _cfg(C)
  one = C.lib.tfr_dasalc_param_count(ctypes.byref(cfg))
  for t in range(1, 9):
    n = C.lib.tfr_dasalc_param_count_tasks(ctypes.byref(cfg), t)
    assert n == one + 65 * (t - 1) == mref.param_count(16, 64, 8, t)
  for t in (0, 9, -1):
    assert C.lib.tfr_dasalc_param_count_tasks(ctypes.byref(cfg), t) == 0
    assert 'num_tasks' in C.last_error()
    assert C.lib.tfr_dasalc_workspace_bytes_tasks(ctypes.byref(cfg), 100, t) == 0


def _fwd(C, cfg, t=2, precision=None, planes=ROOT_PTR):
  precision = C.PREC_TF32X3 if precision is None else precision
  return C.lib.tfr_dasalc_fwd_tasks(ROOT_PTR, ROOT_PTR, 8, 100, ctypes.byref(cfg), ROOT_PTR,
                                    None, ROOT_PTR, planes, t, precision, None)


def _bwd(C, cfg, t=2, weights=None, precision=None, planes=ROOT_PTR, grads=ROOT_PTR):
  precision = C.PREC_TF32X3 if precision is None else precision
  w = None if weights is None else (ctypes.c_float * len(weights))(*weights)
  return C.lib.tfr_dasalc_bwd_tasks(ROOT_PTR, 100, ctypes.byref(cfg), ROOT_PTR, planes, w, None,
                                    ROOT_PTR, grads, ROOT_PTR, 8, t, precision, None)


@pytest.mark.parametrize('t', [0, 9])
def test_task_count_out_of_range(C, t):
  cfg = _cfg(C)
  assert _fwd(C, cfg, t=t) == 1 and 'num_tasks' in C.last_error()
  assert _bwd(C, cfg, t=t) == 1 and 'num_tasks' in C.last_error()


def test_fp32_precision_refused(C):
  cfg = _cfg(C)
  assert _fwd(C, cfg, precision=C.PREC_FP32) == 1 and 'precision' in C.last_error()
  assert _bwd(C, cfg, precision=C.PREC_FP32) == 1 and 'precision' in C.last_error()


@pytest.mark.parametrize('bad', [math.nan, math.inf, -math.inf])
def test_non_finite_weight_refused(C, bad):
  assert _bwd(C, _cfg(C), t=3, weights=[1.0, bad, 0.5]) == 1
  assert 'finite' in C.last_error()


def test_null_planes_and_grads_refused(C):
  cfg = _cfg(C)
  assert _fwd(C, cfg, planes=None) == 1 and 'NULL' in C.last_error()
  assert _bwd(C, cfg, planes=None) == 1 and 'NULL' in C.last_error()
  assert _bwd(C, cfg, grads=None) == 1 and 'NULL' in C.last_error()


def test_trainer_and_scorer_arguments(C):
  """The host checks that need no device tensor."""
  from ranking_b200 import train
  tp = train._TaskPlanes()
  with pytest.raises(ValueError, match='output units'):
    tp._set_tasks({'a': _FusedLoss(), 'b': _FusedLoss()}, None, 3)
  with pytest.raises(ValueError, match='unknown tasks'):
    tp._set_tasks({'a': _FusedLoss()}, {'z': 1.0}, 1)
  with pytest.raises(ValueError, match='finite'):
    tp._set_tasks({'a': _FusedLoss()}, {'a': math.nan}, 1)
  assert tp._set_tasks({'a': _FusedLoss(), 'b': _FusedLoss()}, {'b': 0.5}, 2) is not None
  assert tp.loss_weights == [1.0, 0.5]


class _FusedLoss(object):
  fused_single_score = True

  def fused_fwd_bwd(self, *args):
    raise AssertionError('not called')
