"""GAMLayer / GAMScorer known answers of the reference (keras/layers_test.py:277-324,
keras/model_test.py:436-450), against the oracle and (-m gpu) the CUDA layer; plus the
C ABI's configuration checks without a GPU."""
import ctypes

import pytest
import torch

from oracle import gam as OG


class _OracleGAM(object):
  """The oracle behind the GAMLayer call signature (parameters made at first call)."""

  def __init__(self, example_feature_num, example_hidden_layer_dims, context_feature_num=None,
               context_hidden_layer_dims=None, **kw):
    if context_feature_num and not context_hidden_layer_dims:
      raise ValueError('When `context_feature_num` > 0, `context_hidden_layer_dims` is '
                       'required!')
    self.args = (example_feature_num, example_hidden_layer_dims, context_feature_num or 0,
                 context_hidden_layer_dims)
    self.kw = kw
    self.params = None

  def __call__(self, inputs):
    ex, cx = inputs
    f, hid, c, chid = self.args
    if self.params is None:
      dims = [t.shape[1] for t in ex] if len(ex) == f else [1] * f
      cdims = [t.shape[1] for t in cx] if cx and len(cx) == c else [1] * c
      self.params = OG.init_gam_params(dims, hid, cdims, chid,
                                       use_batch_norm=self.kw.get('use_batch_norm', True))
    ex = [t.double() for t in ex]
    cx = [t.double() for t in cx] if cx else cx
    return OG.gam_layer(ex, cx, self.params, use_batch_norm=self.kw.get('use_batch_norm', True))


@pytest.fixture(params=['oracle', pytest.param('cuda', marks=pytest.mark.gpu)])
def gam_api(request):
  if request.param == 'oracle':
    return _OracleGAM, torch.device('cpu')
  if not torch.cuda.is_available():
    pytest.skip('no CUDA device')
  import ranking_b200 as tfr
  return tfr.keras.layers.GAMLayer, torch.device('cuda:0')


def _t(x, dev):
  return torch.tensor(x, dtype=torch.float32, device=dev)


def test_gam_layer_call(gam_api):
  GAM, dev = gam_api
  example_inputs = _t([[1], [0], [-1]], dev)
  context_inputs = _t([[1, 2], [0, 1], [-1, 1]], dev)
  gam = GAM(2, [3, 2, 1], 2, [3, 2, 1])
  outputs, sublogits_list, subweights_list = gam(
      ([example_inputs, example_inputs], [context_inputs, context_inputs]))
  assert list(outputs.shape) == [3, 1]
  assert len(sublogits_list) == 2
  assert all(list(s.shape) == [3, 1] for s in sublogits_list)
  assert len(subweights_list) == 2
  assert all(list(s.shape) == [3, 2] for s in subweights_list)


def test_gam_layer_call_without_context(gam_api):
  GAM, dev = gam_api
  example_inputs = _t([[1], [0], [-1]], dev)
  for gam in (GAM(2, [3, 2, 1], 2, [3, 2, 1]), GAM(2, [3, 2, 1])):
    outputs, sublogits_list, subweights_list = gam(([example_inputs, example_inputs], None))
    assert list(outputs.shape) == [3, 1]
    assert len(sublogits_list) == 2
    assert all(list(s.shape) == [3, 1] for s in sublogits_list)
    assert len(subweights_list) == 0


def test_gam_layer_feature_count_errors(gam_api):
  GAM, dev = gam_api
  example_inputs = _t([[1], [0], [-1]], dev)
  context_inputs = _t([[1, 2], [0, 1], [-1, 1]], dev)
  gam = GAM(3, [3, 2, 1], 2, [3, 2, 1])
  with pytest.raises(ValueError):
    gam(([example_inputs], [context_inputs, context_inputs]))
  gam = GAM(1, [3, 2, 1], 2, [3, 2, 1])
  with pytest.raises(ValueError):
    gam(([example_inputs], [context_inputs]))


def test_gam_layer_requires_context_hidden_dims(gam_api):
  GAM, _ = gam_api
  with pytest.raises(ValueError):
    GAM(2, [3], 2, None)


def test_gam_scorer_output_shape(gam_api):
  """model_test.py:436-450."""
  GAM, dev = gam_api
  ctx = {'context_1': _t([[1]], dev)}
  ex = {'feature_1': _t([[[0.], [1], [2]]], dev), 'feature_2': _t([[[0.], [1], [2]]], dev)}
  mask = torch.tensor([[True, True, True]], device=dev)
  if dev.type == 'cpu':
    params = OG.init_gam_params([1, 1], [10, 10], [1], [10, 10])
    out = OG.gam_scorer({k: v.double() for k, v in ctx.items()},
                        {k: v.double() for k, v in ex.items()}, mask, params)
  else:
    import ranking_b200 as tfr
    scorer = tfr.keras.model.GAMScorer(example_hidden_layer_dims=[10, 10],
                                       context_hidden_layer_dims=[10, 10])
    out = scorer(ctx, ex, mask)
  assert list(out.shape) == [1, 3]


def _cfg(_C, dims, hidden, ctx=(), ctx_hidden=(), bn=True):
  cfg = _C.GamCfg()
  cfg.n_features = len(dims)
  o = 0
  for i, d in enumerate(dims):
    o += d
    cfg.feature_offsets[i + 1] = o
  cfg.n_hidden = len(hidden)
  for i, h in enumerate(hidden):
    cfg.hidden[i] = h
  cfg.n_context = len(ctx)
  for j, d in enumerate(ctx):
    cfg.context_dims[j] = d
  cfg.n_context_hidden = len(ctx_hidden)
  for i, h in enumerate(ctx_hidden):
    cfg.context_hidden[i] = h
  cfg.use_batch_norm = int(bn)
  cfg.bn_epsilon = 1e-3
  cfg.bn_momentum = 0.999
  cfg.activation = 1
  return cfg


def test_param_count_validates_config_without_gpu():
  import __graft_entry__ as g
  g.build()
  from ranking_b200 import _C
  count = lambda c: _C.lib.tfr_gam_param_count(ctypes.byref(c))
  # canned-GAM recipe: 136 scalar features, [16, 8], BN
  per = 1 * 16 + 16 + 16 * 8 + 8 + 8 + 1 + 2 * (16 + 8)
  assert count(_cfg(_C, [1] * 136, [16, 8])) == 136 * per
  assert _C.lib.tfr_gam_bn_state_count(ctypes.byref(_cfg(_C, [1] * 136, [16, 8]))) == \
      136 * 2 * 24
  # widths per feature, a context tower (dims [2, 3, F = 2]), no BN, linear GAM
  assert count(_cfg(_C, [1, 3], [], [2], [3], bn=False)) == \
      (1 + 1) + (3 + 1) + (2 * 3 + 3 + 3 * 2 + 2)
  too_deep = _cfg(_C, [1], [4] * 4)
  too_deep.n_hidden = 5
  for bad in (_cfg(_C, [1] * 4, [65]), _cfg(_C, [33], [8]), too_deep,
              _cfg(_C, [1] * 9, [4], [2], [3]), _cfg(_C, [], [4])):
    assert count(bad) == 0 and _C.last_error()
  assert _C.lib.tfr_gam_workspace_bytes(ctypes.byref(_cfg(_C, [1] * 136, [16, 8])),
                                        204800) > 0
