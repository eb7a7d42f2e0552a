"""Oracle restatement of GAMLayer / GAMScorer (keras/layers.py:591-803,
keras/model.py:820-865) from `scorer.tower_forward` plus a softmax.  fp64 and
autograd-able; test infrastructure only (see oracle/__init__.py)."""
import torch

from oracle import scorer


def init_gam_params(example_dims, example_hidden, context_dims=(), context_hidden=None,
                    use_batch_norm=False, seed=7, dtype=torch.float64):
  """{'example': [tower params], 'context': [tower params]} in create_tower order."""
  context_dims = list(context_dims or [])
  if context_dims and not context_hidden:
    raise ValueError('When `context_feature_num` > 0, `context_hidden_layer_dims` is '
                     'required!')
  f = len(example_dims)
  ex = [scorer.init_tower_params(d, example_hidden, 1, seed=seed + i,
                                 use_batch_norm=use_batch_norm, dtype=dtype)
        for i, d in enumerate(example_dims)]
  cx = [scorer.init_tower_params(d, context_hidden, f, seed=seed + 1000 + j,
                                 use_batch_norm=use_batch_norm, dtype=dtype)
        for j, d in enumerate(context_dims)]
  return {'example': ex, 'context': cx}


def gam_layer(example_inputs, context_inputs, params, activation=None,
              use_batch_norm=False, training=True, bn_moving=None, momentum=0.999,
              keep_masks=None):
  """GAMLayer.call: (logits [M, 1], sub_logits_list, sub_weights_list).
  bn_moving / keep_masks: {'example': [per tower], 'context': [per tower]} as
  scorer.tower_forward takes them per tower (or None)."""
  ex_p, cx_p = params['example'], params['context']
  if len(example_inputs) != len(ex_p):
    raise ValueError('Mismatched number of features in `example_inputs` ({}) '
                     'with `example_feature_num` ({})'.format(len(example_inputs), len(ex_p)))
  if context_inputs:
    if not cx_p or len(context_inputs) != len(cx_p):
      raise ValueError('Mismatched number of features in `context_inputs` ({}) '
                       'with `_context_feature_num` ({})'.format(len(context_inputs),
                                                                 len(cx_p)))

  def run(kind, i, x, p):
    return scorer.tower_forward(
        x.reshape(x.shape[0], -1), p, activation=activation, use_batch_norm=use_batch_norm,
        training=training, bn_moving=None if bn_moving is None else bn_moving[kind][i],
        momentum=momentum, keep_masks=None if keep_masks is None else keep_masks[kind][i])

  sub = [run('example', i, x, p) for i, (x, p) in enumerate(zip(example_inputs, ex_p))]
  weights = []
  if context_inputs and cx_p:
    weights = [torch.softmax(run('context', j, c, p), dim=-1)
               for j, (c, p) in enumerate(zip(context_inputs, cx_p))]
  if weights:
    logits = (torch.cat(sub, -1) * sum(weights)).sum(-1, keepdim=True)
  else:
    logits = sum(sub)
  return logits, sub, weights


def gam_scorer(context_features, example_features, mask, params, **gam_kw):
  """UnivariateScorer.__call__ + GAMScorer._score_flattened: features flattened, each
  group in sorted key order."""
  flat_ctx, flat_ex = scorer.flatten_list(context_features, example_features, mask)
  ctx = [flat_ctx[k].reshape(flat_ctx[k].shape[0], -1) for k in sorted(flat_ctx)]
  ex = [flat_ex[k].reshape(flat_ex[k].shape[0], -1) for k in sorted(flat_ex)]
  logits, _, _ = gam_layer(ex, ctx, params, **gam_kw)
  return scorer.restore_list(logits, mask)
