"""Oracle restatement of pooled embedding lookups (K12):

  * tf.feature_column.embedding_column over a categorical column, combiner 'sum' / 'mean' /
    'sqrtn' (feature_column `_safe_embedding_lookup_sparse`: ids of -1 are pruned, an empty
    bag gives zeros, a repeated id counts once per occurrence)
  * the same with Keras Embedding + reduce over the token axis (antique_kpl_din.py:269-278)

Test infrastructure only (see oracle/__init__.py).  Plain torch on the CPU: a gather and a
weighted sum, so autograd gives the table gradient.
"""
import torch


def pool(ids, table, combiner='mean'):
  """ids int [..., T] (-1 = empty slot; every other id must lie in [0, V)), table [V, E]
  -> [..., E]."""
  ids = torch.as_tensor(ids, dtype=torch.int64)
  valid = ids >= 0
  if bool((ids[valid] >= table.shape[0]).any()) or bool((ids < -1).any()):
    raise ValueError('ids outside [-1, V)')
  rows = table[ids.clamp(min=0)]                                   # [..., T, E]
  w = valid.to(table.dtype)
  summed = (rows * w.unsqueeze(-1)).sum(-2)
  count = w.sum(-1, keepdim=True)
  if combiner == 'sum':
    scale = torch.ones_like(count)
  elif combiner == 'mean':
    scale = torch.where(count > 0, 1.0 / count.clamp(min=1), torch.zeros_like(count))
  elif combiner == 'sqrtn':
    scale = torch.where(count > 0, count.clamp(min=1).rsqrt(), torch.zeros_like(count))
  else:
    raise ValueError(combiner)
  return summed * scale


def sequence_embedding(ids, table):
  """sequence_categorical_column + embedding_column (feature_test.py:170-239): one row per
  slot, zeros for -1."""
  ids = torch.as_tensor(ids, dtype=torch.int64)
  valid = (ids >= 0).to(table.dtype).unsqueeze(-1)
  return table[ids.clamp(min=0)] * valid
