"""The scorer part of `tfr.keras.model` (keras/model.py:668-865): `Scorer`,
`UnivariateScorer`, `DNNScorer`, `GAMScorer`.

`scorer(context_features, example_features, mask) -> [batch_size, list_size]`
with `context_features: {name: [B, Dc]}`, `example_features: {name: [B, N, Dk]}`,
`mask: [B, N]` bool, exactly the reference call contract (keras/model.py:690-710).
Features are concatenated context-first, each group in sorted key order
(keras/model.py:806-814).
"""
import abc

import torch

from ranking_b200.keras import layers


class Scorer(torch.nn.Module, metaclass=abc.ABCMeta):
  """keras/model.py:668-710."""

  @abc.abstractmethod
  def forward(self, context_features, example_features, mask):
    raise NotImplementedError('Calling an abstract method.')


class UnivariateScorer(Scorer, metaclass=abc.ABCMeta):
  """keras/model.py:713-777."""

  def __init__(self):
    super().__init__()
    self._flatten = layers.FlattenList()
    self._restore = layers.RestoreList()

  @abc.abstractmethod
  def _score_flattened(self, context_features, example_features):
    raise NotImplementedError('Calling an abstract method.')

  def forward(self, context_features, example_features, mask):
    flat_ctx, flat_ex = self._flatten((context_features, example_features, mask))
    flattened_logits = self._score_flattened(flat_ctx, flat_ex)
    if isinstance(flattened_logits, dict):
      return {k: self._restore((v, mask)) for k, v in flattened_logits.items()}
    return self._restore((flattened_logits, mask))


class DNNScorer(UnivariateScorer):
  """keras/model.py:780-817: `DNNScorer(**create_tower kwargs)`."""

  def __init__(self, **dnn_kwargs):
    super().__init__()
    self._dnn_kwargs = dnn_kwargs
    self.tower = None

  def _score_flattened(self, context_features, example_features):
    cols = [context_features[k].reshape(context_features[k].shape[0], -1)
            for k in sorted(context_features)]
    cols += [example_features[k].reshape(example_features[k].shape[0], -1)
             for k in sorted(example_features)]
    input_layer = cols[0] if len(cols) == 1 else torch.cat(cols, 1)
    if self.tower is None:   # built at first call, like a Keras layer
      kw = dict(self._dnn_kwargs)
      kw['input_dim'] = input_layer.shape[1]
      self.tower = layers.create_tower(**kw)
    return self.tower(input_layer)


class GAMScorer(UnivariateScorer):
  """keras/model.py:820-865: `GAMScorer(**GAMLayer kwargs)`.  Both feature counts come
  from the inputs; every feature is flattened and features go in sorted key order."""

  def __init__(self, **gam_kwargs):
    super().__init__()
    self._gam_kwargs = gam_kwargs
    self.gam = None

  def _score_flattened(self, context_features, example_features):
    context_inputs = [context_features[k].reshape(context_features[k].shape[0], -1)
                      for k in sorted(context_features)]
    example_inputs = [example_features[k].reshape(example_features[k].shape[0], -1)
                      for k in sorted(example_features)]
    if self.gam is None:   # built at first call, like a Keras layer
      kw = dict(self._gam_kwargs)
      kw.update(example_feature_num=len(example_inputs),
                context_feature_num=len(context_inputs))
      self.gam = layers.GAMLayer(**kw)
    logits, _, _ = self.gam((example_inputs, context_inputs))
    return logits
