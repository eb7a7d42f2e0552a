"""Multi-task input and pipeline: `data.elwc_multilabel_batches` on records written by
`data.encode_elwc`, `pipeline.MultiTaskPipeline`'s argument checks (CPU), and its
train_and_validate end to end on the GPU (log keys, resume, best checkpoint, early stopping)."""
import os

import pytest
import torch

CTX = {'qf': (2, 0.0)}
EX = {'f': (3, 0.0), 'rel': (1, -1.0), 'w': (1, 1.0), 'click': (1, -1.0)}


def _lib():
  import __graft_entry__ as entry
  entry.build()
  from ranking_b200 import data
  return data


def _records(n_lists, seed=0, n_items=(3, 5)):
  from ranking_b200 import data
  g = torch.Generator().manual_seed(seed)
  recs = []
  for i in range(n_lists):
    k = n_items[i % len(n_items)]
    items = []
    for j in range(k):
      f = torch.randn(3, generator=g).tolist()
      e = {'f': f, 'rel': [float((i + j) % 3)], 'w': [0.5 + j]}
      if j != 1:                       # item 1 has no click label
        e['click'] = [float(j % 2)]
      items.append(e)
    recs.append(data.encode_elwc({'qf': [float(i), 1.0]}, items))
  return recs


def _write(tmp_path, recs, name='a.tfrecord'):
  from ranking_b200 import data
  path = os.path.join(str(tmp_path), name)
  data.write_tfrecords(path, recs)
  return path


def test_multilabel_batches(tmp_path):
  data = _lib()
  path = _write(tmp_path, _records(5))
  out = list(data.elwc_multilabel_batches(path, 2, 4, CTX, EX,
                                          {'relevance': 'rel', 'click': 'click'},
                                          sample_weight_feature='w', drop_remainder=False,
                                          pin_memory=False))
  assert len(out) == 3
  x, labels, mask, w = out[0]
  assert x.shape == (2, 4, 2 + 3)           # label and weight columns removed
  assert list(labels) == ['relevance', 'click']
  # list 0 has 3 items, list 1 has 4 of its 5 (truncated to list_size)
  assert mask.tolist() == [[True, True, True, False], [True, True, True, True]]
  assert labels['relevance'][0].tolist() == [0.0, 1.0, 2.0, -1.0]
  assert labels['relevance'][1].tolist() == [1.0, 2.0, 0.0, 1.0]
  assert labels['click'][0].tolist() == [0.0, -1.0, 0.0, -1.0]
  assert w[0, :3].tolist() == [0.5, 1.5, 2.5]
  assert x[0, 0, :2].tolist() == [0.0, 1.0] and x[1, 2, :2].tolist() == [1.0, 1.0]
  # the example features are f, in order
  ref = data.parse_from_example_list(_records(5)[:2], 4, CTX, EX)
  assert torch.equal(x[..., 2:], ref['examples'][..., 0:3])
  # without a weight feature: weights None, the weight column stays in x
  x2, _, _, w2 = next(data.elwc_multilabel_batches(path, 2, 4, CTX, EX, {'r': 'rel'},
                                                   pin_memory=False))
  assert w2 is None and x2.shape == (2, 4, 2 + 3 + 1 + 1)
  with pytest.raises(ValueError):
    next(data.elwc_multilabel_batches(path, 2, 4, CTX, EX, {'r': 'nope'}))
  with pytest.raises(ValueError):
    next(data.elwc_multilabel_batches(path, 2, 4, CTX, EX, {'r': 'f'}))
  with pytest.raises(ValueError):
    next(data.elwc_multilabel_batches(path, 2, 4, CTX, EX, {'r': 'rel'},
                                      sample_weight_feature='rel'))


def _hp(tmp_path, **kw):
  from ranking_b200 import pipeline
  base = dict(model_dir=str(tmp_path), num_epochs=3, steps_per_epoch=2, validation_steps=1,
              learning_rate=0.05, loss={'relevance': 'softmax_loss',
                                        'click': 'sigmoid_cross_entropy_loss'})
  base.update(kw)
  return pipeline.PipelineHparams(**base)


def test_pipeline_argument_errors(tmp_path):
  _lib()
  from ranking_b200 import pipeline
  mk = lambda **kw: pipeline.MultiTaskPipeline(None, None, None, _hp(tmp_path, **kw))
  with pytest.raises(ValueError, match='dict'):
    mk(loss='softmax_loss')
  with pytest.raises(ValueError, match='unknown tasks'):
    mk(loss_weights={'buy': 1.0})
  with pytest.raises(ValueError, match='loss_weights'):
    mk(loss_weights=0.5)
  with pytest.raises(ValueError, match='optimizer'):
    mk(optimizer='adam')
  with pytest.raises(ValueError, match='at most 8'):
    mk(loss={str(i): 'softmax_loss' for i in range(9)})
  p = mk(loss_weights={'click': 2.0})
  assert p.tasks == ['relevance', 'click']
  # the single-task hparams check still refuses loss maps
  with pytest.raises(ValueError):
    _hp(tmp_path).validate()


@pytest.mark.gpu
def test_train_and_validate(tmp_path):
  if not torch.cuda.is_available():
    pytest.skip('no CUDA device')
  data = _lib()
  import ranking_b200 as tfr
  from ranking_b200 import pipeline
  path = _write(tmp_path, _records(16, n_items=(3, 5, 4)))
  labels = {'relevance': 'rel', 'click': 'click'}

  def batches():
    return data.elwc_multilabel_batches(path, 4, 4, CTX, EX, labels, sample_weight_feature='w')

  def tower_fn():
    return tfr.keras.layers.create_tower([16], 2, activation='relu', use_batch_norm=False,
                                         input_dim=5, seed=1, precision='fp32')

  logs_seen = []
  hp = _hp(os.path.join(str(tmp_path), 'run'), use_weighted_metrics=True,
           loss_weights={'click': 0.5}, export_best_model=True,
           best_exporter_metric='relevance_metric/ndcg_5',
           best_exporter_metric_higher_better=True)
  p = pipeline.MultiTaskPipeline(tower_fn, batches, batches, hp, log_fn=logs_seen.append)
  hist = p.train_and_validate(verbose=1)
  assert len(hist) == 3 and len(logs_seen) == 3
  keys = {'epoch', 'step', 'train_loss', 'loss'}
  for t in ('relevance', 'click'):
    keys.add(t + '_loss')
    for kind in ('_metric/', '_weighted_metric/'):
      keys.update(t + kind + k for k in ('ndcg_1', 'ndcg_5', 'ndcg_10', 'ndcg'))
  assert set(hist[-1]) == keys
  for h in hist:
    assert abs(h['loss'] - (h['relevance_loss'] + 0.5 * h['click_loss'])) < 1e-9
  assert os.path.exists(os.path.join(hp.model_dir, 'best_checkpoint', 'ckpt.pt'))
  flat = p.trainer.tower.flat.detach().clone()

  # resume: a fresh pipeline over the same model_dir finds all epochs done
  p2 = pipeline.MultiTaskPipeline(tower_fn, batches, batches, hp, log_fn=logs_seen.append)
  assert p2.train_and_validate() == []
  assert torch.equal(p2.trainer.tower.flat, flat)

  # early stopping: a metric that never improves stops after `patience` epochs
  hp3 = _hp(os.path.join(str(tmp_path), 'stop'), num_epochs=6, learning_rate=0.0,
            early_stopping_patience=2)
  p3 = pipeline.MultiTaskPipeline(tower_fn, batches, batches, hp3)
  assert len(p3.train_and_validate()) == 3
