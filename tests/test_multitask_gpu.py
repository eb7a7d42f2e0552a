"""MultiTaskRankingTrainer on the GPU: the fused multi-task step against an fp64 oracle
composition (oracle/scorer.py tower, RestoreList per task, oracle/keras_losses per task, the
weighted sum, autograd, Adagrad); one task reproducing RankingTrainer bit for bit; predict's
per-task planes; checkpoint resume."""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu

B, N, D = 16, 24, 12


@pytest.fixture(autouse=True)
def _need_cuda():
  if not torch.cuda.is_available():
    pytest.skip('no CUDA device')


def _tfr():
  import __graft_entry__ as entry
  entry.build()
  import ranking_b200 as tfr
  return tfr


def _data(seed, tasks, partial=True):
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(B, N, D, generator=g)
  labels = {}
  pad = torch.zeros(B, N, dtype=torch.bool)
  pad[:, N - 5:] = True
  pad[3, 4:] = True
  for i, t in enumerate(tasks):
    y = torch.randint(0, 3, (B, N), generator=g).float()
    if i % 2:
      y = (y > 1).float()       # a binary task (clicks)
    y[pad] = -1.0
    if partial and i == 1:      # items that carry only the other task's label
      y[:, 0:2] = -1.0
    labels[t] = y
  weight = torch.rand(B, N, generator=g) + 0.5
  return x, labels, weight


def _oracle_step(tower, loss_names, weights, x, labels, sample_weight, accum, lr):
  from oracle import keras_losses as OL
  from oracle import scorer as OS
  L = len(tower.dims) - 1
  params = {'dense_w': [tower.kernel(i).detach().cpu().double().clone().requires_grad_()
                        for i in range(L)],
            'dense_b': [tower.bias(i).detach().cpu().double().clone().requires_grad_()
                        for i in range(L)]}
  tasks = list(labels)
  mask = torch.zeros(B, N, dtype=torch.bool)
  for t in tasks:
    mask |= labels[t] >= 0
  out = OS.tower_forward(x.double().reshape(B * N, D), params, activation='relu')
  cls = {'softmax_loss': OL.SoftmaxLoss, 'pairwise_logistic_loss': OL.PairwiseLogisticLoss,
         'approx_ndcg_loss': OL.ApproxNDCGLoss,
         'sigmoid_cross_entropy_loss': OL.SigmoidCrossEntropyLoss,
         'mean_squared_loss': OL.MeanSquaredLoss}
  total = 0.0
  per_task = []
  for i, t in enumerate(tasks):
    logits = OS.restore_list(out[:, i], mask)
    sw = None if sample_weight is None else sample_weight.double()
    lt = cls[loss_names[t]]()(labels[t].double(), logits, sw)
    per_task.append(lt)
    total = total + weights.get(t, 1.0) * lt
  total.backward()
  grads = torch.cat([torch.cat([w.grad.reshape(-1), b.grad.reshape(-1)])
                     for w, b in zip(params['dense_w'], params['dense_b'])])
  flat = tower.flat.detach().cpu().double()
  acc = accum.cpu().double() + grads * grads
  new = flat - lr * grads / (acc.sqrt() + 1e-7)
  return float(total.detach()), [float(v.detach()) for v in per_task], grads, new, mask


def _tower(tfr, precision, out, seed=5):
  t = tfr.keras.layers.create_tower([32, 16], out, activation='relu', use_batch_norm=False,
                                    dropout=0, input_dim=D, seed=seed, precision=precision)
  g = torch.Generator().manual_seed(seed)   # equal seeds give equal towers
  with torch.no_grad():
    for i in range(len(t.dims) - 1):
      t.bias(i).copy_(torch.rand(t.dims[i + 1], generator=g) * 0.2 - 0.1)
  return t


LOSS_SETS = [
    {'rel': 'softmax_loss', 'click': 'pairwise_logistic_loss'},
    {'rel': 'approx_ndcg_loss', 'click': 'sigmoid_cross_entropy_loss',
     'buy': 'mean_squared_loss'},
]


@pytest.mark.parametrize('weighted', [False, True])
@pytest.mark.parametrize('set_id', [0, 1])
@pytest.mark.parametrize('precision', ['fp32', 'tf32x3'])
def test_step_against_oracle(precision, set_id, weighted):
  tfr = _tfr()
  names = LOSS_SETS[set_id]
  tasks = list(names)
  loss_weights = {'rel': 1.0, 'click': 0.5} if set_id == 0 else {'click': 3.0, 'buy': 0.25}
  tower = _tower(tfr, precision, len(tasks))
  losses = {t: tfr.keras.losses.get(names[t]) for t in tasks}
  tr = tfr.train.MultiTaskRankingTrainer(tower, losses, loss_weights=loss_weights,
                                         optimizer='adagrad', learning_rate=0.05)
  x, labels, w = _data(11 + set_id, tasks)
  sw = w if weighted else None
  accum0 = tr.accum.clone()
  ref_total, ref_tasks, ref_grads, ref_new, mask = _oracle_step(
      tower, names, loss_weights, x, labels, sw, accum0, 0.05)
  got = tr.train_step(x.cuda(), {t: y.cuda() for t, y in labels.items()},
                      sample_weight=None if sw is None else sw.cuda())
  torch.cuda.synchronize()
  assert got.dim() == 0
  assert abs(float(got) - ref_total) <= 1e-5 * max(1.0, abs(ref_total)), (float(got), ref_total)
  for v, r in zip(tr.task_losses.tolist(), ref_tasks):
    assert abs(v - r) <= 1e-5 * max(1.0, abs(r)), (v, r)
  err = (tr.grads.cpu().double() - ref_grads).abs().max() / ref_grads.abs().max()
  assert float(err) < 1e-4, float(err)
  perr = (tower.flat.detach().cpu().double() - ref_new).abs().max()
  assert float(perr) < 1e-5, float(perr)
  # every plane holds RestoreList's fill where no task has a label
  for i in range(len(tasks)):
    assert (tr.scores[i].cpu()[~mask] == -23.025850929940457).all()


@pytest.mark.parametrize('precision', ['fp32', 'tf32x3', 'tf32'])
def test_one_task_is_ranking_trainer(precision):
  tfr = _tfr()
  t1, t2 = _tower(tfr, precision, 1), _tower(tfr, precision, 1)
  a = tfr.train.RankingTrainer(t1, tfr.keras.losses.get('softmax_loss'), learning_rate=0.05)
  b = tfr.train.MultiTaskRankingTrainer(t2, {'rel': tfr.keras.losses.get('softmax_loss')},
                                        loss_weights={'rel': 1.0}, learning_rate=0.05)
  for step in range(3):
    x, labels, w = _data(20 + step, ['rel'])
    xd, yd, wd = x.cuda(), labels['rel'].cuda(), w.cuda()
    mask = yd >= 0
    la = a.train_step(xd, yd, sample_weight=wd, mask=mask)
    lb = b.train_step(xd, {'rel': yd}, sample_weight=wd, mask=mask)
    torch.cuda.synchronize()
    assert torch.equal(la, lb), step
    assert torch.equal(a.scores, b.scores[0]), step
    assert torch.equal(a.grads, b.grads), step
    assert torch.equal(t1.flat, t2.flat), step
    assert torch.equal(a.accum, b.accum), step


def test_predict_and_resume(tmp_path):
  tfr = _tfr()
  from ranking_b200 import pipeline
  tasks = ['rel', 'click']

  def make():
    tower = _tower(tfr, 'tf32x3', 2)
    return tfr.train.MultiTaskRankingTrainer(
        tower, {'rel': tfr.keras.losses.get('softmax_loss'),
                'click': tfr.keras.losses.get('sigmoid_cross_entropy_loss')},
        loss_weights={'click': 2.0}, learning_rate=0.05)

  batches = [_data(40 + i, tasks) for i in range(4)]

  def step(tr, i):
    x, labels, _ = batches[i]
    return tr.train_step(x.cuda(), {t: y.cuda() for t, y in labels.items()})

  a = make()
  for i in range(4):
    step(a, i)
  b = make()
  for i in range(2):
    step(b, i)
  path = os.path.join(str(tmp_path), 'ckpt.pt')
  pipeline.save_checkpoint(b, path, 2)
  c = make()
  assert pipeline.load_checkpoint(c, path) == 2
  for i in range(2, 4):
    step(c, i)
  torch.cuda.synchronize()
  assert torch.equal(a.tower.flat, c.tower.flat)
  assert torch.equal(a.accum, c.accum)

  x, labels, _ = batches[0]
  ld = {t: y.cuda() for t, y in labels.items()}
  out = a.predict(x.cuda(), labels=ld)
  assert list(out) == tasks
  mask = (ld['rel'] >= 0) | (ld['click'] >= 0)
  for i, t in enumerate(tasks):
    assert out[t].shape == (B, N)
    assert (out[t][~mask] == -23.025850929940457).all()
    assert torch.isfinite(out[t][mask]).all()
  # the planes are tfr_mlp_fwd's columns on valid items
  flat = a.tower(x.cuda().reshape(B * N, D)).reshape(B, N, 2)
  for i, t in enumerate(tasks):
    assert torch.equal(out[t][mask], flat[..., i][mask])


def test_constructor_errors():
  tfr = _tfr()
  L = tfr.keras.losses
  tower = _tower(tfr, 'tf32x3', 2)
  ok = {'rel': L.get('softmax_loss'), 'click': L.get('sigmoid_cross_entropy_loss')}
  with pytest.raises(ValueError, match='unknown tasks'):
    tfr.train.MultiTaskRankingTrainer(tower, ok, loss_weights={'buy': 1.0})
  with pytest.raises(ValueError, match='output units'):
    tfr.train.MultiTaskRankingTrainer(tower, {'rel': L.get('softmax_loss')})
  with pytest.raises(ValueError, match='at most 8'):
    tfr.train.MultiTaskRankingTrainer(tower, {str(i): L.get('softmax_loss') for i in range(9)})
  for bad in (L.ClickEMLoss(), L.MixtureEMLoss(), L.OrdinalLoss(), L.CoupledRankDistilLoss()):
    with pytest.raises(ValueError, match='fused step'):
      tfr.train.MultiTaskRankingTrainer(tower, {'rel': L.get('softmax_loss'), 'x': bad})


def test_recovery(tmp_path):
  """The oracle experiment of test_golden_multitask.py on the fused trainers: each task's plane
  of one two-task tower ranks its task at least DELTA better (NDCG@5) than a model trained on
  the other task's labels alone, and reaches FLOOR."""
  import _multitask_refs as MR
  from test_golden_multitask import DELTA, FLOOR
  tfr = _tfr()
  L = tfr.keras.losses
  batches, (vx, vy) = MR.synthetic(str(tmp_path))

  def tower(out):
    return tfr.keras.layers.create_tower(MR.HIDDEN, out, activation='relu', use_batch_norm=False,
                                         dropout=0, input_dim=MR.D, seed=MR.SEED,
                                         precision='fp32')

  tasks = list(MR.LABELS)
  multi = tfr.train.MultiTaskRankingTrainer(tower(2), {t: L.get(MR.LOSSES[t]) for t in tasks},
                                            learning_rate=MR.LR)
  single = {t: tfr.train.RankingTrainer(tower(1), L.get(MR.LOSSES[t]), learning_rate=MR.LR)
            for t in tasks}
  for _ in range(MR.EPOCHS):
    for x, ys in batches:
      xd, yd = x.cuda(), {t: y.cuda() for t, y in ys.items()}
      multi.train_step(xd, yd)
      for t in tasks:
        single[t].train_step(xd, yd[t])
  xv = vx.cuda()
  planes = {t: s.clone() for t, s in multi.predict(xv).items()}
  others = {t: single[t].predict(xv).clone() for t in tasks}
  for task, (own, other) in MR.margins(planes, others, vy).items():
    print('%s: NDCG@%d %.4f, model of the other task %.4f' % (task, MR.TOP_K, own, other))
    assert own >= FLOOR, (task, own)
    assert own >= other + DELTA, (task, own, other)


def test_example_synthetic(tmp_path):
  """examples/multitask_train.py --synthetic runs end to end and reports both tasks."""
  import subprocess
  import sys
  root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
  out = subprocess.run([sys.executable, os.path.join(root, 'examples', 'multitask_train.py'),
                        '--synthetic', '--work_dir', str(tmp_path),
                        '--model_dir', os.path.join(str(tmp_path), 'model')],
                       capture_output=True, text=True, timeout=600)
  assert out.returncode == 0, out.stderr[-2000:]
  lines = {l.split()[0]: l for l in out.stdout.splitlines() if 'NDCG@5' in l}
  assert set(lines) == {'relevance', 'click'}, out.stdout
  for line in lines.values():
    ndcg5 = float(line.split('NDCG@5')[1].split()[0])
    assert ndcg5 > 0.9, line
