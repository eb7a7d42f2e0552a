"""The gated fp64 tower reference (tests/_tower_fp64.py) on the CPU.

  * It reproduces oracle/scorer.py (tower_forward, autograd, moving statistics) when the
    gates it is handed are the oracle's own, which are unambiguous in fp64.
  * An fp32 evaluation of the same chain stays inside the fp32 bound.
  * Negative controls: each defect the GPU matrix (tests/test_tower_edges_gpu.py) is there to
    catch, injected into a stand-in for a kernel result and sent through the same comparison
    (_tower_fp64.check: gates from the stored activations, their admissibility, then every
    output against its bound), fails it in at least one element.
"""
import math

import pytest
import torch

import _tower_fp64 as R
from oracle import scorer as OS

SMS = 132


def _params(dims, cfg, seed):
  g = torch.Generator().manual_seed(seed)
  p = {'w': [], 'b': [], 'gamma': [], 'beta': []}
  for i in range(len(dims) - 1):
    lim = math.sqrt(6.0 / (dims[i] + dims[i + 1]))
    p['w'].append((torch.rand(dims[i], dims[i + 1], generator=g, dtype=torch.float64) * 2 - 1)
                  * lim)
    p['b'].append(torch.rand(dims[i + 1], generator=g, dtype=torch.float64) * 0.4 - 0.2)
  if cfg.use_bn:
    for n in dims[1:-1]:
      p['gamma'].append(torch.rand(n, generator=g, dtype=torch.float64) + 0.5)
      p['beta'].append(torch.rand(n, generator=g, dtype=torch.float64) * 0.4 - 0.2)
  if cfg.input_bn:
    p['in_gamma'] = torch.rand(dims[0], generator=g, dtype=torch.float64) + 0.5
    p['in_beta'] = torch.rand(dims[0], generator=g, dtype=torch.float64) * 0.4 - 0.2
  moving = {}
  keys = (['input'] if cfg.input_bn else []) + (list(range(cfg.L)) if cfg.use_bn else [])
  for k in keys:
    n = dims[0] if k == 'input' else dims[k + 1]
    moving[k] = (torch.randn(n, generator=g, dtype=torch.float64) * 0.1,
                 torch.rand(n, generator=g, dtype=torch.float64) + 0.5)
  return p, moving


def _oracle(x, p, cfg, moving, ds, mask, keep, monkeypatch):
  """oracle.scorer.tower_forward + autograd; returns (scores, flat grads, dx, moving after,
  hidden activations H_d)."""
  leaves = {'w': [w.clone().requires_grad_() for w in p['w']],
            'b': [b.clone().requires_grad_() for b in p['b']],
            'gamma': [t.clone().requires_grad_() for t in p['gamma']],
            'beta': [t.clone().requires_grad_() for t in p['beta']]}
  op = {'dense_w': leaves['w'], 'dense_b': leaves['b'], 'bn_gamma': leaves['gamma'],
        'bn_beta': leaves['beta'], 'in_bn_gamma': None, 'in_bn_beta': None}
  if cfg.input_bn:
    op['in_bn_gamma'] = p['in_gamma'].clone().requires_grad_()
    op['in_bn_beta'] = p['in_beta'].clone().requires_grad_()
  mv = {k: [a.clone(), b.clone()] for k, (a, b) in moving.items()}
  acts = []
  real_act = OS._act

  def spy(v, activation):
    out = real_act(v, activation)
    acts.append(out)
    return out

  monkeypatch.setattr(OS, '_act', spy)
  xr = x.clone().requires_grad_()
  s = OS.tower_forward(xr, op, activation='relu' if cfg.relu else None,
                       use_batch_norm=cfg.use_bn, input_batch_norm=cfg.input_bn,
                       training=cfg.training, bn_moving=mv, momentum=cfg.momentum,
                       keep_masks=keep)
  monkeypatch.undo()
  if mask is not None and s.shape[1] == 1:
    s = torch.where(mask.reshape(-1, 1), s, torch.full_like(s, R.LOG_EPSILON))
  (s * ds).sum().backward()
  parts = []
  for w, b in zip(leaves['w'], leaves['b']):
    parts += [w.grad.reshape(-1), b.grad]
  if cfg.input_bn:
    parts += [op['in_bn_gamma'].grad, op['in_bn_beta'].grad]
  if cfg.use_bn:
    for g, b in zip(leaves['gamma'], leaves['beta']):
      parts += [g.grad, b.grad]
  hidden = [a * k for a, k in zip(acts, keep)] if keep is not None else acts
  return s.detach(), torch.cat(parts), xr.grad, mv, hidden, acts


ORACLE_CASES = {
    'relu': dict(relu=True),
    'identity_masked': dict(relu=False, masked=True),
    'relu_dropout': dict(relu=True, dropout=0.3),
    'identity_dropout': dict(relu=False, dropout=0.3),
    'bn_train_relu': dict(relu=True, use_bn=True),
    'bn_infer_relu': dict(relu=True, use_bn=True, training=False),
    'bn_train_identity_dropout_inbn': dict(relu=False, use_bn=True, dropout=0.25,
                                           input_bn=True),
    'inbn_infer_identity': dict(relu=False, input_bn=True, training=False),
    'no_hidden_inbn': dict(relu=True, input_bn=True, hidden=[]),
    'o3': dict(relu=True, out=3),
}


@pytest.mark.parametrize('name', sorted(ORACLE_CASES))
def test_reference_matches_oracle(name, monkeypatch):
  kw = dict(ORACLE_CASES[name])
  hidden, out = kw.pop('hidden', [24, 16]), kw.pop('out', 1)
  masked = kw.pop('masked', False)
  dims = [12] + hidden + [out]
  cfg = R.Cfg(dims, momentum=0.9, **kw)
  m = 70
  p, moving = _params(dims, cfg, seed=len(name))
  g = torch.Generator().manual_seed(7)
  x = torch.randn(m, dims[0], generator=g, dtype=torch.float64)
  ds = torch.randn(m, out, generator=g, dtype=torch.float64)
  mask = torch.rand(m, generator=g) > 0.2 if masked else None
  keep = None
  if cfg.drop_active:
    keep = [(torch.rand(m, n, generator=g) >= cfg.dropout).double() / (1 - cfg.dropout)
            for n in hidden]
  s, grads, dx, mv, hs, acts = _oracle(x, p, cfg, moving, ds, mask, keep, monkeypatch)
  if cfg.relu:   # no pre-activation near a ReLU kink: the oracle's gates are unambiguous
    for a in acts:
      assert a[a > 0].min() > 1e-9
  gates = R.gates_from(hs, cfg)
  ref = R.forward_backward(x, p, cfg, gates, ds, mask, moving)
  close = lambda a, b: torch.allclose(a, b, rtol=1e-12, atol=1e-12)
  assert close(ref['scores'], s)
  assert close(ref['grads'], grads)
  if cfg.L > 0 and not cfg.input_bn:
    assert close(ref['dx'], dx)
  if cfg.training:
    for k, (a, b) in ref['moving'].items():
      assert close(a, mv[k][0]) and close(b, mv[k][1]), k
  assert set(ref['moving']) == (set(moving) if cfg.training else set())
  # magnitudes bound the exact values they stand for (a masked row's fill is exact: mag 0)
  live = torch.ones(m, dtype=torch.bool) if mask is None or out > 1 else mask
  assert (ref['mag']['scores'][live] >= ref['scores'][live].abs() * (1 - 1e-12)).all()
  assert (ref['mag']['grads'] >= ref['grads'].abs() * (1 - 1e-12)).all()


@pytest.mark.parametrize('use_bn,training', [(False, True), (True, True), (True, False)])
def test_fp32_chain_inside_fp32_bound(use_bn, training):
  """An fp32 evaluation of the same chain (CPU BLAS, its own summation order, ReLU decided on
  its own rounded values) is a stand-in for a correct fp32 kernel: it must pass the whole
  comparison, gate admissibility included."""
  cfg = R.Cfg([40, 96, 64, 2], relu=True, use_bn=use_bn, input_bn=use_bn, training=training,
              momentum=0.9)
  m, dims = 600, cfg.dims
  p, moving = _params(dims, cfg, 3)
  g = torch.Generator().manual_seed(4)
  x = torch.randn(m, dims[0], generator=g, dtype=torch.float64).float().double()
  ds = torch.randn(m, dims[-1], generator=g, dtype=torch.float64).float().double()
  p = {k: [t.float().double() for t in v] if isinstance(v, list) else v.float().double()
       for k, v in p.items()}
  moving = {k: (a.float().double(), b.float().double()) for k, (a, b) in moving.items()}
  ones = [torch.ones(m, n, dtype=torch.float64) for n in dims[1:-1]]
  gates = []
  for d in range(cfg.L):   # layer by layer: each gate depends on the ones before it
    y = R.forward_backward(x, p, cfg, gates + ones[d:], ds, None, moving,
                           dtype=torch.float32)['Y'][d]
    gates.append((y > 0).double())
  run = R.forward_backward(x, p, cfg, gates, ds, None, moving, dtype=torch.float32)
  got = {'hidden': run['A'][1:], 'scores': run['scores'], 'grads': run['grads'],
         'moving': run['moving'], 'dx': [] if cfg.input_bn else [(0, dims[0], run['dx'])]}
  ratios = dict(R.check(cfg, 'fp32', R.Plan(cfg, m, SMS), x, p, ds, got, moving=moving))
  print('fp32 chain:', {k: '%.3g' % v for k, v in ratios.items()})
  assert all(r <= 1 for r in ratios.values()), ratios
  assert ratios['scores'] > 0 and ratios['grads'] > 0
  assert len(ratios) == 3 + cfg.L + 2 * len(run['moving']) + len(got['dx'])


# ------------------------------------------------------------------ negative controls ---
NEG_DIMS = [136, 128, 128, 3]
NEG_M = 300
NEG_SEED = (1234 << 32) | 5     # a dropout seed as Tower._run_cfg forms it
# k block of the Dense GEMMs: the SGEMM's BK (mlp_simt.cu), the wgmma engine's (wgmma_gemm.cuh)
K_BLOCK = {'fp32': 8, 'tf32x3': 32, 'tf32': 32}


def _kernel_standin(x, p, cfg, ds, corrupt=None):
  """What a correct kernel returns, up to rounding: the exact chain under its own gates (the
  sign of each exact Y_d and the replayed dropout stream).  corrupt(d, gate) may change layer
  d's gate before the next layer is computed: the defect under test.  Returns the `got` dict
  of _tower_fp64.check, and the run itself."""
  m = x.shape[0]
  ones = [torch.ones(m, n, dtype=torch.float64) for n in cfg.dims[1:-1]]
  gates = []
  for d in range(cfg.L):
    y = R.forward_backward(x, p, cfg, gates + ones[d:], ds)['Y'][d]
    keep = torch.ones_like(y, dtype=torch.bool)
    if cfg.drop_active:
      keep = R.dropout_keep(NEG_SEED, d, m, y.shape[1], cfg.dropout)
    g = (keep & (y > 0) if cfg.relu else keep).double()
    gates.append(corrupt(d, g) if corrupt else g)
  run = R.forward_backward(x, p, cfg, gates, ds)
  got = {'hidden': run['A'][1:], 'scores': run['scores'], 'grads': run['grads'],
         'dx': [(0, cfg.dims[0], run['dx'])]}
  return got, run


def _neg_setup(precision, **kw):
  cfg = R.Cfg(NEG_DIMS, **kw)
  p, _ = _params(NEG_DIMS, cfg, seed=21)
  g = torch.Generator().manual_seed(22)
  x = torch.randn(NEG_M, NEG_DIMS[0], generator=g, dtype=torch.float64)
  ds = torch.randn(NEG_M, NEG_DIMS[-1], generator=g, dtype=torch.float64)
  plan = R.Plan(cfg, NEG_M, SMS)

  def worst(got):
    return max(r for _, r in R.check(cfg, precision, plan, x, p, ds, got,
                                     dropout_seed=NEG_SEED))

  return cfg, p, x, ds, plan, worst


def _zero_corner(layer):
  """One 8-column corner (8 x 8) of the first 128 x 128 output tile of H_layer never stored."""
  def corrupt(d, g):
    if d == layer:
      g = g.clone()
      g[120:128, 120:128] = 0
    return g
  return corrupt


@pytest.mark.parametrize('precision', sorted(K_BLOCK))
def test_negative_controls_exceed_bound(precision):
  """Each defect goes through the same pipeline as a kernel result on the GPU: gates derived
  from the (corrupted) stored activations, then every comparison of _tower_fp64.check."""
  cfg, p, x, ds, plan, worst = _neg_setup(precision, relu=True)
  got, run = _kernel_standin(x, p, cfg, ds)
  assert worst(got) == 0
  ratios = {}

  # one row missing from one row split of dW_1 (the last row of the first split)
  row = min(plan.rows_per_split, NEG_M) - 1
  dw = torch.outer(run['A'][1][row], run['dz'][1][row])
  off = NEG_DIMS[0] * 128 + 128
  bad = dict(got, grads=got['grads'].clone())
  bad['grads'][off:off + dw.numel()] -= dw.reshape(-1)
  ratios['dW row'] = worst(bad)

  ratios['tile corner'] = worst(_kernel_standin(x, p, cfg, ds, _zero_corner(0))[0])

  # a whole 128 x 128 tile of H_1 never stored
  def zero_tile(d, g):
    return g * 0 if d == 1 else g
  ratios['zero tile'] = worst(_kernel_standin(x, p, cfg, ds, zero_tile)[0])

  # the last k block of layer 1's forward dropped
  p2 = dict(p, w=[w.clone() for w in p['w']])
  p2['w'][1][-K_BLOCK[precision]:] = 0
  ratios['k block'] = worst(_kernel_standin(x, p2, cfg, ds)[0])

  # layer 1 gated with layer 0's mask
  gates0 = []

  def wrong_layer(d, g):
    gates0.append(g)
    return gates0[0] if d == 1 else g
  ratios['wrong gates'] = worst(_kernel_standin(x, p, cfg, ds, wrong_layer)[0])

  # output units 0 and 1 swapped
  ratios['swapped units'] = worst(dict(got, scores=got['scores'][:, [1, 0, 2]]))

  print(precision, {k: '%.3g' % v for k, v in ratios.items()})
  for k, v in ratios.items():
    assert v > 1, (k, v)


@pytest.mark.parametrize('relu', [True, False])
@pytest.mark.parametrize('precision', sorted(K_BLOCK))
def test_negative_controls_with_dropout(precision, relu):
  """With dropout the gates also hold the dropped elements: zeros written where the stream
  keeps, or another stream, are inadmissible gates."""
  cfg, p, x, ds, plan, worst = _neg_setup(precision, relu=relu, dropout=0.3)
  got, _ = _kernel_standin(x, p, cfg, ds)
  assert worst(got) == 0
  ratios = {'tile corner': worst(_kernel_standin(x, p, cfg, ds, _zero_corner(0))[0])}
  m, n = NEG_M, NEG_DIMS[1]
  other = R.dropout_keep(NEG_SEED + 1, 0, m, n, cfg.dropout).double()
  ratios['other stream'] = worst(_kernel_standin(
      x, p, cfg, ds, lambda d, g: g * other / other.clamp(min=1) if d == 0 else g)[0])
  print(precision, relu, {k: '%.3g' % v for k, v in ratios.items()})
  for k, v in ratios.items():
    assert v > 1, (k, v)


def test_identity_zero_corner_exceeds_bound():
  """Without ReLU or dropout every gate is 1, so zeros in H show in the H comparison itself."""
  cfg, p, x, ds, plan, worst = _neg_setup('fp32', relu=False)
  assert worst(_kernel_standin(x, p, cfg, ds)[0]) == 0
  assert worst(_kernel_standin(x, p, cfg, ds, _zero_corner(0))[0]) > 1


def test_dropout_stream_rate():
  """dropout_keep keeps about 1 - p of the elements and differs between layers and seeds."""
  a = R.dropout_keep(NEG_SEED, 0, 500, 200, 0.3)
  b = R.dropout_keep(NEG_SEED, 1, 500, 200, 0.3)
  c = R.dropout_keep(NEG_SEED + 1, 0, 500, 200, 0.3)
  assert abs(a.double().mean().item() - 0.7) < 0.01
  assert (a != b).double().mean().item() > 0.3 and (a != c).double().mean().item() > 0.3
