"""Shared set-up for the GAM tests (tests/test_gam_gpu.py, tests/test_gam_limits_gpu.py).

A GAMLayer and the fp64 oracle parameters of oracle/gam.py with identical values, seeded
inputs, the oracle's gradient in the layer's flat parameter order, the moving BN statistics
of every tower, and a host replay of the dropout keep mask the GAM kernels draw."""
import numpy as np
import torch

from oracle import gam as OG


def _leaves(p):
  out = []
  for w, b in zip(p['dense_w'], p['dense_b']):
    out += [w, b]
  for g, b in zip(p['bn_gamma'], p['bn_beta']):
    out += [g, b]
  return out


def _pack(p):
  return torch.cat([t.detach().reshape(-1) for t in _leaves(p)])


def _grad(p):
  return torch.cat([t.grad.reshape(-1) if t.grad is not None else torch.zeros(t.numel(),
                                                                           dtype=t.dtype)
                    for t in _leaves(p)])


def _make(tfr, ex_dims, hidden, ctx_dims=(), ctx_hidden=None, act=None, bn=False,
          dropout=0.0, seed=5, momentum=0.999):
  """A built GAMLayer and oracle parameters (fp64, requires_grad) with identical values;
  biases / BN affine parameters are randomised so that every term is exercised."""
  gam = tfr.keras.layers.GAMLayer(len(ex_dims), hidden, len(ctx_dims), ctx_hidden,
                                  activation=act, use_batch_norm=bn,
                                  batch_norm_moment=momentum, dropout=dropout, seed=seed)
  gam.build(ex_dims, list(ctx_dims) or None)
  params = OG.init_gam_params(ex_dims, hidden, ctx_dims, ctx_hidden, use_batch_norm=bn,
                              seed=seed)
  g = torch.Generator().manual_seed(seed)
  towers = params['example'] + params['context']
  for i, p in enumerate(towers):
    for b in p['dense_b']:
      b.uniform_(-0.3, 0.3, generator=g)
    for t in p['bn_gamma']:
      t.uniform_(0.5, 1.5, generator=g)
    for t in p['bn_beta']:
      t.uniform_(-0.3, 0.3, generator=g)
    with torch.no_grad():
      gam.tower_slice(i)[0].copy_(_pack(p).float())
    for t in _leaves(p):
      t.requires_grad_()
  return gam, params


def _moving(gam, params):
  """Moving mean / variance of every BN layer of every tower (fp64 copies)."""
  out = {'example': [], 'context': []}
  for i, _ in enumerate(params['example'] + params['context']):
    _, st, dims = gam.tower_slice(i)
    kind = 'example' if i < len(params['example']) else 'context'
    mv, o = {}, 0
    for d, h in enumerate(dims[1:-1] if st.numel() else []):
      mv[d] = [st[o:o + h].detach().cpu().double().clone(),
               st[o + h:o + 2 * h].detach().cpu().double().clone()]
      o += 2 * h
    out[kind].append(mv)
  return out


def _inputs(m, dims, seed):
  g = torch.Generator().manual_seed(seed)
  return [torch.randn(m, d, generator=g) for d in dims]


def _flat_grad(gam, params):
  return torch.cat([_grad(p) for p in params['example'] + params['context']])


def _keep(seed, layer, m, width, rate):
  """Keep mask [m, width] of hidden layer `layer`: element i is kept unless the kernels'
  uniform draw for (seed, layer, i) falls below `rate`."""
  with np.errstate(over='ignore'):
    s = np.uint64(seed) * np.uint64(0x100000001B3) + np.uint64(layer + 1)
    idx = np.arange(m * width, dtype=np.uint64)
    z = s + np.uint64(0x9E3779B97F4A7C15) * (idx + np.uint64(1))
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    z = z ^ (z >> np.uint64(31))
  u = (z >> np.uint64(40)).astype(np.float32) * np.float32(1.0 / 16777216.0)
  return torch.from_numpy(~(u < np.float32(rate))).reshape(m, width)
