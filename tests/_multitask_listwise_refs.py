"""fp64 restatement of multi-task DASALC (tfr_dasalc_fwd_tasks / _bwd_tasks, include/tfr_b200.h):
_dasalc_refs.py's scorer with a [W, T] output layer.  Everything before the output layer is
shared by the tasks, so task u's plane is _dasalc_refs.forward over the single-task parameter
vector that holds w_o[:, u] and b_o[u]; the vectors are views of one fp64 leaf, so autograd
gives the [W, T] gradient.  Test infrastructure only."""
import numpy as np
import torch

import _dasalc_refs as ref


def _head(d, w, h):
  """(offset of w_o, count of the parameters after b_o) in the single-task layout."""
  off = 0
  for name, shape in ref.param_shapes(d, w, h):
    if name == 'wo':
      break
    off += int(np.prod(shape))
  return off, ref.param_count(d, w, h) - off - w - 1


def param_count(d, w, h, t):
  return ref.param_count(d, w, h) + (w + 1) * (t - 1)


def task_flat(flat, d, w, h, t, u):
  """The single-task parameter vector of task u (a differentiable function of `flat`)."""
  o, tail = _head(d, w, h)
  wo = flat[o:o + w * t].reshape(w, t)[:, u]
  bo = flat[o + w * t + u:o + w * t + u + 1]
  return torch.cat([flat[:o], wo, bo, flat[o + w * t + t:]])


def single_to_tasks(flats, d, w, h):
  """The T-task vector whose task u is the single-task vector flats[u] (which must agree
  everywhere but w_o, b_o)."""
  o, _ = _head(d, w, h)
  wo = torch.stack([f[o:o + w] for f in flats], 1).reshape(-1)
  bo = torch.cat([f[o + w:o + w + 1] for f in flats])
  return torch.cat([flats[0][:o], wo, bo, flats[0][o + w + 1:]])


def forward_tasks(x, e, flat, d, w, h, t, **kw):
  """-> (planes [T, M], batch stats of the shared layers); kw as _dasalc_refs.forward."""
  planes, stats = [], None
  for u in range(t):
    s, st = ref.forward(x, e, task_flat(flat, d, w, h, t, u), d, w, h, **kw)
    planes.append(s)
    stats = stats if stats is not None else st
  return torch.stack(planes), stats


def block_errors(got, want, d, w, h, t):
  """{name: relative L2 error} of every parameter block ('wo' is the whole [W, T] block, 'bo'
  the [T] one); a block whose reference is exactly 0 counts its absolute error."""
  got, want = got.double().reshape(-1), want.double().reshape(-1).to(got.device)
  o, _ = _head(d, w, h)
  shared_g = torch.cat([got[:o], got[o + w * t + t:]])
  shared_w = torch.cat([want[:o], want[o + w * t + t:]])
  pad = torch.zeros(w + 1, dtype=got.dtype, device=got.device)
  out = ref.block_errors(torch.cat([shared_g[:o], pad, shared_g[o:]]),
                         torch.cat([shared_w[:o], pad, shared_w[o:]]), d, w, h)
  for name, a, b in (('wo', got[o:o + w * t], want[o:o + w * t]),
                     ('bo', got[o + w * t:o + w * t + t], want[o + w * t:o + w * t + t])):
    bn = float(b.norm())
    out[name] = float((a - b).norm() / bn) if bn > 0 else float((a - b).norm())
  return out
