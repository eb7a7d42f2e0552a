"""The groupwise references of tests/_group_refs.py on the CPU.

  * Its rolling-window group formation equals oracle.scorer.form_group_indices (no shuffle) and
    ranking_b200.model._form_group_indices (with caller-supplied permutations) exactly.
  * With exact gates, its fp64 forward and backward equal oracle.scorer.groupwise_logits and
    autograd through it.
  * Negative controls: each defective reference the GPU tests (test_groupwise_limits_gpu.py) must
    reject differs from the true reference by more than the tf32x3 bound somewhere.
"""
import math

import pytest
import torch

import _group_refs as GR
import _tower_fp64 as R
from oracle import scorer as OS

SMS = 132


def _perm(nv, n, g, full):
  """A permutation of the valid-first order: of the whole list (full) or of the valid prefix."""
  if full:
    return torch.randperm(n, generator=g)
  p = torch.arange(n)
  p[:nv] = torch.randperm(nv, generator=g)
  return p


@pytest.mark.parametrize('gs', range(1, 9))
def test_group_formation_matches_oracle_and_model(gs):
  from ranking_b200 import model as M
  g = torch.Generator().manual_seed(gs)
  for n in range(1, 41):
    # one list per valid count 0..N, then random masks
    valid = torch.zeros(n + 1, n, dtype=torch.bool)
    for nv in range(n + 1):
      valid[nv, torch.randperm(n, generator=g)[:nv]] = True
    for s in (1, 2, 3):
      idx, gmask, _, cnt = GR.form_groups(valid, gs, num_shuffles=s)
      # every valid item fills each slot of each shuffle once: cnt = S gs, else 0
      nv = valid.sum(1, keepdim=True)
      order = torch.sort((~valid).int(), dim=1, stable=True).indices
      assert torch.equal(torch.gather(cnt, 1, order),
                         torch.where(torch.arange(n)[None] < nv, s * gs, 0))
      o_idx, o_mask = OS.form_group_indices(valid, gs)
      assert torch.equal(idx, torch.cat([o_idx] * s, 1)), (n, s)
      assert torch.equal(gmask, torch.cat([o_mask] * s, 1)), (n, s)
      for full in (False, True):
        perms = torch.stack([torch.stack([_perm(int(valid[b].sum()), n, g, full)
                                          for b in range(n + 1)]) for _ in range(s)])
        idx, gmask, _, _ = GR.form_groups(valid, gs, perms)
        m_idx = torch.cat([M._form_group_indices(valid, gs, perms[k])[0] for k in range(s)], 1)
        m_mask = torch.cat([M._form_group_indices(valid, gs, perms[k])[1] for k in range(s)], 1)
        assert torch.equal(idx, m_idx), (n, s, full)
        assert torch.equal(gmask, m_mask), (n, s, full)


def _case(B, N, D, gs, hidden, S, relu, seed):
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(B, N, D, generator=g, dtype=torch.float64)
  nv = [0, 1, max(gs - 1, 1), gs, N] + [int(v) for v in torch.randint(0, N + 1, (B,), generator=g)]
  valid = torch.zeros(B, N, dtype=torch.bool)
  for b in range(B):
    valid[b, torch.randperm(N, generator=g)[:min(nv[b], N)]] = True
  dims = [gs * D] + hidden + [gs]
  p = {'w': [], 'b': []}
  for i in range(len(dims) - 1):
    lim = math.sqrt(6.0 / (dims[i] + dims[i + 1]))
    p['w'].append((torch.rand(dims[i], dims[i + 1], generator=g, dtype=torch.float64) * 2 - 1)
                  * lim)
    p['b'].append(torch.rand(dims[i + 1], generator=g, dtype=torch.float64) * 0.4 - 0.2)
  dlogits = torch.randn(B, N, generator=g, dtype=torch.float64)
  return x, valid, R.Cfg(dims, relu=relu), p, dlogits


CASES = [(6, 9, 8, 2, [16, 8], 1), (5, 13, 4, 3, [12], 2), (7, 11, 4, 8, [20, 8], 3),
         (5, 10, 12, 1, [8, 8, 4], 2)]


@pytest.mark.parametrize('relu', [True, False])
@pytest.mark.parametrize('case', CASES)
def test_fp64_reference_matches_oracle(case, relu):
  B, N, D, gs, hidden, S = case
  x, valid, cfg, p, dlogits = _case(B, N, D, gs, hidden, S, relu, seed=B * N + gs)
  groups = GR.form_groups(valid, gs, num_shuffles=S)
  gates = GR.exact_gates(GR.gathered(x, groups[0]), p, cfg)
  ref = GR.forward_backward(x, p, cfg, gates, groups, dlogits)
  leaves = {'dense_w': [w.clone().requires_grad_() for w in p['w']],
            'dense_b': [b.clone().requires_grad_() for b in p['b']]}

  def score_fn(gf):
    return OS.tower_forward(gf.reshape(gf.shape[0], -1), leaves,
                            activation='relu' if relu else None)
  logits = OS.groupwise_logits(x, valid, gs, score_fn, num_shuffles=S)
  (logits * dlogits).sum().backward()
  grads = torch.cat([torch.cat([w.grad.reshape(-1), b.grad.reshape(-1)])
                     for w, b in zip(leaves['dense_w'], leaves['dense_b'])])
  scale = max(1.0, float(logits.detach().abs().max()))
  assert float((ref['logits'] - logits.detach()).abs().max()) <= 1e-12 * scale
  assert float((ref['grads'] - grads).abs().max()) <= 1e-12 * max(1.0, float(grads.abs().max()))
  # items in no valid group hold exactly 0
  assert (ref['logits'][groups[3] == 0] == 0).all()


def _ratio(got, want, mag, u):
  return R.err_ratio(got, want, mag, u)[0]


@pytest.mark.parametrize('defect', ['swap_slots', 'divide_by_S_gs', 'wrap_at_n', 'no_bias0'])
def test_negative_controls_exceed_the_bound(defect):
  """Each defective reference is rejected by the tf32x3 bound on the logits or the gradient.
  Rolling windows give every valid item S gs member scores, so the count only differs from S gs
  when the shuffles bring different items into the valid groups: the permutations here reorder
  the whole valid-first order, invalid items included."""
  B, N, D, gs, hidden, S = 6, 12, 8, 3, [16, 8], 2
  x, valid, cfg, p, dlogits = _case(B, N, D, gs, hidden, S, True, seed=7)
  g = torch.Generator().manual_seed(8)
  perms = torch.stack([torch.stack([torch.randperm(N, generator=g) for _ in range(B)])
                       for _ in range(S)])
  groups = GR.form_groups(valid, gs, perms)
  assert ((groups[3] != 0) & (groups[3] != S * gs)).any()
  gates = GR.exact_gates(GR.gathered(x, groups[0]), p, cfg)
  ref = GR.forward_backward(x, p, cfg, gates, groups, dlogits)
  bound = GR.Bound(cfg, 'tf32x3', B, N, S, gs, SMS)
  bad_groups = GR.form_groups(valid, gs, perms, wrap_at_n=True) \
      if defect == 'wrap_at_n' else groups
  bad = GR.forward_backward(x, p, cfg, gates, bad_groups, dlogits,
                            defect=None if defect == 'wrap_at_n' else defect)
  mag = ref['mag']
  worst = max(_ratio(bad['logits'], ref['logits'], mag['logits'], bound.logits),
              _ratio(bad['grads'], ref['grads'], mag['grads'], bound.grads(cfg)))
  assert worst > 1, (defect, worst)
  # and the true reference passes its own check
  got = {'hidden': [a for a in ref['A'][1:]], 'logits': ref['logits'], 'grads': ref['grads']}
  assert all(r <= 1 for _, r in GR.check(cfg, bound, ref, got))
