"""3xTF32 scorer tower whose dZ GEMM takes bias column sums over 1000 columns: the GEMM engine
then fits only three pipeline stages beside the column-sum accumulator (four otherwise).  The
widths also give k tails of one and three k steps and tiles of 64 and 128 live columns."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel_err(got, ref):
  got = got.detach().double().cpu()
  ref = ref.detach().double().cpu()
  return float((got - ref).abs().max() / (ref.abs().max() + 1e-30))


def test_tower_wide_colsum_three_stages(oracle_api):
  import ranking_b200 as tfr
  m, d, hidden = 3000, 64, [40, 1000, 24]
  tower = tfr.keras.layers.create_tower(hidden, 1, activation=None, use_batch_norm=False,
                                        dropout=0, input_dim=d, seed=7, precision='tf32x3')
  with torch.no_grad():
    for i in range(len(tower.dims) - 1):
      tower.bias(i).uniform_(-0.2, 0.2)
  nl = len(tower.dims) - 1
  params = {'dense_w': [tower.kernel(i).detach().cpu().double().clone().requires_grad_()
                        for i in range(nl)],
            'dense_b': [tower.bias(i).detach().cpu().double().clone().requires_grad_()
                        for i in range(nl)]}
  g = torch.Generator().manual_seed(m)
  x = torch.randn(m, d, generator=g)
  up = torch.randn(m, 1, generator=g)
  y = tower(x.cuda())
  (y * up.cuda()).sum().backward()
  ref = oracle_api.scorer.tower_forward(x.double(), params, activation=None)
  (ref * up.double()).sum().backward()
  assert _rel_err(y, ref) <= 1e-5, _rel_err(y, ref)
  want = torch.cat([torch.cat([w.grad.reshape(-1), b.grad.reshape(-1)])
                    for w, b in zip(params['dense_w'], params['dense_b'])])
  err = _rel_err(tower.flat.grad, want)
  assert err <= 5e-5, err
