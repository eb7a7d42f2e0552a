"""pytest configuration: `gpu` marker + the `api` fixture.

Golden-vector tests are written once against a small namespace (`api`) and run
against (a) the CPU oracle (always, `-m "not gpu"`) and (b) the CUDA product
path through the C-ABI (`-m gpu`, on an H100).
"""
import os
import sys
import types

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
  sys.path.insert(0, ROOT)


def pytest_configure(config):
  config.addinivalue_line('markers', 'gpu: needs a CUDA device (H100)')


def _oracle_api():
  from oracle import keras_losses, losses_impl, metrics_impl, scorer, utils
  api = types.SimpleNamespace()
  api.name = 'oracle'
  api.device = torch.device('cpu')
  api.losses_impl = losses_impl
  api.keras_losses = keras_losses
  api.metrics_impl = metrics_impl
  api.utils = utils
  api.scorer = scorer
  api.Reduction = losses_impl.Reduction
  api.KerasReduction = keras_losses.Reduction
  api.fns = losses_impl       # identity / inverse / pow_minus_1 / log2_inverse ...
  api.t = lambda x, dtype=torch.float32: torch.tensor(x, dtype=dtype)
  return api


def _cuda_api():
  import ranking_b200 as tfr
  api = types.SimpleNamespace()
  api.name = 'cuda'
  api.device = torch.device('cuda:0')
  api.losses_impl = tfr.losses_impl
  api.keras_losses = tfr.keras.losses
  api.metrics_impl = tfr.metrics_impl
  api.utils = tfr.utils
  api.scorer = None
  api.Reduction = tfr.losses_impl.Reduction
  api.KerasReduction = tfr.keras.losses.Reduction
  api.fns = tfr.keras.utils
  api.t = lambda x, dtype=torch.float32: torch.tensor(
      x, dtype=dtype, device='cuda:0')
  return api


@pytest.fixture(params=['oracle', pytest.param('cuda', marks=pytest.mark.gpu)])
def api(request):
  if request.param == 'oracle':
    return _oracle_api()
  if not torch.cuda.is_available():
    pytest.skip('no CUDA device')
  return _cuda_api()


@pytest.fixture
def oracle_api():
  return _oracle_api()


@pytest.fixture
def cuda_api():
  if not torch.cuda.is_available():
    pytest.skip('no CUDA device')
  return _cuda_api()
