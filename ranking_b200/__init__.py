"""ranking_b200 — H100-native learning-to-rank training path.

Drop-in for the hot path of tensorflow/ranking: `keras.losses`, `keras.metrics`,
`keras.model` / `keras.layers` scorer, plus the numeric cores `losses_impl`,
`metrics_impl`, `utils`.  Host code is Python over torch tensors; all arithmetic
runs in hand-written sm_90a CUDA kernels behind the C ABI in
`include/tfr_b200.h` (loaded by `ranking_b200._C`; importing this package
without the built library raises).
"""
from ranking_b200 import _C  # noqa: F401  (fails loudly if the .so is missing)
from ranking_b200 import keras
from ranking_b200 import losses_impl
from ranking_b200 import losses
from ranking_b200 import metrics_impl
from ranking_b200 import metrics
from ranking_b200 import utils
from ranking_b200 import dp
from ranking_b200 import model
from ranking_b200 import train
from ranking_b200 import data
from ranking_b200 import pipeline
from ranking_b200 import research
from ranking_b200 import extension

__version__ = '0.1.0'
