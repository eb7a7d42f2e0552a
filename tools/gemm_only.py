"""Runs ONE scorer GEMM shape of the bench configuration through the TF32 engine, a few times,
for `ncu --set full --import-source on -k regex:gemm_kernel -c 1` captures.
usage: gemm_only.py {fwd1|fwd2|fwd3|dz1|dz2|dw1|dw2|dw3}"""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from ranking_b200 import _C

M = 204800
SHAPES = {   # gm, gn, gk, a_mn, b_mn, split_b, epi, transposed, splits
    'fwd1': (M, 256, 136, 0, 0, 0, 1, 0, 1), 'fwd2': (M, 128, 256, 0, 0, 0, 1, 0, 1),
    'fwd3': (M, 64, 128, 0, 0, 0, 1, 0, 1), 'dz1': (M, 256, 128, 0, 0, 0, 3, 0, 1),
    'dz2': (M, 128, 64, 0, 0, 0, 3, 0, 1), 'dw1': (256, 136, M, 1, 1, 1, 0, 1, 146),
    'dw2': (256, 128, M, 1, 1, 1, 0, 0, 146), 'dw3': (128, 64, M, 1, 1, 1, 0, 0, 146)}
gm, gn, gk, a_mn, b_mn, split_b, epi, transposed, splits = SHAPES[sys.argv[1] if len(sys.argv) > 1 else 'fwd1']
A = torch.randn((gk, gm) if a_mn else (gm, gk), device='cuda')
B = torch.randn((gk, gn) if b_mn else (gn, gk), device='cuda')
Blo = None if split_b else torch.randn_like(B) * 1e-4
bias = torch.randn(gn, device='cuda')
bits = torch.randint(-2 ** 31, 2 ** 31 - 1, ((gn + 31) // 32, gm), dtype=torch.int32, device='cuda')
kb = (gk + 31) // 32
stride = ((gm + 127) // 128 * 128) * max(gn, 256) if splits > 1 else 0
C = torch.empty(max(splits, 1) * max(stride, gm * gn), device='cuda')
ldc = gm if transposed else gn
for rep in range(3):
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  _C.check(_C.lib.tfr_tc_gemm(_C.ptr(A), A.shape[1], _C.ptr(B), B.shape[1], _C.ptr(Blo), _C.ptr(C),
                              ldc, gm, gn, gk, a_mn, b_mn, 3, split_b, epi, _C.ptr(bias), None, 1,
                              transposed, splits, stride, _C.ptr(bits if epi == 1 else None),
                              _C.ptr(bits if epi == 3 else None), _C.stream()))
  e1.record()
  torch.cuda.synchronize()
  print('%s: %.1f us' % (sys.argv[1] if len(sys.argv) > 1 else 'fwd1', e0.elapsed_time(e1) * 1e3), flush=True)
