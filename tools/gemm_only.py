"""Times the eight scorer GEMMs of the config-2 training step (fwd1-3, dz1-2, dw1-3) through
the 3xTF32 engine, with the shapes, orientations and split-K counts the trainer uses, and
prints per GEMM the time, the algorithmic TFLOP/s (2 GM GN GK) and the GB/s of the tensors it
must move (operands read once, output and sign words written once), and from the shapes the
time per 128 x 128 tile of a CTA (time x CTAs / tiles) and per 32-wide k block of it.  dw1t-dw3t time the dW
GEMMs as they would run on a transposed dZ (dZ^T [width][M]): direct orientation, A the
MN-major activations, B = dZ^T K-major, copied by cp.async and split in shared memory; same
shapes and split-K count as dw1-dw3.  The last line times the
whole 3xTF32 forward of the config-2 tower (136-256-128-64-1, the fused kernel) through
tfr_mlp_fwd: X read once; H1, H2, H3, their sign words and the scores written once.  It
also prints fwd1 + fwd2 + fwd3 from the same run, the per-layer forward's GEMMs, to compare
against.  The line after it times the fused dW_0 backward kernel (tower_fused_dw0_kernel, which
replaces dz1 + dw1 with the same splits) at the config-2 shapes: its device time from
torch.profiler over a tfr_mlp_bwd loop of the config-2 tower, against dz1 + dw1 from this run.
usage: gemm_only.py [--reps R] [--warmup W] [--out FILE.json]"""
import argparse
import json
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from ranking_b200 import _C

M = 204800                  # B * N rows of the config-2 batch
DIMS = [136, 256, 128, 64]  # Dense widths before the 64 -> 1 output layer (CUDA cores)


def folded_cols(gn):        # wg::folded_cols (wgmma_gemm.cuh): columns folded into the last tile
  return gn % 128 if gn > 128 and gn % 128 <= 8 else 0


def tile_units(gm, gn):     # tc::tile_units (tc_gemm.cu): picks the dW orientation
  return ((gm + 127) // 128) * ((gn - folded_cols(gn) + 63) // 64)


def splits_for(m, sms):     # rows_per_split / splits of the dW GEMMs (capi.cu)
  per = (m + sms - 1) // sms
  rows = 256 if per < 256 else (per + 127) // 128 * 128
  return (m + rows - 1) // rows


def per_tile(gm, gn, gk, splits, fold, sms, us):
  """(tiles per CTA, k blocks per tile, us per tile, us per k block) on the persistent grid.
  fold: the GEMM folds a remainder of up to 8 columns into its last tile (A and B MN-major)."""
  tiles = ((gm + 127) // 128) * ((gn - (folded_cols(gn) if fold else 0) + 127) // 128) * splits
  per_cta = tiles / min(tiles, sms)
  kb = ((gk + 31) // 32 + splits - 1) // splits
  return per_cta, kb, us / per_cta, us / per_cta / kb


def shapes(sms):
  """name -> (gm, gn, gk, a_mn, b_mn, split_b, epi, transposed, splits), as mlp_tc.cu calls."""
  out, L = {}, len(DIMS) - 1
  for d in range(L):         # forward: H = act(A W + b), W^T pre-split (K-major), sign bits out
    out['fwd%d' % (d + 1)] = (M, DIMS[d + 1], DIMS[d], 0, 0, 0, 1, 0, 1)
  for d in range(L - 1, 0, -1):   # dZ_{d-1} = (dZ_d W_d^T) * relu'(H), W pre-split (K-major)
    out['dz%d' % d] = (M, DIMS[d], DIMS[d + 1], 0, 0, 0, 3, 0, 1)
  s = splits_for(M, sms)
  for d in range(L):         # dW = A^T dZ, both MN-major, split on the fly, split-K partials
    kin, nout = DIMS[d], DIMS[d + 1]
    if tile_units(nout, kin) < tile_units(kin, nout):
      out['dw%d' % (d + 1)] = (nout, kin, M, 1, 1, 1, 0, 1, s)
    else:
      out['dw%d' % (d + 1)] = (kin, nout, M, 1, 1, 1, 0, 0, s)
  for d in range(L):         # dW = A^T (dZ^T)^T: A MN-major, B = dZ^T K-major through cp.async
    out['dw%dt' % (d + 1)] = (DIMS[d], DIMS[d + 1], M, 1, 0, 1, 0, 0, s)
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=50)
  ap.add_argument('--warmup', type=int, default=5)
  ap.add_argument('--out', default=None)
  args = ap.parse_args()
  dev = torch.device('cuda')
  sms = torch.cuda.get_device_properties(dev).multi_processor_count
  g = torch.Generator(device=dev).manual_seed(0)
  calls = {}
  for name, (gm, gn, gk, a_mn, b_mn, split_b, epi, tr, splits) in shapes(sms).items():
    A = torch.randn((gk, gm) if a_mn else (gm, gk), device=dev, generator=g)
    B = torch.randn((gk, gn) if b_mn else (gn, gk), device=dev, generator=g)
    Blo = None if split_b else torch.randn(B.shape, device=dev, generator=g) * 1e-4
    bias = torch.randn(gn, device=dev, generator=g)
    bits = torch.randint(-2 ** 31, 2 ** 31 - 1, ((gn + 31) // 32, gm), dtype=torch.int32,
                         device=dev, generator=g)
    stride = (gm + 127) // 128 * 128 * max(gn, 256) if splits > 1 else 0
    C = torch.empty(splits * max(stride, gm * gn), device=dev)
    ldc = gm if tr else gn
    nbytes = 4 * (A.numel() + B.numel() * (1 if split_b else 2) + splits * gm * gn)
    if epi in (1, 3):
      nbytes += 4 * bits.numel()

    def call(A=A, B=B, Blo=Blo, C=C, bias=bias, bits=bits, gm=gm, gn=gn, gk=gk, a_mn=a_mn,
             b_mn=b_mn, split_b=split_b, epi=epi, tr=tr, splits=splits, stride=stride, ldc=ldc):
      _C.check(_C.lib.tfr_tc_gemm(
          _C.ptr(A), A.shape[1], _C.ptr(B), B.shape[1], _C.ptr(Blo), _C.ptr(C), ldc, gm, gn, gk,
          a_mn, b_mn, 3, split_b, epi, _C.ptr(bias), None, 1, tr, splits, stride,
          _C.ptr(bits if epi == 1 else None), _C.ptr(bits if epi == 3 else None), _C.stream()))
    calls[name] = (call, 2.0 * gm * gn * gk, nbytes, (gm, gn, gk, splits, a_mn and b_mn))

  for call, _, _, _ in calls.values():   # every shape warm before any is timed
    for _ in range(args.warmup):
      call()
  torch.cuda.synchronize()
  rows = []
  for name, (call, flop, nbytes, shape) in calls.items():
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.reps):
      call()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / args.reps
    per_cta, kb, us_tile, us_kb = per_tile(*shape, sms, us)
    rows.append(dict(gemm=name, gm=shape[0], gn=shape[1], gk=shape[2], splits=shape[3],
                     us=round(us, 2), tflops=round(flop / us * 1e-6, 2),
                     gbps=round(nbytes / us * 1e-3, 1), tiles_per_cta=round(per_cta, 2),
                     k_blocks_per_tile=kb, us_per_tile=round(us_tile, 2),
                     us_per_k_block=round(us_kb, 2)))
    print('%-5s GM %6d GN %4d GK %6d splits %4d  %8.1f us  %6.1f TFLOP/s  %7.1f GB/s  '
          '%5.1f tiles/CTA x %3d k blocks: %6.2f us/tile %5.2f us/block' % (
              name, shape[0], shape[1], shape[2], shape[3], us, rows[-1]['tflops'],
              rows[-1]['gbps'], per_cta, kb, us_tile, us_kb), flush=True)
  step = [r for r in rows if not r['gemm'].endswith('t')]   # the eight GEMMs the step runs
  total = sum(r['us'] for r in step)
  print('total %.1f us' % total, flush=True)
  dw = sum(r['us'] for r in step if r['gemm'].startswith('dw'))
  dwt = sum(r['us'] for r in rows if r['gemm'].startswith('dw') and r['gemm'].endswith('t'))
  print('dw1-dw3 %.1f us, dw1t-dw3t %.1f us (%+.1f %%)' % (dw, dwt, 100.0 * (dwt / dw - 1.0)),
        flush=True)
  fwd = time_tower_fwd(dev, g, args.reps, args.warmup)
  per_layer = sum(r['us'] for r in step if r['gemm'].startswith('fwd'))
  print('tower fwd (tfr_mlp_fwd, M %d)  %8.1f us  %6.1f TFLOP/s  %7.1f GB/s  '
        '(fwd1 + fwd2 + fwd3 %.1f us, %+.1f %%)' % (
            M, fwd['us'], fwd['tflops'], fwd['gbps'], per_layer,
            100.0 * (fwd['us'] / per_layer - 1.0)), flush=True)
  fused = time_fused_dw0(dev, g, args.reps, args.warmup, sms)
  pair = sum(r['us'] for r in step if r['gemm'] in ('dz1', 'dw1'))
  print('fused dW_0 (tower_fused_dw0_kernel, M %d, %d units)  %8.1f us  %6.2f us/tile-half  '
        '(dz1 + dw1 %.1f us, %+.1f %%)' % (
            M, fused['units'], fused['us'], fused['us_per_tile_half'], pair,
            100.0 * (fused['us'] / pair - 1.0)), flush=True)
  if args.out:
    with open(args.out, 'w') as f:
      json.dump(dict(device=torch.cuda.get_device_name(dev), sms=sms, reps=args.reps,
                     gemms=rows, total_us=round(total, 2), dw_us=round(dw, 2),
                     dwt_us=round(dwt, 2), fwd_per_layer_us=round(per_layer, 2),
                     tower_fwd=fwd, fused_dw0=fused, dz1_dw1_us=round(pair, 2)), f, indent=1)


def time_tower_fwd(dev, g, reps, warmup):
  """The config-2 tower's whole 3xTF32 forward (parameter split included) at M rows."""
  import ctypes
  from ranking_b200.keras import layers
  tower = layers.create_tower(DIMS[1:], 1, activation='relu', use_batch_norm=False, dropout=0,
                              input_dim=DIMS[0], seed=0, precision='tf32x3')
  x = torch.randn(M, DIMS[0], device=dev, generator=g)
  ws = tower._new_workspace(M)
  out = torch.empty(M, 1, device=dev)
  cfg = tower._run_cfg()

  def call():
    _C.check(_C.lib.tfr_mlp_fwd(_C.ptr(x), M, ctypes.byref(cfg), _C.ptr(tower.flat.data),
                                None, _C.ptr(ws), _C.ptr(out), _C.PREC_TF32X3, _C.stream()))
  for _ in range(warmup):
    call()
  torch.cuda.synchronize()
  e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  e0.record()
  for _ in range(reps):
    call()
  e1.record()
  torch.cuda.synchronize()
  us = e0.elapsed_time(e1) * 1e3 / reps
  dims = DIMS + [1]
  flop = sum(2.0 * M * dims[i] * dims[i + 1] for i in range(len(dims) - 1))
  words = sum((n + 31) // 32 for n in DIMS[1:])          # sign words per row
  nbytes = 4 * M * (DIMS[0] + sum(DIMS[1:]) + words + 1)
  return dict(m=M, us=round(us, 2), tflops=round(flop / us * 1e-6, 2),
              gbps=round(nbytes / us * 1e-3, 1), bytes=nbytes, flop=flop)


def time_fused_dw0(dev, g, reps, warmup, sms):
  """Device time of tower_fused_dw0_kernel per call, from torch.profiler over `reps` backward
  calls of the config-2 tower (the kernel runs once per call).  A work unit is one row split
  times one 128-column half of dZ_0; a tile-half is one 128-row tile of a unit."""
  import ctypes
  from ranking_b200.keras import layers
  tower = layers.create_tower(DIMS[1:], 1, activation='relu', use_batch_norm=False, dropout=0,
                              input_dim=DIMS[0], seed=0, precision='tf32x3')
  x = torch.randn(M, DIMS[0], device=dev, generator=g)
  ds = torch.randn(M, device=dev, generator=g)
  ws = tower._new_workspace(M)
  out = torch.empty(M, 1, device=dev)
  grads = torch.empty_like(tower.flat.data)
  cfg = tower._run_cfg()
  _C.check(_C.lib.tfr_mlp_fwd(_C.ptr(x), M, ctypes.byref(cfg), _C.ptr(tower.flat.data), None,
                              _C.ptr(ws), _C.ptr(out), _C.PREC_TF32X3, _C.stream()))

  def call():
    _C.check(_C.lib.tfr_mlp_bwd(_C.ptr(x), M, ctypes.byref(cfg), _C.ptr(tower.flat.data),
                                _C.ptr(ds), None, _C.ptr(ws), _C.ptr(grads), _C.PREC_TF32X3,
                                _C.stream()))
  for _ in range(warmup):
    call()
  torch.cuda.synchronize()
  from torch.profiler import ProfilerActivity, profile
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(reps):
      call()
    torch.cuda.synchronize()
  ev = [e for e in prof.key_averages() if 'tower_fused_dw0_kernel' in e.key]
  if len(ev) != 1 or ev[0].count != reps:
    raise RuntimeError('expected %d tower_fused_dw0_kernel launches, profiled %s' % (
        reps, [(e.key, e.count) for e in ev]))
  us = ev[0].device_time_total / reps
  splits = splits_for(M, sms)
  units = 2 * splits
  rows = ((M + 31) // 32 + splits - 1) // splits * 32
  tiles = sum((min(M, (s + 1) * rows) - s * rows + 127) // 128 for s in range(splits)) * 2
  return dict(us=round(us, 2), units=units, tile_halves=tiles,
              us_per_tile_half=round(us * min(units, sms) / tiles, 3))


if __name__ == '__main__':
  main()
