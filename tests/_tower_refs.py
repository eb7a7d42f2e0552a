"""fp64 restatement of the bf16 scorer tower's arithmetic (TFR_PREC_BF16), shared by
tests/test_parity_round2_gpu.py and tests/test_tower_output_layer_gpu.py, and a record of
the CUDA kernels a call launches, so that a test can assert which kernel variant ran."""
import json
import os
import re
import tempfile

import torch


def kernel_launches(fn):
  """Runs fn() under torch.profiler; returns (fn's result, [(kernel, grid, block)]) in
  launch order.  `kernel` is the bare name with its template arguments, e.g.
  'out_layer_bwd2_vec_kernel<4>'; grid and block are (x, y, z) tuples.

  A profiling session can lose GPU kernel records: most often those of the first kernels
  it sees, now and then all of them (seen on H100 with torch 2.11, more often late in a
  long test run).  So a session runs fn() three times, each run in its own annotated
  range, and the launches of the first run whose every kernel launch call has its GPU
  record (matched by correlation id) are returned; if no run is complete, the session is
  repeated, up to three times.  fn() must therefore be repeatable: it resets whatever
  state it changes (gradients, BN statistics, dropout counters)."""
  from torch.profiler import ProfilerActivity, profile, record_function
  runs = 3
  launches = []
  for _ in range(3):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
      for r in range(runs):
        with record_function('kernel_launches %d' % r):
          out = fn()
          torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
      path = os.path.join(d, 'trace.json')
      prof.export_chrome_trace(path)
      with open(path) as f:
        events = json.load(f)['traceEvents']
    spans = {e['name']: e for e in events if e.get('cat') == 'user_annotation'}
    for r in range(runs):
      span = spans.get('kernel_launches %d' % r)
      if span is None:
        continue
      calls = {e['args']['correlation'] for e in events
               if e.get('cat') in ('cuda_runtime', 'cuda_driver')
               and re.search(r'Launch\w*Kernel', e['name'])
               and span['ts'] <= e['ts'] <= span['ts'] + span['dur']}
      records = sorted((e for e in events
                        if e.get('cat') == 'kernel' and e['args'].get('correlation') in calls),
                       key=lambda e: e['ts'])
      launches = []
      for e in records:
        m = re.search(r'(\w+(?:<[^<>()]*>)?)\(', e['name'])
        name = (m.group(1) if m else e['name']).replace(' ', '')
        launches.append((name, tuple(e['args']['grid']), tuple(e['args']['block'])))
      if calls and len(records) == len(calls):
        return out, launches
  return out, launches


def _bf(t):
  return t.bfloat16().double()


def _emulated_bf16_tower(x, ws, bs, dscores, relu=True):
  """fp64 restatement of the bf16 tower's arithmetic: bf16 inputs / weights / stored
  activations and backward signals, exact accumulation.  Returns scores, flat grads."""
  L = len(ws) - 1
  h = [_bf(x)]
  for d in range(L):
    z = h[-1] @ _bf(ws[d]) + bs[d].double()
    a = torch.relu(z) if relu else z
    h.append(_bf(a))
  scores = h[-1] @ ws[L].double() + bs[L].double()
  grads_w, grads_b = [None] * (L + 1), [None] * (L + 1)
  ds = dscores.double()
  grads_w[L] = h[-1].t() @ ds
  grads_b[L] = ds.sum(0)
  dz_full = ds @ ws[L].double().t()
  if relu:
    dz_full = dz_full * (h[-1] > 0)
  for d in range(L - 1, -1, -1):
    grads_b[d] = dz_full.sum(0)            # column sums are taken before the bf16 rounding
    dz = _bf(dz_full)
    grads_w[d] = h[d].t() @ dz
    if d > 0:
      dz_full = dz @ _bf(ws[d]).t()
      if relu:
        dz_full = dz_full * (h[d] > 0)
  flat = torch.cat([torch.cat([w.reshape(-1), b.reshape(-1)])
                    for w, b in zip(grads_w, grads_b)])
  return scores, flat
