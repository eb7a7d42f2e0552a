"""ncu-rep -> compact per-kernel CSV (duration, DRAM bytes, pipe utilisation).
usage: python tools/ncu_summary.py step.ncu-rep step_ncu_full_summary.csv"""
import csv
import io
import json
import subprocess
import sys

COLS = ['Kernel Name', 'Grid Size', 'Block Size', 'gpu__time_duration.sum',
        'dram__bytes_read.sum', 'dram__bytes_write.sum',
        'gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed',
        'lts__throughput.avg.pct_of_peak_sustained_elapsed',
        'sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active',
        'sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active',
        'sm__warps_active.avg.pct_of_peak_sustained_active',
        'smsp__issue_active.avg.pct_of_peak_sustained_active',
        'launch__registers_per_thread', 'launch__shared_mem_per_block_dynamic',
        'sm__throughput.avg.pct_of_peak_sustained_elapsed']

raw = subprocess.run(['ncu', '-i', sys.argv[1], '--page', 'raw', '--csv'], check=True,
                     capture_output=True, text=True).stdout
rows = list(csv.reader(io.StringIO(raw)))
head, units = rows[0], rows[1]
idx = [head.index(c) for c in COLS]
with open(sys.argv[2], 'w', newline='') as f:
  w = csv.writer(f)
  w.writerow(COLS)
  w.writerow([units[i] for i in idx])
  for r in rows[2:]:
    w.writerow([r[i] for i in idx])
if len(sys.argv) > 3:
  def to_bytes(v, u):
    v = float(v.replace(',', ''))
    return v * {'byte': 1, 'Kbyte': 1e3, 'Mbyte': 1e6, 'Gbyte': 1e9}[u]
  ir, iw, ik = head.index('dram__bytes_read.sum'), head.index('dram__bytes_write.sum'), head.index('Kernel Name')
  def total(pred):
    return int(sum(to_bytes(r[ir], units[ir]) + to_bytes(r[iw], units[iw]) for r in rows[2:]
                   if pred(r[ik])))
  # the scorer: GEMM engines, output-layer kernels, group gather / scatter, their reductions
  scorer = lambda k: any(t in k for t in ('gemm_kernel', 'out_layer', 'out_fwd', 'out_bwd', 'group_',
                                          'reduce', 'split_params', 'shadow_params'))
  loss = lambda k: any(t in k for t in ('approx_loss', 'pairwise_tri', 'pairwise_loss', 'softmax_loss'))
  json.dump({'source': sys.argv[2] + ' (ncu --set full, one training step of the bench workload)',
             'scorer_gemm_dram_bytes_per_step': total(scorer),
             'loss_dram_bytes_per_step': total(loss),
             'all_kernels_dram_bytes_per_step': total(lambda k: True)},
            open(sys.argv[3], 'w'), indent=1)
