"""Times one TFR-BERT training step (tfr_bert_fwd, softmax loss, tfr_bert_bwd, AdamW) at the
reference recipe's shape, against batched PyTorch autograd of the same math, alternating the
arms within one run:

  ours-fp32    3xTF32 GEMMs, FP32 attention core          (precision 'fp32')
  ours-tf32    TF32 GEMMs, wgmma TF32 attention core      (precision 'tf32')
  ours-bf16    bf16 GEMMs and wgmma attention core on fp32 master weights (precision 'bf16')
  ours-fp16    the same in fp16 with dynamic loss scaling (precision 'fp16': tfr_loss_scale_mul,
               tfr_global_norm, tfr_adamw_step_scaled, tfr_loss_scale_update)
  ours-*-clip  the same with gradient_clip_norm 1.0 (the recipe's AdamWeightDecay clipping:
               tfr_global_norm + tfr_adamw_step_clipped), for tf32 and bf16
  torch-fp32   torch autograd + torch.optim.AdamW, TF32 matmul off
  torch-tf32   the same with TF32 matmul on
  torch-bf16   the same under torch.autocast('cuda', dtype=torch.bfloat16): ours-bf16's
               like-for-like competitor (fp32 parameters and optimizer, bf16 compute)
  torch-fp16   torch.autocast('cuda', dtype=torch.float16) with torch.amp.GradScaler (dynamic
               loss scale): ours-fp16's competitor

BERT-base (12 layers, E 768, H 12, I 3072), seq 64, lists of 10, at 4 lists (the reference
yaml) and 32.  Dropout 0.1 everywhere in both.  Then one profiled step of each of our arms,
kernel time summed by family (embedding, attention, FFN, LayerNorm, GEMM, pooler and loss,
optimizer).  Prints one JSON line per (shape, arm) and one per profile; writes them to
--out too.  --arms picks a subset (the profiles cover the chosen ours-* arms).

  python tools/tfrbert_step.py --steps 20 --warmup 5 --out /tmp/tfrbert_step.jsonl
  python tools/tfrbert_step.py --lists 32 --arms ours-tf32 ours-tf32-clip ours-bf16 \
      ours-bf16-clip
"""
import argparse
import json
import math
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch                                   # noqa: E402

from ranking_b200 import train                 # noqa: E402
from ranking_b200.extension import tfrbert     # noqa: E402
from ranking_b200.keras import losses          # noqa: E402

E, H, I, NL, V, SEQ, N = 768, 12, 3072, 12, 30522, 64, 10


def _batch(b, seed=0):
  g = torch.Generator().manual_seed(seed)
  wid = torch.randint(0, V, (b, N, SEQ), generator=g, dtype=torch.int32).cuda()
  mask = torch.ones(b, N, SEQ, dtype=torch.uint8)
  mask[..., 48:] = 0
  tid = torch.zeros(b, N, SEQ, dtype=torch.int32)
  tid[..., 20:48] = 1
  y = torch.randint(0, 3, (b, N), generator=g).float()
  return wid, mask.cuda(), tid.cuda(), y.cuda()


class TorchBert(torch.nn.Module):
  """The same post-LN encoder, pooler and head in plain torch (fp32 parameters)."""

  def __init__(self):
    super().__init__()
    self.word = torch.nn.Embedding(V, E)
    self.pos = torch.nn.Embedding(512, E)
    self.types = torch.nn.Embedding(2, E)
    self.ln = torch.nn.LayerNorm(E, eps=1e-12)
    self.layers = torch.nn.ModuleList([
        torch.nn.TransformerEncoderLayer(E, H, I, dropout=0.1, batch_first=True,
                                         activation=lambda u: torch.nn.functional.gelu(
                                             u, approximate='tanh'), layer_norm_eps=1e-12)
        for _ in range(NL)])
    self.pool = torch.nn.Linear(E, E)
    self.head = torch.nn.Linear(E, 1)
    self.drop = torch.nn.Dropout(0.1)

  def forward(self, wid, mask, tid):
    s = wid.shape[-1]
    x = self.word(wid.long()) + self.pos.weight[:s] + self.types(tid.long())
    x = self.drop(self.ln(x))
    pad = mask == 0
    for layer in self.layers:
      x = layer(x, src_key_padding_mask=pad)
    return self.head(self.drop(torch.tanh(self.pool(x[:, 0])))).squeeze(-1)


def _softmax_loss(y, s):
  valid = y >= 0
  s = torch.where(valid, s, torch.full_like(s, -1e30))
  lab = torch.where(valid, y, torch.zeros_like(y))
  den = lab.sum(1, keepdim=True)
  keep = den[:, 0] > 0
  p = lab / den.clamp_min(1e-30)
  return -(p * torch.log_softmax(s, 1)).sum(1)[keep].sum() / max(int(keep.sum()), 1)


def _ours(precision, clip=None):
  enc = tfrbert.BertEncoder(seed=1, precision=precision)
  tr = tfrbert.TFRBertRankingTrainer(tfrbert.TFRBertScorer(enc, 0.1), losses.get('softmax_loss'),
                                     learning_rate=train.PolynomialWarmUp(3e-5, 10000, 1000),
                                     gradient_clip_norm=clip)
  return lambda wid, mask, tid, y: tr.train_step(wid, mask, tid, y)


def _torch(tf32, dtype=None):
  torch.manual_seed(1)
  model = TorchBert().cuda().train()
  decay = [p for n, p in model.named_parameters()
           if 'norm' not in n and not n.startswith('ln.') and not n.endswith('bias')]
  rest = [p for n, p in model.named_parameters() if not any(p is q for q in decay)]
  opt = torch.optim.AdamW([{'params': decay, 'weight_decay': 0.01},
                           {'params': rest, 'weight_decay': 0.0}], lr=3e-5, eps=1e-6)
  scaler = torch.amp.GradScaler('cuda', enabled=dtype == torch.float16)

  def step(wid, mask, tid, y):
    torch.backends.cuda.matmul.allow_tf32 = tf32
    torch.backends.cudnn.allow_tf32 = tf32
    b = wid.shape[0]
    with torch.autocast('cuda', dtype=dtype or torch.bfloat16, enabled=dtype is not None):
      s = model(wid.reshape(b * N, SEQ), mask.reshape(b * N, SEQ),
                tid.reshape(b * N, SEQ)).reshape(b, N)
    loss = _softmax_loss(y, s.float())
    opt.zero_grad(set_to_none=True)
    scaler.scale(loss).backward()   # no-ops without fp16
    scaler.step(opt)
    scaler.update()
    return loss
  return step


_FAMILIES = [('embedding', ('emb_ln', 'embedding', 'radix', 'segment', 'scatter_rows')),
             ('attention', ('attn_',)),
             ('ffn_gelu', ('gelu',)),
             ('layernorm', ('ln_fwd', 'ln_bwd', 'reduce_partials')),
             ('pooler_loss', ('head_', 'loss', 'softmax', 'cls_scatter')),
             ('optimizer', ('adamw', 'sumsq_partials', 'norm_final', 'loss_scale')),
             ('gemm', ('gemm', 'wgmma', 'colsum', 'tc_', 'weight_grad', 'split', 'shadow'))]


def _family(name):
  low = name.lower()
  for fam, keys in _FAMILIES:
    if any(k in low for k in keys):
      return fam
  return 'other'


_ARMS = {'ours-fp32': lambda: _ours('fp32'), 'ours-tf32': lambda: _ours('tf32'),
         'ours-tf32-clip': lambda: _ours('tf32', 1.0), 'ours-bf16': lambda: _ours('bf16'),
         'ours-bf16-clip': lambda: _ours('bf16', 1.0), 'ours-fp16': lambda: _ours('fp16'),
         'torch-fp32': lambda: _torch(False), 'torch-tf32': lambda: _torch(True),
         'torch-bf16': lambda: _torch(True, torch.bfloat16),
         'torch-fp16': lambda: _torch(True, torch.float16)}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--warmup', type=int, default=5)
  ap.add_argument('--rounds', type=int, default=3)
  ap.add_argument('--lists', type=int, nargs='+', default=[4, 32])
  ap.add_argument('--out')
  ap.add_argument('--arms', nargs='+', choices=sorted(_ARMS), default=None,
                  help='default: every arm')
  args = ap.parse_args()
  if not torch.cuda.is_available():
    raise SystemExit('tfrbert_step: no CUDA device')
  gpu = torch.cuda.get_device_name()
  try:
    power = subprocess.run(['nvidia-smi', '--query-gpu=power.limit,clocks.max.sm',
                            '--format=csv,noheader'], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
  except Exception:   # noqa: BLE001
    power = 'unknown'
  lines = []
  for b in args.lists:
    batch = _batch(b)
    arms = {name: make() for name, make in _ARMS.items()
            if args.arms is None or name in args.arms}
    for fn in arms.values():
      for _ in range(args.warmup):
        fn(*batch)
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(args.rounds):   # alternate the arms
      for name, fn in arms.items():
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.steps):
          loss = fn(*batch)
        t1.record()
        torch.cuda.synchronize()
        times[name].append(t0.elapsed_time(t1) / args.steps)
        assert math.isfinite(float(loss))
    for name, ts in times.items():
      rec = {'lists': b, 'list_size': N, 'seq': SEQ, 'arm': name, 'ms_per_step': min(ts),
             'ms_rounds': ts, 'gpu': gpu, 'power_limit_and_max_sm_clock': power}
      lines.append(rec)
      print(json.dumps(rec), flush=True)
    for name in [a for a in arms if a.startswith('ours-')]:
      fn = arms[name]
      with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn(*batch)
        torch.cuda.synchronize()
      fam = {}
      for ev in prof.key_averages():
        us = getattr(ev, 'device_time_total', None)
        if us is None:
          us = ev.cuda_time_total
        if us:
          fam[_family(ev.key)] = fam.get(_family(ev.key), 0.0) + us / 1000.0
      rec = {'lists': b, 'arm': name, 'profile_ms_by_kernel_family':
             {k: round(v, 3) for k, v in sorted(fam.items())}}
      lines.append(rec)
      print(json.dumps(rec), flush=True)
    del arms
    torch.cuda.empty_cache()
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
      for rec in lines:
        f.write(json.dumps(rec) + '\n')


if __name__ == '__main__':
  main()
