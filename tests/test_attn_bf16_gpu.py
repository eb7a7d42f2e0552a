"""TFR-BERT's bf16 attention core (csrc/din_bf16.cu) on its own, through tfr_attn_bf16_fwd /
tfr_attn_bf16_bwd, against the fp64 replay of its rounding points (_tfrbert_bf16_refs.attention)
on the same bf16 qkv and dO, with autograd supplying dQ, dK and dV.

Per-element bars (attn_bars) and the RMS ratio ||kernel - replay|| / ||unrounded - replay||
on O, dQ, dK and dV; lse and dsum against fp64; exact checks (identical calls, every output
element written and nothing past it, NULL mask, single-valid and all-padded lists); negative
controls that each move the replay past a bar or the ratio; the entry's argument checks.

The case table puts every head-size bucket (16 / 32 / 64 / 128, TFR_DIN_BF16_DISPATCH) on both
sides of its edges, N on both sides of the 64-row tiles (N <= 64 takes the forward's one-tile
path) up to 1024, H h up to 1024, the mask kinds ragged / all-padded / single-valid / NULL,
dropout 0 and 0.1 - 0.3, and logits of magnitude ~50.
"""
import ctypes
import math
import os
import re

import numpy as np
import pytest
import torch

import _tfrbert_bf16_refs as B

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INVALID_ARGUMENT = 1
ROWS = 64   # din_bf16.cu kT: rows of a CTA, keys of a tile
GUARD = 64  # sentinel elements after every output buffer

# (B, N, H, h, mask, dropout, sigma of q and k)
CASES = [
    (3, 1, 2, 8, 'ragged', 0.0, 1.0),
    (3, 2, 4, 16, 'single', 0.0, 1.0),
    (3, 63, 2, 24, 'ragged', 0.2, 1.0),
    (2, 64, 3, 32, 'null', 0.0, 1.0),
    (3, 65, 2, 40, 'ragged', 0.1, 1.0),
    (2, 127, 2, 64, 'single', 0.0, 1.0),
    (3, 128, 2, 72, 'ragged', 0.3, 1.0),
    (3, 129, 2, 120, 'ragged', 0.0, 1.0),
    (3, 511, 2, 128, 'ragged', 0.1, 1.0),
    (2, 512, 4, 32, 'padded', 0.0, 1.0),
    (3, 200, 4, 8, 'ragged', 0.2, 1.0),
    (2, 130, 8, 128, 'null', 0.0, 4.0),    # |logits| ~ 50: max subtraction; H h = 1024
    (1, 1024, 16, 64, 'ragged', 0.1, 1.0),  # TFR_DIN_MAX_LIST, H h = 1024
]
# RMS ratio limit: the kernel against the replay, a fraction of the rounding's own effect
# (the replay against the unrounded op).  Measured on an H100 SXM (700 W power limit), the
# largest ratios of the table are O 0.054 and dV 0.053 (N 511), dQ 0.076 and dK 0.093
# (N 1024); cases with few enough terms that no bf16 rounding flips give exactly 0.
RATIO = 1.0 / 8.0


def _id(c):
  return 'B%d-N%d-H%d-h%d-%s-p%g-s%g' % c


def _bucket_src():
  src = open(os.path.join(ROOT, 'ranking_b200', 'csrc', 'din_bf16.cu')).read()
  body = re.search(r'constexpr int bucket\(int h\) \{(.*?)\}', src, re.S).group(1)
  pairs = [(int(a), int(b)) for a, b in re.findall(r'h <= (\d+) \? (\d+)', body)]
  return pairs, int(re.search(r': (\d+);', body).group(1))


def bucket(h):
  pairs, last = _bucket_src()
  for edge, hp in pairs:
    if h <= edge:
      return hp
  return last


def _mask(kind, b, n, g):
  """uint8 [B, N]: ragged (prefix of random length, the last list all padded), padded (no
  valid key), single (only key 0 in even lists, only key N - 1 in odd ones); None for null."""
  if kind == 'null':
    return None
  m = torch.zeros(b, n, dtype=torch.uint8)
  if kind == 'ragged':
    for i in range(b - 1):
      m[i, :n if i == 0 else int(torch.randint(1, n + 1, (1,), generator=g))] = 1
    if b == 1:
      m[0, :max(1, n - 37)] = 1
  elif kind == 'single':
    for i in range(b):
      m[i, 0 if i % 2 == 0 else n - 1] = 1
  return m


def _inputs(case, seed=0):
  b, n, H, h, kind, drop, sigma = case
  g = torch.Generator().manual_seed(seed + n + h)
  E = H * h
  qkv = torch.randn(b, n, 3 * E, generator=g)
  qkv[..., :2 * E] *= sigma
  dO = torch.randn(b, n, E, generator=g)
  return qkv.bfloat16(), _mask(kind, b, n, g), dO.bfloat16()


def _seed(case):
  return 1000 + case[1], 7 + case[3]   # (seed, site)


def _dseed(seed, site):
  return (seed * 0x100000001B3 + site) & 0xFFFFFFFFFFFFFFFF


def _guarded(n, dtype, fill):
  """(buffer of n elements + GUARD sentinels, its first n) on the device."""
  buf = torch.empty(n + GUARD, dtype=dtype, device='cuda')
  buf[:n] = float('nan')
  buf[n:] = fill
  return buf


def run_kernel(case, qkv, mask, dO, lmask='given'):
  """Kernel outputs {O, lse, dsum, dqkv} (device), after checking that every element of the
  B N rows is written and the guard band after each buffer is untouched."""
  from ranking_b200 import _C
  b, n, H, h, _, drop, _ = case
  E = H * h
  m = b * n
  seed, site = _seed(case)
  q = qkv.cuda().contiguous()
  d = dO.cuda().contiguous()
  lm = None if mask is None else mask.reshape(-1).cuda()
  if lmask == 'ones':
    lm = torch.ones(m, dtype=torch.uint8, device='cuda')
  bufs = {'O': _guarded(m * E, torch.bfloat16, 3.0), 'lse': _guarded(m * H * 2, torch.float32, 5.0),
          'dsum': _guarded(m * H, torch.float32, 7.0),
          'dqkv': _guarded(m * 3 * E, torch.bfloat16, 9.0)}
  ds = _dseed(seed, site)
  _C.check(_C.lib.tfr_attn_bf16_fwd(_C.ptr(q), _C.ptr(lm), b, n, H, h, drop, ds,
                                    _C.ptr(bufs['O']), _C.ptr(bufs['lse']), _C.stream()))
  _C.check(_C.lib.tfr_attn_bf16_bwd(_C.ptr(q), _C.ptr(lm), b, n, H, h, drop, ds,
                                    _C.ptr(bufs['O']), _C.ptr(bufs['lse']), _C.ptr(d),
                                    _C.ptr(bufs['dsum']), _C.ptr(bufs['dqkv']), _C.stream()))
  torch.cuda.synchronize()
  out = {}
  for k, fill in (('O', 3.0), ('lse', 5.0), ('dsum', 7.0), ('dqkv', 9.0)):
    body, guard = bufs[k][:-GUARD], bufs[k][-GUARD:]
    assert not torch.isnan(body.float()).any(), (k, 'unwritten elements')
    assert (guard.float() == fill).all(), (k, 'guard band overwritten')
    out[k] = body
  out['O'] = out['O'].reshape(b, n, E)
  out['lse'] = out['lse'].reshape(b, n, H, 2)
  out['dsum'] = out['dsum'].reshape(b, n, H)
  out['dqkv'] = out['dqkv'].reshape(b, n, 3 * E)
  return out


def replay(case, qkv, mask, dO, rounding=True, round_out=True, dev='cpu', **kw):
  """(O, dqkv) fp64 of the replay on the same bf16 values; dqkv rounded to bf16 as stored
  (round_out False: not)."""
  b, n, H, h, _, drop, _ = case
  seed, site = _seed(case)
  x = qkv.to(dev).double().requires_grad_()
  m = torch.ones(b, n, dtype=torch.uint8) if mask is None else mask
  o = B.attention(x, m, H, drop, seed, site, rounding=rounding, **kw)
  o.backward(dO.to(dev).double())
  g = x.grad
  if rounding and round_out:
    g = B.bf16(g)
  return o.detach(), g


def _split(dqkv, E):
  return {'dQ': dqkv[..., :E], 'dK': dqkv[..., E:2 * E], 'dV': dqkv[..., 2 * E:]}


def _tensors(O, dqkv, E):
  t = {'O': O}
  t.update(_split(dqkv, E))
  return t


def _rms_ratio(got, rep, ex):
  """None where the rounding has no effect (an exactly zero gradient: N = 1, or a list with
  one valid key and no dropout); the per-element bar still holds there."""
  den = float((ex - rep).norm())
  num = float((got.double() - rep).norm())
  return num / den if den > 0 else None


def _dev(case):
  return 'cuda' if case[0] * case[2] * case[1] ** 2 >= 1 << 20 else 'cpu'


@pytest.fixture(scope='module')
def lib():
  import __graft_entry__ as g
  g.build()
  from ranking_b200 import _C
  return _C


@pytest.mark.gpu
@pytest.mark.parametrize('case', CASES, ids=_id)
def test_core_against_the_bf16_replay(lib, case):
  b, n, H, h, kind, drop, sigma = case
  E = H * h
  qkv, mask, dO = _inputs(case)
  got = run_kernel(case, qkv, mask, dO)
  again = run_kernel(case, qkv, mask, dO)
  for k in got:   # identical calls give identical bits
    assert torch.equal(got[k], again[k]), k
  dev = _dev(case)
  rep_o, rep_g = replay(case, qkv, mask, dO, dev=dev)
  ex_o, ex_g = replay(case, qkv, mask, dO, rounding=False, dev=dev)
  bars = B.attn_bars(qkv.to(dev).double(), mask, H, dO.to(dev).double(), rep_o, drop,
                     *_seed(case))
  gt = _tensors(got['O'].to(dev).double(), got['dqkv'].to(dev).double(), E)
  rt = _tensors(rep_o, rep_g, E)
  et = _tensors(ex_o, ex_g, E)
  worst, ratios = {}, {}
  for k in gt:
    err = (gt[k] - rt[k]).abs()
    worst[k] = float((err / bars[k].clamp(min=1e-300)).max()) if err.max() > 0 else 0.0
    assert (err <= bars[k]).all(), (k, worst[k])
    ratios[k] = _rms_ratio(gt[k], rt[k], et[k])
  print('[attn bf16 %s] err/bar %s; RMS ratio %s (limit %.3f)' %
        (_id(case), ' '.join('%s %.3f' % kv for kv in worst.items()),
         ' '.join('%s %s' % (k, 'n/a' if r is None else '%.4f' % r) for k, r in ratios.items()),
         RATIO))
  assert all(r is None or r <= RATIO for r in ratios.values()), ratios
  # lse: the row max against the fp64 max of the fp32 masked logits, 1 / sum to fp32 accuracy
  m_ref, inv_ref, m_tol, inv_tol = B.attn_lse(qkv.to(dev).double(), mask, H)
  lse = got['lse'].to(dev).double()
  assert ((lse[..., 0] - m_ref).abs() <= m_tol).all(), float((lse[..., 0] - m_ref).abs().max())
  assert ((lse[..., 1] - inv_ref).abs() <= inv_tol).all(), \
      float(((lse[..., 1] - inv_ref).abs() / inv_tol).max())
  # dsum: dO . O over the stored bf16 values, within h 2^-24 of sum |dO| |O|
  do = dO.to(dev).double().reshape(b, n, H, h)
  oo = got['O'].to(dev).double().reshape(b, n, H, h)
  want = (do * oo).sum(-1)
  tol = h * 2.0 ** -24 * (do.abs() * oo.abs()).sum(-1)
  assert ((got['dsum'].to(dev).double() - want).abs() <= tol).all()
  # exact cases
  if kind == 'null':
    ones = run_kernel(case, qkv, mask, dO, lmask='ones')
    for k in got:
      assert torch.equal(got[k], ones[k]), k
  if kind == 'single' and drop == 0:
    v = qkv.reshape(b, n, 3 * E)[..., 2 * E:]
    for i in range(b):
      j = 0 if i % 2 == 0 else n - 1
      assert torch.equal(got['O'][i].cpu(), v[i, j].expand(n, E)), i
  if mask is not None:
    for i in range(b):
      if not mask[i].any():   # exact for a list with no valid item
        inv = got['lse'][i, ..., 1].cpu()
        assert torch.equal(inv, torch.full_like(inv, float(np.float32(1.0 / n)))), i


def test_cases_cover_every_variant():
  """Every bucket, a padded head size in each, both sides of each bucket edge, both forward
  paths (one key tile, N <= 64, and several) and both sides of the 64-row tiles, H h = 1024,
  every mask kind, dropout on and off, the large-logit case."""
  pairs, last = _bucket_src()
  hs = {c[3] for c in CASES}
  buckets = {hp for _, hp in pairs} | {last}
  assert buckets == {16, 32, 64, 128}
  assert {bucket(h) for h in hs} == buckets
  for hp in buckets:
    assert any(bucket(h) == hp and h < hp for h in hs), hp   # a padded head size
    assert hp in hs
  for edge, _ in pairs:
    assert any(h <= edge and bucket(h) == bucket(edge) for h in hs)
    assert any(h > edge and bucket(h) != bucket(edge) for h in hs)
  assert hs >= {8, 16, 24, 32, 40, 64, 72, 120, 128}
  ns = {c[1] for c in CASES}
  assert ns >= {1, 2, 63, 64, 65, 127, 128, 129, 511, 512, 1024}
  assert any(n <= ROWS for n in ns) and any(n > ROWS for n in ns)
  assert any(n > ROWS and n % ROWS for n in ns) and any(n > ROWS and n % ROWS == 0 for n in ns)
  assert any(c[2] * c[3] == 1024 and c[1] == 1024 for c in CASES)
  assert max(c[2] for c in CASES) == 16
  assert {c[4] for c in CASES} == {'ragged', 'padded', 'single', 'null'}
  assert any(c[5] == 0 for c in CASES) and {c[5] for c in CASES if c[5]} >= {0.1, 0.2, 0.3}
  assert any(c[6] >= 4 for c in CASES)
  # every bucket on both forward paths
  for hp in buckets:
    assert any(bucket(c[3]) == hp and c[1] > ROWS for c in CASES), hp


def test_replay_without_rounding_is_softmax_attention():
  """B.attention with rounding off is plain fp64 softmax attention (with the -1e9 adder and
  the dropout keep), values and gradients."""
  S, L, H, dh = 3, 7, 2, 8
  E = H * dh
  g = torch.Generator().manual_seed(4)
  qkv = torch.randn(S, L, 3 * E, generator=g, dtype=torch.float64)
  mask = (torch.rand(S, L, generator=g) < 0.6).to(torch.uint8)
  mask[0] = 1
  mask[2] = 0
  dO = torch.randn(S, L, E, generator=g, dtype=torch.float64)
  seed, site, rate = 3, 5, 0.25
  x1 = qkv.clone().requires_grad_()
  o1 = B.attention(x1, mask, H, rate, seed, site, rounding=False)
  o1.backward(dO)
  x2 = qkv.clone().requires_grad_()
  q, k, v = [x2[..., i * E:(i + 1) * E].reshape(S, L, H, dh).permute(0, 2, 1, 3)
             for i in range(3)]
  s = torch.einsum('bhid,bhjd->bhij', q, k) / math.sqrt(dh)
  # Keras' rule: the -1e9 adder in fp32, so a list with no valid key attends 1 / L
  s = torch.where(mask[:, None, None, :] != 0, s, (s.float() - 1e9).double())
  p = torch.exp(s - s.max(-1, keepdim=True).values)
  p = p / p.sum(-1, keepdim=True)
  from oracle import din as odin
  u = odin.uniform(seed, site, S * H * L * L).reshape(S, H, L, L)
  keep = torch.from_numpy((u >= np.float32(rate)).astype(np.float64)) / (1 - float(np.float32(rate)))
  o2 = torch.einsum('bhij,bhjd->bhid', p * keep, v).permute(0, 2, 1, 3).reshape(S, L, E)
  o2.backward(dO)
  assert torch.allclose(o1, o2, rtol=1e-12, atol=1e-12)
  assert torch.allclose(x1.grad, x2.grad, rtol=1e-10, atol=1e-12)
  # the all-padded list attends 1 / L to every key before dropout
  assert torch.equal(p[2], torch.full_like(p[2], 1.0 / L))
  # and with rounding on, the outputs sit on the bf16 grid
  x3 = qkv.clone().requires_grad_()
  o3 = B.attention(x3, mask, H, rate, seed, site)
  assert torch.equal(o3, B.bf16(o3)) and not torch.equal(o3, o1)


# ----------------------------------------------------------------- negative controls ---
CONTROL_CASE = (3, 63, 2, 24, 'ragged', 0.2, 1.0)   # 1 / sqrt(24) is not a power of two
CONTROLS = {
    'no_p_rounding': dict(skip=('p',)),
    'd_i_from_unrounded_pv': dict(skip=('d_i',)),
    'ds_scaled_before_rounding': dict(ds_scaled_first=True),
    'dropout_i_j_swapped': dict(swap_ij=True),
    'mask_ignored': dict(mask_logits=False),
}


def _fails(case, got, ctrl_kw):
  """(fails, description): a control replay against the kernel, with the true replay's bars
  and ratio denominators."""
  b, n, H, h, _, drop, _ = case
  E = H * h
  qkv, mask, dO = _inputs(case)
  rep_o, rep_g = replay(case, qkv, mask, dO)
  ex_o, ex_g = replay(case, qkv, mask, dO, rounding=False)
  c_o, c_g = replay(case, qkv, mask, dO, **ctrl_kw)
  bars = B.attn_bars(qkv.double(), mask, H, dO.double(), rep_o, drop, *_seed(case))
  gt = _tensors(got['O'].cpu().double(), got['dqkv'].cpu().double(), E)
  rt, et, ct = _tensors(rep_o, rep_g, E), _tensors(ex_o, ex_g, E), _tensors(c_o, c_g, E)
  out = []
  for k in gt:
    over = float(((gt[k] - ct[k]).abs() - bars[k]).max())
    den = float((et[k] - rt[k]).norm())
    ratio = float((gt[k] - ct[k]).norm()) / den
    out.append((k, over > 0, ratio))
  return any(o or r > RATIO for _, o, r in out), out


@pytest.mark.gpu
@pytest.mark.parametrize('control', sorted(CONTROLS))
def test_negative_control_fails(lib, control):
  qkv, mask, dO = _inputs(CONTROL_CASE)
  got = run_kernel(CONTROL_CASE, qkv, mask, dO)
  fails, out = _fails(CONTROL_CASE, got, CONTROLS[control])
  print('[attn bf16 control %s] %s' % (
      control, ' '.join('%s %s ratio %.3f' % (k, 'over-bar' if o else 'in-bar', r)
                        for k, o, r in out)))
  assert fails, out


# ------------------------------------------------------------------- argument checks ---
def test_entry_rejects_bad_arguments_before_any_cuda_call(lib):
  _C = lib
  p = ctypes.c_void_p(1 << 20)      # never dereferenced
  odd = ctypes.c_void_p((1 << 20) + 8)
  good = dict(qkv=p, B=2, N=8, H=2, h=16, drop=0.1, O=p, lse=p, dO=p, dsum=p, dqkv=p)

  def fwd(a):
    return _C.lib.tfr_attn_bf16_fwd(a['qkv'], None, a['B'], a['N'], a['H'], a['h'], a['drop'], 1,
                                    a['O'], a['lse'], None)

  def bwd(a):
    return _C.lib.tfr_attn_bf16_bwd(a['qkv'], None, a['B'], a['N'], a['H'], a['h'], a['drop'], 1,
                                    a['O'], a['lse'], a['dO'], a['dsum'], a['dqkv'], None)

  bad = [dict(qkv=None), dict(O=None), dict(lse=None), dict(h=0), dict(h=4), dict(h=12),
         dict(h=136), dict(h=-8), dict(N=0), dict(N=1025), dict(H=0), dict(H=9, h=128),
         dict(H=130, h=8), dict(B=-1), dict(drop=-0.1), dict(drop=1.0), dict(drop=float('nan')),
         dict(qkv=odd), dict(O=odd), dict(lse=odd)]
  bad_bwd = [dict(dO=None), dict(dsum=None), dict(dqkv=None), dict(dO=odd), dict(dsum=odd),
             dict(dqkv=odd)]
  n0 = _C.lib.tfr_launch_count()
  for d in bad:
    a = dict(good, **d)
    assert fwd(a) == INVALID_ARGUMENT, d
    assert _C.last_error().startswith('bf16 attention'), (d, _C.last_error())
    assert bwd(a) == INVALID_ARGUMENT, d
  for d in bad_bwd:
    assert bwd(dict(good, **d)) == INVALID_ARGUMENT, d
  # B = 0: nothing to do, nothing launched
  assert fwd(dict(good, B=0)) == 0 and bwd(dict(good, B=0)) == 0
  assert _C.lib.tfr_launch_count() == n0
