"""The groupwise path on the GPU (csrc/mlp_group.cu), stage by stage and end to end.

  * Group formation (tfr_group_indices) and circular padding (tfr_circular_pad_gather) against
    tests/_group_refs.form_groups, exactly, across the 256-item chunks of the partition kernel,
    and their argument checks (nothing launched).
  * The folded tower (tfr_group_mlp_fwd / bwd) in tf32x3 and tf32, with ReLU and no activation,
    on towers at the fused forward's limits and just past them.  Every stage is replayed in fp32
    and must match bit for bit: the groups, each P_j (a tfr_tc_gemm over slot j's rows of W_0),
    H_0 and its sign words (bias, then the slots in order), the later layers from that H_0
    (first_layer = 1), the scatter-mean, dgscore and every dP_j.  Then the logits, the softmax
    loss over them and the whole parameter gradient meet the fp64 bound of _group_refs, with the
    gates taken from the kernel's H_d and checked for admissibility.
  * The fold with gs = 1 gives tfr_mlp_fwd's scores bit for bit.
  * GroupwiseRankingTrainer: one Adagrad step against the fp64 chain; its groups, predict(),
    a change of shape and reproducibility.
  * tfr_group_mlp_check's flags, and an index outside the list (guarded: never dereferenced).
  * Negative controls: defective references fail their bound; a reversed-order gather replay
    fails the exact check.

Each case prints its err / bound ratios; the worst per tower and quantity is printed when the
module ends (pytest -s).
"""
import ctypes
import zlib

import pytest
import torch

import _group_refs as GR
import _tower_fp64 as R
from _tower_refs import kernel_launches
from test_tower_fused_bwd_gpu import _floats, _layout
from test_tower_fused_fwd_gpu import _assert_same_bits

pytestmark = pytest.mark.gpu

WORST = {}
FUSED_KERNEL = 'tower_fused_fwd_kernel'

# name: (D, group_size, hidden widths)
TOWERS = {
    'config4': (512, 2, [256, 128, 64]),    # fused forward from layer 1
    'gs1': (136, 1, [256, 128, 64]),        # group_size 1
    'd12_gs3': (12, 3, [36, 16]),           # D % 8 != 0; h1 = 36: a partial sign word
    'gs8': (4, 8, [100, 8]),                # output_units at its limit
    'one_hidden': (16, 2, [32]),            # no layer between the fold and the output layer
    'long_k1': (8, 2, [1024, 64]),          # 32 k blocks in the fused kernel's first segment
    'past_260': (20, 2, [64, 260, 64]),     # dims[2] > 256: per-layer path
    'past_132': (20, 2, [64, 128, 132]),    # dims[L] > 128: per-layer path
}
FUSED_TF32X3 = ('config4', 'gs1', 'd12_gs3', 'gs8', 'long_k1')

# name: (B, N, S, shuffled, valid counts cycled over the lists (None: random), x offset)
SHAPES = {
    'bg1': (1, 1, 1, False, [1], 0),
    'bg127': (1, 127, 1, False, None, 0),
    'bg129': (3, 43, 1, False, 'edges', 0),
    'S2_perm': (5, 37, 2, True, 'edges', 0),
    'S3': (5, 20, 3, False, 'edges', 0),
}


@pytest.fixture(autouse=True, scope='module')
def _report():
  yield
  for key in sorted(WORST):
    print('\nworst err / bound, %s: %.3g (%s)' % (key, *WORST[key]))


@pytest.fixture(autouse=True)
def _need_cuda():
  if not torch.cuda.is_available():
    pytest.skip('no CUDA device')


def _lib():
  import __graft_entry__ as entry
  entry.build()
  from ranking_b200 import _C
  return _C


def _sms():
  return torch.cuda.get_device_properties(0).multi_processor_count


def _prec(_C, precision):
  return {'tf32x3': _C.PREC_TF32X3, 'tf32': _C.PREC_TF32}[precision]


def _tower(precision, D, gs, hidden, act, seed):
  import ranking_b200 as tfr
  t = tfr.keras.layers.create_tower(hidden, gs, activation=act, use_batch_norm=False, dropout=0,
                                    input_dim=gs * D, seed=seed, precision=precision)
  g = torch.Generator().manual_seed(seed)
  with torch.no_grad():
    for i in range(len(t.dims) - 1):
      t.bias(i).copy_(torch.rand(t.dims[i + 1], generator=g) * 0.4 - 0.2)
  return t


def _valid(B, N, gs, counts, g):
  """[B, N] bool on the device: list b has counts[b % len] valid items at random positions."""
  if counts == 'edges':
    counts = [0, 1, max(gs - 1, 1), gs, N]
  valid = torch.zeros(B, N, dtype=torch.bool)
  for b in range(B):
    nv = int(torch.randint(0, N + 1, (1,), generator=g)) if counts is None else counts[b % len(counts)]
    valid[b, torch.randperm(N, generator=g)[:min(nv, N)]] = True
  return valid.cuda()


def _perms(valid, S, g, full=False):
  """[S, B, N] int32 shuffles of the valid-first order: of the valid prefix, or of everything."""
  B, N = valid.shape
  out = torch.arange(N).repeat(S, B, 1)
  for s in range(S):
    for b in range(B):
      k = N if full else int(valid[b].sum())
      out[s, b, :k] = torch.randperm(k, generator=g)
  return out.to(torch.int32).cuda()


def _split_t(w):
  """W^T [out, in] split into the RN-TF32 hi part and the fp32 residual (split_params_kernel)."""
  w_t = w.detach().t().contiguous()
  hi = ((w_t.view(torch.int32) + 4096) & -8192).view(torch.float32)
  return hi, w_t - hi


def _gemm(_C, a, w, passes, bias=None, relu=False, bits=None, w_split=None, k0=None, kc=None):
  """out = a @ w[k0:k0 + kc] (+ bias, act) through tfr_tc_gemm with the operands the tower
  passes: 3xTF32 reads W^T pre-split (K-major, ld = all of W's rows), TF32 reads W as is."""
  K, n = w.shape
  k0, kc = (0, K) if k0 is None else (k0, kc)
  m = a.shape[0]
  out = torch.empty(m, n, device='cuda')
  epi = 1 if bias is not None else 0
  if passes == 3:
    hi, lo = w_split if w_split is not None else _split_t(w)
    args = (_C.ptr(hi[:, k0:]), K, _C.ptr(lo[:, k0:]), 0)
  else:
    args = (_C.ptr(w[k0:]), n, None, 1)
  _C.check(_C.lib.tfr_tc_gemm(
      _C.ptr(a), kc, args[0], args[1], args[2], _C.ptr(out), n, m, n, kc, 0, args[3], passes, 0,
      epi, _C.ptr(bias), None, 1 if relu else 0, 0, 1, 0, _C.ptr(bits), None, _C.stream()))
  return out


def _sign_words(h):
  """ReLU sign words of H [M, n]: word [(col / 32) M + r], bit col % 32 set where H > 0."""
  m, n = h.shape
  nw = (n + 31) // 32
  pos = torch.zeros(m, nw * 32, dtype=torch.int64, device=h.device)
  pos[:, :n] = (h > 0).long()
  w = (pos.view(m, nw, 32) << torch.arange(32, device=h.device)).sum(2)
  return w.t().contiguous().to(torch.int64) & 0xFFFFFFFF


def _as_u32(bits):
  return bits.to(torch.int64) & 0xFFFFFFFF


class GroupRun(object):
  """One tfr_group_mlp_fwd + bwd through the C ABI with every workspace region read back."""

  def __init__(self, _C, tower, precision, x, valid, S, perms, dlogits, idx=None, gmask=None):
    B, N, D = x.shape
    gs = tower.output_units
    G, M = S * N, B * S * N
    self.B, self.N, self.S, self.gs, self.M = B, N, S, gs, M
    prec = _prec(_C, precision)
    if idx is None:
      idx = torch.empty(B, G, gs, dtype=torch.int32, device='cuda')
      gmask = torch.empty(B, G, dtype=torch.uint8, device='cuda')
      _C.check(_C.lib.tfr_group_indices(_C.ptr(valid.to(torch.uint8).contiguous()), _C.ptr(perms),
                                        B, N, S, gs, _C.ptr(idx), _C.ptr(gmask), _C.stream()))
    self.idx, self.gmask = idx, gmask
    cfg = tower._run_cfg()
    nbytes = _C.lib.tfr_group_mlp_workspace_bytes(ctypes.byref(cfg), B, N, G, gs)
    assert nbytes > 0, _C.last_error()
    self.ws = torch.empty(nbytes, dtype=torch.uint8, device='cuda')
    self.logits_buf = torch.full((B * N + 64,), 12345.0, device='cuda')
    self.logits = self.logits_buf[:B * N].view(B, N)
    self.grads = torch.full_like(tower.flat.data, float('nan'))
    args = (_C.ptr(x), B, N, G, gs, _C.ptr(idx), _C.ptr(gmask), ctypes.byref(cfg),
            _C.ptr(tower.flat.data))
    self.fwd = lambda: _C.check(_C.lib.tfr_group_mlp_fwd(*args, _C.ptr(self.ws),
                                                         _C.ptr(self.logits), prec, _C.stream()))
    self.bwd = lambda: _C.check(_C.lib.tfr_group_mlp_bwd(*args, _C.ptr(dlogits), _C.ptr(self.ws),
                                                         _C.ptr(self.grads), prec, _C.stream()))
    self.fwd()
    torch.cuda.synchronize()
    flat = _floats(self.ws)
    dims = tower.dims
    L, h1, bn = len(dims) - 2, dims[1], B * N
    lay = _layout(dims, M, _sms())
    self.hidden = [flat[lay['act'][d]:][:M * dims[d + 1]].view(M, dims[d + 1]).clone()
                   for d in range(L)]
    self.bits = [_as_u32(flat[lay['bits'][d]:][:M * ((dims[d + 1] + 31) // 32)]
                         .view(torch.int32).view(-1, M)) for d in range(L)]
    up = lambda n: (n + 63) // 64 * 64
    g0 = (_C.lib.tfr_mlp_workspace_bytes(ctypes.byref(cfg), M) - 256) // 4
    off = {'P': g0}
    off['inv'] = off['P'] + up(gs * bn * h1)
    off['cnt'] = off['inv'] + up(S * bn * gs)
    off['gscore'] = off['cnt'] + up(bn)
    self.off = off
    self._flat = flat
    self.P = [flat[off['P'] + j * bn * h1:][:bn * h1].view(bn, h1).clone() for j in range(gs)]
    self.inv = flat[off['inv']:][:S * bn * gs].view(torch.int32).view(S, B, N, gs).clone()
    self.cnt = flat[off['cnt']:][:bn].view(B, N).clone()
    self.gscore = flat[off['gscore']:][:M * gs].view(M, gs).clone()
    self.logits_fwd = self.logits.clone()
    self.bwd()
    torch.cuda.synchronize()
    self.dgscore = flat[off['gscore']:][:M * gs].view(M, gs).clone()
    self.dP = [flat[off['P'] + j * bn * h1:][:bn * h1].view(bn, h1).clone() for j in range(gs)]
    self.dz0 = flat[lay['dz'][(L - 1) & 1]:][:M * h1].view(M, h1).clone()
    self.grads_first = self.grads.clone()


def _gather_replay(P, idx, bias, N, relu, reverse=False):
  """H_0 in fp32: the bias, then P_j at each member's row for j = 0 .. gs - 1 (or reversed)."""
  B, G, gs = idx.shape
  rows = (torch.arange(B, device='cuda')[:, None, None] * N + idx.long()).reshape(B * G, gs)
  acc = bias.detach().expand(B * G, -1).clone()
  for j in (range(gs - 1, -1, -1) if reverse else range(gs)):
    acc = acc + P[j][rows[:, j]]
  return torch.relu(acc) if relu else acc


def _check_stages(_C, tower, precision, act, run, x, valid, S, perms, dlogits):
  """Stages 1-6: the groups, P_j, H_0, the later layers, the scatter-mean, dgscore, dP_j."""
  import ranking_b200 as tfr
  B, N, D = x.shape
  gs, M = run.gs, run.M
  passes = 3 if precision == 'tf32x3' else 1
  relu = act == 'relu'
  dims, L = tower.dims, len(tower.dims) - 2
  # 1. groups
  idx, gmask, inv, cnt = GR.form_groups(valid, gs, perms, S)
  _assert_same_bits(run.idx.long(), idx, 'idx')
  _assert_same_bits(run.gmask.bool(), gmask, 'gmask')
  _assert_same_bits(run.inv.long(), inv, 'inv')
  _assert_same_bits(run.cnt, cnt.float(), 'cnt')
  # 2. P_j: slot j's rows of W_0
  w0 = tower.kernel(0).detach()
  split = _split_t(w0) if passes == 3 else None
  xf = x.reshape(B * N, D)
  for j in range(gs):
    _assert_same_bits(run.P[j], _gemm(_C, xf, w0, passes, w_split=split, k0=j * D, kc=D),
                      'P_%d' % j)
  # 3. H_0 and its sign words
  h0 = _gather_replay(run.P, run.idx, tower.bias(0), N, relu)
  _assert_same_bits(run.hidden[0], h0, 'H_0')
  if relu:
    _assert_same_bits(run.bits[0], _sign_words(h0), 'sign words of H_0')
  # 4. layers 1 .. L-1 and the member scores from the kernel's H_0
  h = run.hidden[0]
  for d in range(1, L):
    bits = torch.empty((dims[d + 1] + 31) // 32, M, dtype=torch.int32, device='cuda')
    h = _gemm(_C, h, tower.kernel(d).detach(), passes, bias=tower.bias(d).detach(), relu=relu,
              bits=bits if relu else None)
    _assert_same_bits(run.hidden[d], h, 'H_%d' % d)
    if relu:
      _assert_same_bits(run.bits[d], _as_u32(bits), 'sign words of H_%d' % d)
  head = tfr.keras.layers.create_tower([], gs, input_dim=dims[L], precision='fp32')
  head.load_keras_weights([tower.kernel(L).detach().cpu()], [tower.bias(L).detach().cpu()])
  with torch.no_grad():
    gscore = head(run.hidden[L - 1])
  torch.cuda.synchronize()
  _assert_same_bits(run.gscore, gscore, 'member scores')
  # 5. scatter-mean in (s, j) order, divided by the count
  acc = torch.zeros(B, N, device='cuda')
  sc = run.gscore.view(B, S * N, gs)
  bb = torch.arange(B, device='cuda')[:, None].expand(B, N)
  for s in range(S):
    for j in range(gs):
      g = inv[s, :, :, j]
      acc = torch.where(g >= 0, acc + sc[bb, g.clamp(min=0), j], acc)
  c = cnt.float()
  _assert_same_bits(run.logits_fwd, torch.where(c > 0, acc / c, torch.zeros_like(acc)), 'logits')
  assert (run.logits_fwd[cnt == 0] == 0).all()
  # 6. dgscore, dP_j
  fi = run.idx.long().reshape(B, -1)
  dg = torch.gather(dlogits, 1, fi) / torch.gather(c, 1, fi)
  dg = torch.where(gmask[:, :, None].expand(-1, -1, gs).reshape(B, -1), dg, torch.zeros_like(dg))
  _assert_same_bits(run.dgscore, dg.reshape(M, gs), 'dgscore')
  dz = run.dz0.view(B, S * N, -1)
  for j in range(gs):
    acc = torch.zeros(B, N, dims[1], device='cuda')
    for s in range(S):
      g = inv[s, :, :, j]
      acc = torch.where((g >= 0)[..., None], acc + dz[bb, g.clamp(min=0)], acc)
    _assert_same_bits(run.dP[j], acc.reshape(B * N, -1), 'dP_%d' % j)
  return idx, gmask, inv, cnt


def _loss_ratio(labels, got_logits, ref_logits, mag, u):
  """|softmax loss at the kernel's logits - at the exact ones| over C u sum |dL/dl| mag(l)."""
  from oracle import keras_losses as OK
  y = labels.detach().cpu().double()
  lg = ref_logits.detach().cpu().clone().requires_grad_()
  ref = OK.SoftmaxLoss()(y, lg)
  ref.backward()
  got = OK.SoftmaxLoss()(y, got_logits.detach().cpu().double())
  err = abs(float(got) - float(ref.detach()))
  bound = R.C * u * float((lg.grad.abs() * mag.detach().cpu()).sum())
  return 0.0 if err == 0 else err / bound


def _record(key, name, ratios):
  print('%s: %s' % (name, ', '.join('%s %.3g' % r for r in ratios)))
  for what, ratio in ratios:
    k = '%s %s' % (key, what)
    if ratio > WORST.get(k, (-1.0, ''))[0]:
      WORST[k] = (ratio, name)


def _params(tower):
  L = len(tower.dims) - 2
  return {'w': [tower.kernel(i).detach() for i in range(L + 1)],
          'b': [tower.bias(i).detach() for i in range(L + 1)]}


def run_case(name, precision, act, B, N, S, shuffled, counts, x_offset=0, full_perms=False):
  """Stages 1-8 bit for bit, then the fp64 bound on logits, loss and gradient."""
  _C = _lib()
  D, gs, hidden = TOWERS[name]
  seed = zlib.crc32(repr((name, precision, act, B, N, S)).encode()) & 0xFFFF
  tower = _tower(precision, D, gs, hidden, act, seed)
  g = torch.Generator().manual_seed(seed + 1)
  valid = _valid(B, N, gs, counts, g)
  perms = _perms(valid, S, g, full_perms) if shuffled else None
  store = torch.empty(B * N * D + 4, device='cuda')
  x = store[x_offset:x_offset + B * N * D].view(B, N, D)
  x.copy_(torch.randn(B, N, D, generator=g))
  labels = torch.where(valid.cpu(), torch.randint(0, 5, (B, N), generator=g).float(),
                       torch.full((B, N), -1.0))
  dlogits = torch.randn(B, N, generator=g).cuda()
  run = GroupRun(_C, tower, precision, x, valid, S, perms, dlogits)
  groups = _check_stages(_C, tower, precision, act, run, x, valid, S, perms, dlogits)
  # 7. a second identical call gives the same bits; 8. nothing past the logits, no NaN left
  run.fwd()
  run.bwd()
  torch.cuda.synchronize()
  _assert_same_bits(run.logits, run.logits_fwd, 'logits (second call)')
  _assert_same_bits(run.grads, run.grads_first, 'grads (second call)')
  assert (run.logits_buf[B * N:] == 12345.0).all(), 'the forward wrote past the logits'
  assert not torch.isnan(run.grads).any(), 'the backward left gradient entries unwritten'
  # fp64
  cfg = R.Cfg(tower.dims, relu=act == 'relu')
  ref = GR.forward_backward(x, _params(tower), cfg, R.gates_from(run.hidden, cfg), groups,
                            dlogits)
  bound = GR.Bound(cfg, precision, B, N, S, gs, _sms())
  got = {'hidden': run.hidden, 'logits': run.logits_fwd, 'grads': run.grads}
  ratios = GR.check(cfg, bound, ref, got)
  ratios.append(('loss', _loss_ratio(labels, run.logits_fwd, ref['logits'], ref['mag']['logits'],
                                     bound.logits)))
  label = '%s %s %s B=%d N=%d S=%d%s' % (name, precision, act, B, N, S, ' perm' if shuffled else '')
  _record('%s %s' % (name, precision), label, ratios)
  bad = [(w, r) for w, r in ratios if not r <= 1]
  assert not bad, (label, bad)
  return dict(tower=tower, run=run, ref=ref, bound=bound, cfg=cfg, x=x, groups=groups,
              valid=valid, perms=perms, dlogits=dlogits)


# ------------------------------------------------------------------- group formation ---
PATTERNS = ('none', 'one', 'gs-1', 'all', 'random', 'last', 'past256')


def _pattern_valid(N, gs, g):
  rows = []
  for p in PATTERNS:
    v = torch.zeros(N, dtype=torch.bool)
    if p == 'one':
      v[int(torch.randint(0, N, (1,), generator=g))] = True
    elif p == 'gs-1':
      v[torch.randperm(N, generator=g)[:min(max(gs - 1, 0), N)]] = True
    elif p == 'all':
      v[:] = True
    elif p == 'random':
      v = torch.rand(N, generator=g) < 0.6
    elif p == 'last':
      v[N - 1] = True
    elif p == 'past256':
      v[256:] = torch.rand(max(N - 256, 0), generator=g) < 0.7
    rows.append(v)
  return torch.stack(rows).cuda()


@pytest.mark.parametrize('gs', [1, 2, 3, 8])
@pytest.mark.parametrize('N', [1, 31, 32, 255, 256, 257, 511, 513, 8192])
def test_group_indices_match_reference(N, gs):
  _C = _lib()
  g = torch.Generator().manual_seed(N * 16 + gs)
  valid = _pattern_valid(N, gs, g)
  B = valid.shape[0]
  v8 = valid.to(torch.uint8).contiguous()
  for S in (1, 2, 4):
    for shuffled in (False, True):
      perms = _perms(valid, S, g, full=(S == 2)) if shuffled else None
      idx = torch.full((B, S * N, gs), -7, dtype=torch.int32, device='cuda')
      gmask = torch.full((B, S * N), 7, dtype=torch.uint8, device='cuda')
      _C.check(_C.lib.tfr_group_indices(_C.ptr(v8), _C.ptr(perms), B, N, S, gs, _C.ptr(idx),
                                        _C.ptr(gmask), _C.stream()))
      want_idx, want_mask, _, _ = GR.form_groups(valid, gs, perms, S)
      _assert_same_bits(idx.long(), want_idx, 'idx N=%d S=%d gs=%d' % (N, S, gs))
      _assert_same_bits(gmask.bool(), want_mask, 'gmask N=%d S=%d gs=%d' % (N, S, gs))
      assert (gmask <= 1).all()


def test_group_indices_argument_checks():
  _C = _lib()
  v = torch.ones(2, 8193, dtype=torch.uint8, device='cuda')
  idx = torch.empty(2 * 4 * 8193 * 8, dtype=torch.int32, device='cuda')
  gm = torch.empty(2 * 4 * 8193, dtype=torch.uint8, device='cuda')
  n0 = _C.lib.tfr_launch_count()
  assert _C.lib.tfr_group_indices(_C.ptr(v), None, 0, 8, 1, 2, _C.ptr(idx), _C.ptr(gm),
                                  _C.stream()) == 0
  for B, N, S, gs in [(2, 0, 1, 2), (2, 8193, 1, 2), (2, 8, 1, 0), (2, 8, 0, 2), (-1, 8, 1, 2)]:
    assert _C.lib.tfr_group_indices(_C.ptr(v), None, B, N, S, gs, _C.ptr(idx), _C.ptr(gm),
                                    _C.stream()) != 0, (B, N, S, gs)
  for args in [(None, idx, gm), (v, None, gm), (v, idx, None)]:
    assert _C.lib.tfr_group_indices(_C.ptr(args[0]), None, 2, 8, 1, 2, _C.ptr(args[1]),
                                    _C.ptr(args[2]), _C.stream()) != 0
  assert _C.lib.tfr_launch_count() == n0


@pytest.mark.parametrize('row_bytes', [16, 48, 544, 2048])
@pytest.mark.parametrize('N', [1, 256, 257, 8192])
def test_circular_pad_gather_bytes(N, row_bytes):
  _C = _lib()
  g = torch.Generator().manual_seed(N + row_bytes)
  valid = torch.stack([torch.zeros(N, dtype=torch.bool), torch.ones(N, dtype=torch.bool),
                       torch.rand(N, generator=g) < 0.5,
                       torch.arange(N) >= min(256, N - 1)]).cuda()
  B = valid.shape[0]
  x = torch.randint(0, 256, (B, N, row_bytes), generator=g, dtype=torch.uint8).cuda()
  out = torch.full_like(x, 0xA5)
  idx = torch.full((B, N), -7, dtype=torch.int32, device='cuda')
  _C.check(_C.lib.tfr_circular_pad_gather(_C.ptr(x), _C.ptr(valid.to(torch.uint8).contiguous()),
                                          B, N, row_bytes, _C.ptr(idx), _C.ptr(out), _C.stream()))
  want_idx = GR.form_groups(valid, 1)[0][..., 0]
  _assert_same_bits(idx.long(), want_idx, 'circular padding indices')
  want = torch.gather(x, 1, want_idx[..., None].expand(-1, -1, row_bytes))
  _assert_same_bits(out, want, 'circular padding rows')


def test_circular_pad_gather_rejects_before_launching():
  _C = _lib()
  x = torch.zeros(4096, dtype=torch.uint8, device='cuda')
  v = torch.ones(2, 4, dtype=torch.uint8, device='cuda')
  idx = torch.empty(8, dtype=torch.int32, device='cuda')
  n0 = _C.lib.tfr_launch_count()
  bad = [(x, x, 24), (x[4:], x[2048:], 16), (x, x[2052:], 16), (x, x, 0)]
  for xin, out, rb in bad:
    assert _C.lib.tfr_circular_pad_gather(_C.ptr(xin), _C.ptr(v), 2, 4, rb, _C.ptr(idx),
                                          _C.ptr(out), _C.stream()) != 0, rb
  assert _C.lib.tfr_launch_count() == n0


# ------------------------------------------------------------------------ folded tower ---
@pytest.mark.parametrize('shape', sorted(SHAPES))
@pytest.mark.parametrize('act', ['relu', None])
@pytest.mark.parametrize('precision', ['tf32x3', 'tf32'])
@pytest.mark.parametrize('name', sorted(TOWERS))
def test_folded_tower(name, precision, act, shape):
  B, N, S, shuffled, counts, off = SHAPES[shape]
  run_case(name, precision, act, B, N, S, shuffled, counts, x_offset=off)


@pytest.mark.parametrize('precision', ['tf32x3', 'tf32'])
@pytest.mark.parametrize('name', sorted(TOWERS))
def test_folded_tower_input_at_4_byte_offset(name, precision):
  """X as a contiguous view 4 bytes into its storage: the first layer's GEMMs need 16-byte
  operands, so the forward refuses with ValueError, as the plain tower's TF32 modes do, and
  never faults."""
  try:
    run_case(name, precision, 'relu', 4, 33, 1, False, 'edges', x_offset=1)
  except ValueError as e:
    assert '16-byte' in str(e), e
  torch.cuda.synchronize()


@pytest.mark.parametrize('precision', ['tf32x3', 'tf32'])
@pytest.mark.parametrize('case', [('d12_gs3', 2, 8192, None), ('d12_gs3', 125, 320, 'edges'),
                                  ('config4', 16, 128, 'edges'), ('config4', 256, 128, None)])
def test_folded_tower_large(case, precision):
  """N = 8192; B N = 40000 (about 100 dW_0 splits); a 16-list and a 256-list config-4 chunk."""
  name, B, N, counts = case
  run_case(name, precision, 'relu', B, N, 1, False, counts)
  if B * N == 40000:
    rows, splits = GR.dw0_splits(B * N, R.Plan(R.Cfg([1, 1]), B * N, _sms()))
    assert splits >= 90, splits


@pytest.mark.parametrize('precision', ['tf32x3', 'tf32'])
@pytest.mark.parametrize('name', sorted(TOWERS))
def test_folded_tower_path(name, precision):
  """The fused forward runs from layer 1 exactly where mlp_tc_fused_fwd_ok admits the tower."""
  _C = _lib()
  D, gs, hidden = TOWERS[name]
  tower = _tower(precision, D, gs, hidden, 'relu', seed=3)
  B, N = 3, 43
  g = torch.Generator().manual_seed(4)
  valid = _valid(B, N, gs, 'edges', g)
  x = torch.randn(B, N, D, generator=g).cuda()
  run = GroupRun(_C, tower, precision, x, valid, 1, None, torch.zeros(B, N, device='cuda'))
  _, launches = kernel_launches(run.fwd)
  names = [k for k, _, _ in launches]
  print('%s %s: %s' % (name, precision, ' '.join(names)))
  want_fused = precision == 'tf32x3' and name in FUSED_TF32X3
  assert (FUSED_KERNEL in names) == want_fused, names
  assert 'group_gather_fwd_kernel' in names and 'group_scatter_mean_fwd_kernel' in names


def test_fold_with_group_size_1_matches_plain_tower():
  """gs = 1, S = 1, every item valid: the same operations in the same order as tfr_mlp_fwd."""
  _C = _lib()
  for name, B, N in [('gs1', 16, 128), ('gs1', 3, 43)]:
    D, gs, hidden = TOWERS[name]
    tower = _tower('tf32x3', D, gs, hidden, 'relu', seed=9)
    g = torch.Generator().manual_seed(B)
    x = torch.randn(B, N, D, generator=g).cuda()
    valid = torch.ones(B, N, dtype=torch.bool, device='cuda')
    run = GroupRun(_C, tower, 'tf32x3', x, valid, 1, None, torch.zeros(B, N, device='cuda'))
    with torch.no_grad():
      plain = tower(x.reshape(B * N, D))
    torch.cuda.synchronize()
    _assert_same_bits(run.logits_fwd, plain.view(B, N), 'fold vs tfr_mlp_fwd (%d lists)' % B)


# --------------------------------------------------------------------------- trainer ---
def _trainer_step(tower, B, N, D, gs, S, perms, valid, seed, lr=0.05):
  import ranking_b200 as tfr
  g = torch.Generator().manual_seed(seed)
  x = torch.randn(B, N, D, generator=g).cuda()
  labels = torch.where(valid.cpu(), torch.randint(0, 5, (B, N), generator=g).float(),
                       torch.full((B, N), -1.0)).cuda()
  tr = tfr.train.GroupwiseRankingTrainer(tower, tfr.keras.losses.SoftmaxLoss(), gs,
                                         num_shuffles=S, optimizer='adagrad', learning_rate=lr)
  tr.permutations = perms
  return tr, x, labels


@pytest.mark.parametrize('precision', ['tf32x3', 'tf32'])
@pytest.mark.parametrize('case', [('config4', 16, 128, 1, False, 'edges'),
                                  ('d12_gs3', 3, 13, 1, False, None),
                                  ('gs8', 4, 19, 2, True, 'edges'),
                                  ('one_hidden', 5, 9, 1, False, [0, 3, 9])])
def test_trainer_step_matches_fp64(case, precision):
  """One Adagrad step against the fp64 chain: groups, logits, SoftmaxLoss, gradient, update."""
  from oracle import keras_losses as OK
  from ranking_b200 import model as tfr_model
  name, B, N, S, shuffled, counts = case
  D, gs, hidden = TOWERS[name]
  seed = zlib.crc32(repr(case).encode()) & 0xFFFF
  tower = _tower(precision, D, gs, hidden, 'relu', seed)
  g = torch.Generator().manual_seed(seed)
  valid = _valid(B, N, gs, counts, g)
  if counts is not None:
    assert (valid.sum(1) == 0).any()   # a list with no valid items
  perms = _perms(valid, S, g) if shuffled else None
  tr, x, labels = _trainer_step(tower, B, N, D, gs, S, perms, valid, seed + 1)
  p0 = tower.flat.detach().clone()
  params = {'w': [tower.kernel(i).detach().clone() for i in range(len(tower.dims) - 1)],
            'b': [tower.bias(i).detach().clone() for i in range(len(tower.dims) - 1)]}
  loss = float(tr.train_step(x, labels))
  torch.cuda.synchronize()
  # groups
  groups = GR.form_groups(valid, gs, perms, S)
  _assert_same_bits(tr.idx.long(), groups[0], 'trainer.idx')
  _assert_same_bits(tr.gmask.bool(), groups[1], 'trainer.gmask')
  m_idx = torch.cat([tfr_model._form_group_indices(valid, gs, None if perms is None else
                                                   perms[s].long())[0] for s in range(S)], 1)
  _assert_same_bits(tr.idx.long(), m_idx, 'trainer.idx vs model._form_group_indices')
  # fp64 chain, the loss gradient taken as the trainer's dscores
  cfg = R.Cfg(tower.dims, relu=True)
  M = B * S * N
  hidden = R.hidden_activations(tr.ws, cfg, M)
  ref = GR.forward_backward(x, params, cfg, R.gates_from(hidden, cfg), groups, tr.dscores)
  bound = GR.Bound(cfg, precision, B, N, S, gs, _sms())
  ratios = GR.check(cfg, bound, ref, {'hidden': hidden, 'logits': tr.scores, 'grads': tr.grads})
  ratios.append(('loss', _loss_ratio(labels, tr.scores, ref['logits'], ref['mag']['logits'],
                                     bound.logits)))
  label = 'trainer %s %s B=%d N=%d S=%d' % (name, precision, B, N, S)
  _record('trainer %s' % precision, label, ratios)
  assert all(r <= 1 for _, r in ratios), (label, ratios)
  # the loss kernel: value and gradient at the trainer's own logits
  lg = tr.scores.detach().cpu().double().requires_grad_()
  ref_loss = OK.SoftmaxLoss()(labels.cpu().double(), lg)
  ref_loss.backward()
  assert abs(loss - float(ref_loss)) <= 1e-6 * max(1.0, abs(float(ref_loss))), (loss, ref_loss)
  dl = tr.dscores.detach().cpu().double()
  assert float((dl - lg.grad).abs().max()) <= 1e-6 * max(1e-3, float(lg.grad.abs().max()))
  # the Adagrad update from the trainer's gradient
  gr = tr.grads.detach().double()
  a = 0.1 + gr * gr
  step = 0.05 * gr / (a.sqrt() + 1e-7)
  want = p0.double() - step
  tol = 8 * 2.0 ** -24 * (p0.double().abs() + step.abs()) + 1e-30
  assert bool(((tower.flat.detach().double() - want).abs() <= tol).all())


def test_trainer_predict_shape_change_and_seed():
  import ranking_b200 as tfr
  D, gs, hidden = TOWERS['d12_gs3']
  B, N = 4, 21
  g = torch.Generator().manual_seed(5)
  valid = _valid(B, N, gs, 'edges', g)
  tower = _tower('tf32x3', D, gs, hidden, 'relu', seed=6)
  tr, x, labels = _trainer_step(tower, B, N, D, gs, 1, None, valid, 7)
  # predict without labels: every item valid, the bits of GroupwiseRankingModel
  got = tr.predict(x).clone()
  model = tfr.model.GroupwiseRankingModel(tfr.model.TowerGroupScoreFn(tower), gs)
  with torch.no_grad():
    want = model.compute_logits(x, torch.ones(B, N, dtype=torch.bool, device='cuda'))
  torch.cuda.synchronize()
  _assert_same_bits(got, want, 'predict vs compute_logits')
  # after a change of (B, N), a step gives the bits of a fresh trainer on the same parameters
  tr.train_step(x, labels)
  valid2 = _valid(7, 33, gs, 'edges', g)
  x2 = torch.randn(7, 33, D, generator=g).cuda()
  y2 = torch.where(valid2.cpu(), torch.randint(0, 5, (7, 33), generator=g).float(),
                   torch.full((7, 33), -1.0)).cuda()
  twin = _tower('tf32x3', D, gs, hidden, 'relu', seed=6)
  with torch.no_grad():
    twin.flat.copy_(tower.flat)
  fresh, _, _ = _trainer_step(twin, 7, 33, D, gs, 1, None, valid2, 7)
  l1 = tr.train_step(x2, y2)
  l2 = fresh.train_step(x2, y2)
  torch.cuda.synchronize()
  _assert_same_bits(tr.scores, fresh.scores, 'logits after a shape change')
  _assert_same_bits(tr.grads, fresh.grads, 'gradient after a shape change')
  assert float(l1) == float(l2)
  # two trainers with the same seed: identical parameters after three steps
  flats = []
  for _ in range(2):
    t = _tower('tf32x3', D, gs, hidden, 'relu', seed=11)
    trn, _, _ = _trainer_step(t, B, N, D, gs, 1, None, valid, 7)
    for _ in range(3):
      trn.train_step(x, labels)
    torch.cuda.synchronize()
    flats.append(t.flat.detach().clone())
  _assert_same_bits(flats[0], flats[1], 'parameters after three steps')


# ------------------------------------------------------------------------ check flags ---
def _check_rc(_C, tower, run, B, N, S):
  cfg = tower._run_cfg()
  rc = _C.lib.tfr_group_mlp_check(ctypes.byref(cfg), B, N, S * N, tower.output_units,
                                  _C.ptr(run.ws), _C.stream())
  return rc, (_C.last_error() if rc else '')


def test_group_check_flags():
  _C = _lib()
  D, gs, hidden = TOWERS['d12_gs3']
  tower = _tower('tf32x3', D, gs, hidden, 'relu', seed=12)
  B, N, S = 5, 11, 2
  g = torch.Generator().manual_seed(13)
  valid = _valid(B, N, gs, [0, 1, 2, 3, 11], g)   # nv = 0 and nv < gs included
  x = torch.randn(B, N, D, generator=g).cuda()
  dlogits = torch.randn(B, N, generator=g).cuda()
  run = GroupRun(_C, tower, 'tf32x3', x, valid, S, None, dlogits)
  assert _check_rc(_C, tower, run, B, N, S) == (0, '')
  # one item in the same slot of two valid groups of one shuffle: flag 1
  idx = run.idx.clone()
  gm = run.gmask.clone()
  assert bool(gm[4, 0]) and bool(gm[4, 1])
  idx[4, 1, 0] = idx[4, 0, 0]
  dup = GroupRun(_C, tower, 'tf32x3', x, valid, S, None, dlogits, idx=idx, gmask=gm)
  rc, msg = _check_rc(_C, tower, dup, B, N, S)
  assert rc != 0 and 'same slot' in msg, (rc, msg)
  # an index of N or -1 in a valid group: flag 2; it adds nothing and its gradient is 0
  for bad in (N, -1):
    idx = run.idx.clone()
    idx[3, S * N - N + 1, 1] = bad          # list 3 (nv = 3), shuffle 1, group 1, slot 1
    assert bool(gm[3, S * N - N + 1])
    out = GroupRun(_C, tower, 'tf32x3', x, valid, S, None, dlogits, idx=idx, gmask=gm)
    rc, msg = _check_rc(_C, tower, out, B, N, S)
    assert rc != 0 and 'outside' in msg, (rc, msg)
    r = 3 * S * N + S * N - N + 1
    P = [p.clone() for p in out.P]
    safe = idx.clone()
    safe[3, S * N - N + 1, 1] = 0
    h0 = _gather_replay(P, safe, tower.bias(0), N, True)
    keep = torch.ones(B * S * N, dtype=torch.bool, device='cuda')
    keep[r] = False
    _assert_same_bits(out.hidden[0][keep], h0[keep], 'H_0 of the other groups')
    acc = tower.bias(0).detach().clone()
    for j in range(gs):
      if j != 1:
        acc = acc + P[j][3 * N + int(safe[3, S * N - N + 1, j])]
    _assert_same_bits(out.hidden[0][r], torch.relu(acc), 'H_0 of the group with a bad index')
    assert float(out.dgscore[r, 1]) == 0.0
    assert not torch.isnan(out.grads).any()


# ------------------------------------------------------------------ negative controls ---
def test_negative_controls_fail():
  """Each defective reference fails the bound that the kernel meets; a gather replay that adds
  the slots in reverse order fails the exact check."""
  # a config-4 tower (gs = 2) on lists with nv < N, and shuffles that bring different items
  # into the valid groups, so that the counts vary
  c = run_case('config4', 'tf32x3', 'relu', 8, 128, 2, True, 'edges', full_perms=True)
  groups = c['groups']
  assert ((groups[3] != 0) & (groups[3] != 2 * 2)).any()
  run, cfg = c['run'], c['cfg']
  got = {'hidden': run.hidden, 'logits': run.logits_fwd, 'grads': run.grads}
  gates = R.gates_from(run.hidden, cfg)
  for defect in ('swap_slots', 'divide_by_S_gs', 'wrap_at_n', 'no_bias0'):
    g = groups
    if defect == 'wrap_at_n':
      g = GR.form_groups(c['valid'], 2, c['perms'], wrap_at_n=True)
    bad = GR.forward_backward(c['x'], _params(c['tower']), cfg, gates, g, c['dlogits'],
                              defect=None if defect == 'wrap_at_n' else defect)
    ratios = GR.check(cfg, c['bound'], bad, got)
    print('negative control %s: %s' % (defect, ', '.join('%s %.3g' % r for r in ratios)))
    assert max(r for _, r in ratios) > 1, defect
  # the gather replayed with the slots in reverse order, on a 16-list config-4 chunk
  c = run_case('config4', 'tf32x3', 'relu', 16, 128, 1, False, 'edges')
  run = c['run']
  rev = _gather_replay(run.P, run.idx, c['tower'].bias(0), 128, True, reverse=True)
  differ = int((rev != run.hidden[0]).sum())
  print('reversed gather: %d of %d elements of H_0 differ' % (differ, rev.numel()))
  assert differ > 0
