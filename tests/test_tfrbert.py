"""TFR-BERT on the CPU: the fp64 reference against an independent composition of torch's
TransformerEncoderLayer, the AdamW rule, the learning-rate schedule, the ELWC loader and the
new C ABI symbols."""
import ctypes
import math

import numpy as np
import pytest
import torch

import _tfrbert_refs as R
from ranking_b200 import _C
from ranking_b200 import data
from ranking_b200 import train
from ranking_b200.extension import tfrbert


def _flat(V, E, I, NL, P, Tv, seed=0):
  g = torch.Generator().manual_seed(seed)
  parts = []
  for name, shape in R.weight_shapes(V, E, I, NL, P, Tv):
    if '_g' in name and name.startswith('ln'):
      parts.append(1.0 + 0.1 * torch.randn(shape, generator=g, dtype=torch.float64))
    else:
      parts.append(0.3 * torch.randn(shape, generator=g, dtype=torch.float64))
  return torch.cat([p.reshape(-1) for p in parts])


def _composed(wid, mask, tid, flat, V, E, H, I, NL, P, Tv):
  """The same encoder from torch.nn.TransformerEncoderLayer (post-LN, tanh GELU) with copied
  weights and src_key_padding_mask."""
  p = R.unflatten(flat, V, E, I, NL, P, Tv)
  S, L = wid.shape
  x = p['word'][wid.long()] + p['pos'][:L] + p['type'][tid.long()]
  x = torch.nn.functional.layer_norm(x, (E,), p['ln_e_g'], p['ln_e_b'], eps=1e-12)
  for l in range(NL):
    layer = torch.nn.TransformerEncoderLayer(
        E, H, dim_feedforward=I, dropout=0.0, activation=lambda u: torch.nn.functional.gelu(
            u, approximate='tanh'), layer_norm_eps=1e-12, batch_first=True, norm_first=False,
        dtype=torch.float64)
    with torch.no_grad():
      layer.self_attn.in_proj_weight.copy_(p['wqkv%d' % l].t())
      layer.self_attn.in_proj_bias.copy_(p['bqkv%d' % l])
      layer.self_attn.out_proj.weight.copy_(p['wo%d' % l].t())
      layer.self_attn.out_proj.bias.copy_(p['bo%d' % l])
      layer.norm1.weight.copy_(p['ln1_g%d' % l])
      layer.norm1.bias.copy_(p['ln1_b%d' % l])
      layer.linear1.weight.copy_(p['w1%d' % l].t())
      layer.linear1.bias.copy_(p['b1%d' % l])
      layer.linear2.weight.copy_(p['w2%d' % l].t())
      layer.linear2.bias.copy_(p['b2%d' % l])
      layer.norm2.weight.copy_(p['ln2_g%d' % l])
      layer.norm2.bias.copy_(p['ln2_b%d' % l])
    layer.eval()
    with torch.no_grad():
      x = layer(x, src_key_padding_mask=(mask == 0))
  pooled = torch.tanh(x[:, 0] @ p['wp'] + p['bp'])
  return pooled @ p['ws'] + p['bs'][0]


@pytest.mark.parametrize('E,H,I,NL,L', [(16, 2, 20, 1, 5), (24, 3, 36, 2, 9)])
def test_reference_matches_transformer_encoder_layer(E, H, I, NL, L):
  V, P, Tv, S = 11, 12, 3, 4
  g = torch.Generator().manual_seed(1)
  wid = torch.randint(0, V, (S, L), generator=g)
  tid = torch.randint(0, Tv, (S, L), generator=g)
  mask = (torch.rand(S, L, generator=g) < 0.7).to(torch.uint8)
  mask[:, 0] = 1
  flat = _flat(V, E, I, NL, P, Tv)
  got = R.forward(wid, mask, tid, flat, V, E, H, I, NL, P, Tv)
  want = _composed(wid, mask, tid, flat, V, E, H, I, NL, P, Tv)
  assert torch.allclose(got, want, rtol=0, atol=1e-10), (got - want).abs().max()


def test_reference_all_masked_sequence_attends_uniformly():
  """torch's key padding mask has no answer for a sequence with no valid key; the kernels'
  rule (logit - 1e9, summed in fp32) gives every token weight 1/L."""
  V, E, H, I, NL, P, Tv, S, L = 7, 8, 2, 12, 2, 6, 2, 2, 5
  g = torch.Generator().manual_seed(2)
  wid = torch.randint(0, V, (S, L), generator=g)
  tid = torch.randint(0, Tv, (S, L), generator=g)
  flat = _flat(V, E, I, NL, P, Tv)
  probs = []
  masked = R.forward(wid, torch.zeros(S, L, dtype=torch.uint8), tid, flat, V, E, H, I, NL, P, Tv,
                     probs=probs)
  assert torch.isfinite(masked).all()
  assert len(probs) == NL
  for pr in probs:
    assert torch.equal(pr, torch.full_like(pr, 1.0 / L))


def test_adamw_reference_by_hand():
  """Three steps over a decayed and an excluded element with grad_scale 0.5, against values
  written out by hand from the rule in include/tfr_b200.h."""
  lr, b1, b2, eps, wd, gs = 0.1, 0.9, 0.999, 1e-6, 0.01, 0.5
  p = torch.tensor([1.0, -2.0], dtype=torch.float64)
  m = torch.zeros(2, dtype=torch.float64)
  v = torch.zeros(2, dtype=torch.float64)
  mask = torch.tensor([1, 0], dtype=torch.uint8)
  grads = [torch.tensor([0.4, -0.2]), torch.tensor([0.2, 0.6]), torch.tensor([-1.0, 0.0])]
  hp, hm, hv = [1.0, -2.0], [0.0, 0.0], [0.0, 0.0]
  for t, g in enumerate(grads, 1):
    p, m, v = R.adamw(p, g.double(), m, v, t, lr, b1, b2, eps, wd, mask, gs)
    for i in range(2):
      gi = float(g[i]) * gs
      hm[i] = b1 * hm[i] + (1 - b1) * gi
      hv[i] = b2 * hv[i] + (1 - b2) * gi * gi
      if i == 0:
        hp[i] -= lr * wd * hp[i]
      hp[i] -= lr * math.sqrt(1 - b2 ** t) / (1 - b1 ** t) * hm[i] / (math.sqrt(hv[i]) + eps)
    assert np.allclose(p.numpy(), hp, rtol=0, atol=1e-15), (t, p, hp)
  # step 1 in closed form: m_hat = g, v_hat = g^2 -> p -= lr * g / (|g| + eps / sqrt(1-b2))
  p1, _, _ = R.adamw(torch.tensor([1.0], dtype=torch.float64), torch.tensor([0.2]).double(),
                     torch.zeros(1, dtype=torch.float64), torch.zeros(1, dtype=torch.float64), 1,
                     lr, b1, b2, 0.0, 0.0)
  assert abs(float(p1) - 0.9) < 1e-12


def test_polynomial_warmup_schedule():
  s = train.PolynomialWarmUp(3e-5, decay_steps=10000, warmup_steps=1000)
  assert s(0) == 0.0
  assert math.isclose(s(500), 1.5e-5, rel_tol=1e-12)
  assert math.isclose(s(1000), 3e-5 * (1 - 1000 / 10000), rel_tol=1e-12)
  assert math.isclose(s(5500), 3e-5 * 0.45, rel_tol=1e-12)
  assert s(10000) == 0.0 and s(20000) == 0.0
  nowarm = train.PolynomialWarmUp(1.0, decay_steps=4, end_learning_rate=0.2)
  assert [nowarm(t) for t in range(5)] == pytest.approx([1.0, 0.8, 0.6, 0.4, 0.2])
  with pytest.raises(ValueError):
    train.PolynomialWarmUp(1.0, decay_steps=0)


def _write_elwc(path, lists, seq):
  recs = []
  for items in lists:
    exs = []
    for ids, msk, seg, label in items:
      e = {}
      if ids is not None:
        e['input_ids'] = list(ids) + [0] * (seq - len(ids))
      if msk is not None:
        e['input_mask'] = list(msk) + [0] * (seq - len(msk))
      if seg is not None:
        e['segment_ids'] = list(seg) + [0] * (seq - len(seg))
      e['label'] = [int(label)]
      exs.append(e)
    recs.append(data.encode_elwc(None, exs))
  data.write_tfrecords(path, recs)


def test_tfrbert_batches(tmp_path):
  seq, n = 6, 3
  big = (1 << 24) - 1
  lists = [[([101, 7, 8, 102], [1, 1, 1, 1], [0, 0, 1, 1], 2),
            ([101, big, 102], [1, 1, 1], [0, 1, 1], 0)],
           [([101, 5, 102, 9, 9, 102], [1] * 6, [0, 0, 0, 1, 1, 1], 1),
            (None, None, None, 1),          # every BERT feature missing: the defaults
            ([101, 3], [1, 1], None, 0)]]
  path = str(tmp_path / 'bert.tfrecord')
  _write_elwc(path, lists, seq)
  (feats, y), = list(tfrbert.tfrbert_batches(path, 2, n, seq, vocab_size=1 << 24,
                                             type_vocab_size=2))
  assert set(feats) == {'input_word_ids', 'input_mask', 'input_type_ids'}
  for t in feats.values():
    assert tuple(t.shape) == (2, n, seq)
  assert feats['input_word_ids'].dtype == torch.int32
  assert feats['input_type_ids'].dtype == torch.int32
  assert feats['input_mask'].dtype == torch.uint8
  assert feats['input_word_ids'][0, 1].tolist() == [101, big, 102, 0, 0, 0]
  assert feats['input_word_ids'][0, 0].tolist() == [101, 7, 8, 102, 0, 0]
  assert feats['input_mask'][0, 0].tolist() == [1, 1, 1, 1, 0, 0]
  assert feats['input_type_ids'][1, 0].tolist() == [0, 0, 0, 1, 1, 1]
  # padded item (list 0 has two) and missing features: zeros, all masked
  assert feats['input_word_ids'][0, 2].tolist() == [0] * seq
  assert feats['input_mask'][0, 2].tolist() == [0] * seq
  assert feats['input_word_ids'][1, 1].tolist() == [0] * seq
  assert feats['input_mask'][1, 1].tolist() == [0] * seq
  assert feats['input_type_ids'][1, 2].tolist() == [0] * seq
  assert y.tolist() == [[2.0, 0.0, -1.0], [1.0, 1.0, 0.0]]
  with pytest.raises(ValueError):
    list(tfrbert.tfrbert_batches(path, 2, n, seq, vocab_size=200))
  bad = str(tmp_path / 'bad.tfrecord')
  _write_elwc(bad, [[([101, 1, 102], [1, 1, 1], [0, 2, 0], 1)]], seq)
  with pytest.raises(ValueError):
    list(tfrbert.tfrbert_batches(bad, 1, n, seq, type_vocab_size=2))


def test_bert_symbols_in_library():
  for name in ('tfr_bert_param_count', 'tfr_bert_workspace_bytes', 'tfr_bert_fwd',
               'tfr_bert_bwd', 'tfr_adamw_step'):
    assert hasattr(_C.lib, name), name
    assert name in _C.EXPORTED_SYMBOLS


def test_param_count_and_layout_names():
  cfg = tfrbert.BertEncoderConfig(vocab_size=50, hidden_size=32, num_layers=2,
                                  num_attention_heads=4, intermediate_size=40,
                                  max_position_embeddings=16, type_vocab_size=2)
  c = _C.BertCfg(vocab_size=50, hidden_size=32, num_heads=4, intermediate_size=40, num_layers=2,
                 max_position=16, type_vocab_size=2)
  n = _C.lib.tfr_bert_param_count(ctypes.byref(c))
  assert n == R.param_count(50, 32, 40, 2, 16, 2)
  assert n == sum(int(np.prod(s)) for _, s in tfrbert.weight_shapes(cfg))
  c.num_heads = 3   # 32 / 3 is not a whole head size
  assert _C.lib.tfr_bert_param_count(ctypes.byref(c)) == 0
