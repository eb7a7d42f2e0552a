"""Pretrained checkpoint import for TFR-BERT (ranking_b200/extension/bert_checkpoint.py) and
the argument checks of global-norm clipping, on the CPU.

Fixtures (tests/golden/bert/): tf-models' TF2 BertEncoder test checkpoint `bert_lite`
(copied from TensorFlow Ranking's extension/testdata) and `hf_tiny`, a Hugging Face BertModel
written by tests/golden/make_bert_fixture.py with its fp64 pooler outputs."""
import ctypes
import json
import math
import os
import re
import shutil
import struct

import pytest
import torch

import _tfrbert_refs as R
from ranking_b200 import _C
from ranking_b200 import train as train_lib
from ranking_b200.extension import bert_checkpoint as bc
from ranking_b200.extension import tfrbert
from ranking_b200.keras import losses as klosses

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'bert')
LITE = os.path.join(GOLDEN, 'bert_lite_tf2.ckpt')
LITE_CONFIG = os.path.join(GOLDEN, 'bert_lite_config.json')
HF = os.path.join(GOLDEN, 'hf_tiny')


def _names(config):
  return [n for n, _ in tfrbert.weight_shapes(config)][:-2]


def _sizes(c):
  return dict(V=c.vocab_size, E=c.hidden_size, I=c.intermediate_size, NL=c.num_layers,
              P=c.max_position_embeddings, Tv=c.type_vocab_size)


def _flat64(weights, config, head=None):
  """fp64 flat buffer: the imported weights, then a score head (default w_s = 0, b_s = 0)."""
  e = config.hidden_size
  ws, bs = head if head is not None else (torch.zeros(e), torch.zeros(1))
  return torch.cat([w.reshape(-1).double() for w in weights.values()] +
                   [ws.double(), bs.double()])


# --- TF2 tensor bundle: bert_lite -----------------------------------------------------


def test_bert_lite_bundle_entries():
  t = bc.read_tf_bundle(LITE)
  # 25 entries: 21 encoder variables, the pooler's 2, save_counter and the object graph
  # (the last two skipped)
  assert len(t) == 23
  prefix = 'model/layer_with_weights-'
  suffix = '/.ATTRIBUTES/VARIABLE_VALUE'
  expect = {
      '0/embeddings': (10, 2), '1/embeddings': (4, 2), '2/embeddings': (2, 2),
      '3/gamma': (2,), '3/beta': (2,), '5/kernel': (2, 2), '5/bias': (2,)}
  for n in ('query', 'key', 'value'):
    expect['4/_attention_layer/_%s_dense/kernel' % n] = (2, 1, 2)
    expect['4/_attention_layer/_%s_dense/bias' % n] = (1, 2)
  expect.update({'4/_attention_output_dense/kernel': (1, 2, 2),
                 '4/_attention_output_dense/bias': (2,),
                 '4/_intermediate_dense/kernel': (2, 2), '4/_intermediate_dense/bias': (2,),
                 '4/_output_dense/kernel': (2, 2), '4/_output_dense/bias': (2,)})
  for ln in ('_attention_layer_norm', '_output_layer_norm'):
    expect['4/%s/gamma' % ln] = (2,)
    expect['4/%s/beta' % ln] = (2,)
  assert sorted(t) == sorted(prefix + k + suffix for k in expect)
  for k, shape in expect.items():
    v = t[prefix + k + suffix]
    assert v.dtype == torch.float32 and tuple(v.shape) == shape, k
    if k.endswith('gamma'):
      assert torch.equal(v, torch.ones(shape)), k
    if k.endswith('beta'):
      assert torch.equal(v, torch.zeros(shape)), k
  # the kernels hold the initializer's draws, not zeros
  assert float(t[prefix + '0/embeddings' + suffix].abs().sum()) > 0


def test_bert_lite_checksums_are_masked_crc32c():
  """Every numeric entry's field 6 is the masked crc32c of its bytes (the reader's check)."""
  data = open(LITE + '.data-00000-of-00001', 'rb').read()
  idx = open(LITE + '.index', 'rb').read()
  footer = idx[-48:]
  _, j = bc._varint(footer, 0, 'f')
  _, j = bc._varint(footer, j, 'f')
  off, j = bc._varint(footer, j, 'f')
  size, _ = bc._varint(footer, j, 'f')
  entries = []
  for _, h in bc._block_entries(bc._read_block(idx, off, size, 'i'), 'i'):
    o, k = bc._varint(h, 0, 'h')
    s, _ = bc._varint(h, k, 'h')
    entries += bc._block_entries(bc._read_block(idx, o, s, 'i'), 'i')
  assert len(entries) == 26   # the header entry + 25
  checked = 0
  for key, value in entries[1:]:
    e = bc._bundle_entry(key.decode(), value)
    if e['dtype'] == 7:   # the object graph's checksum is composed differently
      continue
    assert _C.lib.tfr_masked_crc32c(data[e['offset']:e['offset'] + e['size']],
                                    e['size']) == e['crc'], key
    checked += 1
  assert checked == 24


def test_bert_lite_config_and_mapping():
  c = tfrbert.BertEncoderConfig.from_json(LITE_CONFIG)
  assert (c.vocab_size, c.hidden_size, c.num_layers, c.num_attention_heads,
          c.intermediate_size, c.max_position_embeddings, c.type_vocab_size) == \
      (10, 2, 1, 1, 2, 4, 2)
  w = bc.read_bert_weights(LITE, c)
  assert list(w) == _names(c)
  shapes = dict(tfrbert.weight_shapes(c))
  for n, t in w.items():
    assert tuple(t.shape) == tuple(shapes[n]) and t.dtype == torch.float32, n
  t = bc.read_tf_bundle(LITE)
  p = 'model/layer_with_weights-4/_attention_layer/_%s_dense/%s/.ATTRIBUTES/VARIABLE_VALUE'
  qkv = w['transformer/layer_0/attention/qkv/kernel']
  for i, n in enumerate(('query', 'key', 'value')):
    assert torch.equal(qkv[:, 2 * i:2 * i + 2], t[p % (n, 'kernel')].reshape(2, 2))
    assert torch.equal(w['transformer/layer_0/attention/qkv/bias'][2 * i:2 * i + 2],
                       t[p % (n, 'bias')].reshape(2))
  # the same through the .index path and the directory
  w2 = bc.read_bert_weights(LITE + '.index', c)
  assert all(torch.equal(w[k], w2[k]) for k in w)
  # the fp64 reference runs on the imported weights
  ids = torch.tensor([[1, 5, 9, 0], [3, 2, 0, 0]])
  mask = torch.tensor([[1, 1, 1, 0], [1, 1, 0, 0]])
  s = R.forward(ids, mask, torch.zeros_like(ids), _flat64(w, c, (torch.ones(2), torch.zeros(1))),
                H=c.num_attention_heads, **_sizes(c))
  assert s.shape == (2,) and bool(torch.isfinite(s).all())


def _copy_lite(tmp_path):
  for suffix in ('.index', '.data-00000-of-00001'):
    shutil.copy(LITE + suffix, str(tmp_path / ('ck' + suffix)))
  return str(tmp_path / 'ck')


def test_bert_lite_flipped_data_byte(tmp_path):
  prefix = _copy_lite(tmp_path)
  data = bytearray(open(prefix + '.data-00000-of-00001', 'rb').read())
  data[100] ^= 0x10
  open(prefix + '.data-00000-of-00001', 'wb').write(bytes(data))
  with pytest.raises(ValueError, match=r'layer_with_weights-.*crc32c'):
    bc.read_tf_bundle(prefix)


def test_bert_lite_truncated_index(tmp_path):
  prefix = _copy_lite(tmp_path)
  idx = open(prefix + '.index', 'rb').read()
  for cut in (len(idx) - 1, len(idx) - 48, 10):
    open(prefix + '.index', 'wb').write(idx[:cut])
    with pytest.raises(ValueError, match='truncated'):
      bc.read_tf_bundle(prefix)


def test_bert_lite_corrupt_index_block(tmp_path):
  prefix = _copy_lite(tmp_path)
  idx = bytearray(open(prefix + '.index', 'rb').read())
  idx[50] ^= 0x01
  open(prefix + '.index', 'wb').write(bytes(idx))
  with pytest.raises(ValueError, match='crc32c'):
    bc.read_tf_bundle(prefix)


def test_bert_lite_wrong_config_and_missing_layer():
  c = tfrbert.BertEncoderConfig.from_json(LITE_CONFIG)
  bad = tfrbert.BertEncoderConfig(**dict(vars(c), vocab_size=11))
  with pytest.raises(ValueError, match=r'layer_with_weights-0/embeddings.*disagrees'):
    bc.read_bert_weights(LITE, bad)
  bad = tfrbert.BertEncoderConfig(**dict(vars(c), intermediate_size=4))
  with pytest.raises(ValueError, match=r'_intermediate_dense/kernel'):
    bc.read_bert_weights(LITE, bad)
  # two transformer layers in the config: the second is missing (layer 5 is the pooler)
  two = tfrbert.BertEncoderConfig(**dict(vars(c), num_layers=2))
  with pytest.raises(ValueError, match=r'layer_with_weights-(5|6)'):
    bc.read_bert_weights(LITE, two)
  # the pooler named as a transformer layer -> unrecognised layout
  t = bc.read_tf_bundle(LITE)
  t = {k: v for k, v in t.items() if 'layer_with_weights-5' not in k}
  with pytest.raises(ValueError, match=r'layer_with_weights-5: layer missing'):
    bc._from_tf_encoder(t, c)
  with pytest.raises(ValueError, match='TF1'):
    bc._from_tf_encoder({'bert/embeddings/word_embeddings': torch.zeros(1)}, c)
  with pytest.raises(ValueError, match='unrecognised'):
    bc._from_tf_encoder({'model/_embedding_layer/embeddings': torch.zeros(1)}, c)


def test_bert_lite_prefix_detected():
  c = tfrbert.BertEncoderConfig.from_json(LITE_CONFIG)
  t = bc.read_tf_bundle(LITE)
  enc = {k.replace('model/', 'encoder/', 1): v for k, v in t.items()}
  a, b = bc._from_tf_encoder(t, c), bc._from_tf_encoder(enc, c)
  assert all(torch.equal(a[k], b[k]) for k in a)


def test_snappy_round_trips():
  # literal + overlapping copy: "abcd" then copy-1 (len 8, offset 4) -> "abcd" * 3
  buf = bytes([12, 3 << 2]) + b'abcd' + bytes([((8 - 4) << 2) | 1, 4])
  assert bc.snappy_decompress(buf) == b'abcd' * 3
  with pytest.raises(ValueError):
    bc.snappy_decompress(bytes([12, 3 << 2]) + b'abcd' + bytes([((8 - 4) << 2) | 1, 9]))
  with pytest.raises(ValueError):
    bc.snappy_decompress(bytes([13, 3 << 2]) + b'abcd' + bytes([((8 - 4) << 2) | 1, 4]))


def test_unsupported_entries_raise():
  def entry(dtype, shape, extra=b''):
    dims = b''.join(b'\x12' + bytes([2, 8, d]) for d in shape)
    return bytes([8, dtype, 0x12, len(dims)]) + dims + b'\x28\x08' + extra
  e = bc._bundle_entry('x', entry(1, (2,)))
  assert e['dtype'] == 1 and e['shape'] == (2,) and e['size'] == 8
  with pytest.raises(ValueError, match='sliced'):
    bc._bundle_entry('x', entry(1, (2,), b'\x3a\x00'))


# --- Hugging Face ---------------------------------------------------------------------


def _hf_outputs():
  with open(os.path.join(HF, 'outputs.json')) as f:
    return json.load(f)


def test_config_from_json():
  c = tfrbert.BertEncoderConfig.from_json(os.path.join(HF, 'config.json'))
  assert (c.vocab_size, c.hidden_size, c.num_layers, c.num_attention_heads,
          c.intermediate_size, c.max_position_embeddings, c.type_vocab_size) == \
      (64, 32, 2, 2, 64, 16, 2)
  assert c.hidden_dropout_prob == pytest.approx(0.1)
  assert c.attention_dropout_prob == pytest.approx(0.1)


@pytest.mark.parametrize('act,ok', [('gelu', True), ('gelu_new', True),
                                    ('gelu_pytorch_tanh', True), ('relu', False),
                                    ('gelu_fast', False), ('silu', False)])
def test_config_hidden_act(tmp_path, act, ok):
  p = str(tmp_path / 'config.json')
  d = json.load(open(os.path.join(HF, 'config.json')))
  d['hidden_act'] = act
  json.dump(d, open(p, 'w'))
  if ok:
    assert tfrbert.BertEncoderConfig.from_json(p).hidden_size == 32
  else:
    with pytest.raises(ValueError, match='hidden_act'):
      tfrbert.BertEncoderConfig.from_json(p)


@pytest.mark.parametrize('key,value,ok', [('layer_norm_eps', 1e-12, True),
                                          ('layer_norm_eps', 1e-5, False),
                                          ('position_embedding_type', 'absolute', True),
                                          ('position_embedding_type', 'relative_key', False),
                                          ('position_embedding_type', 'relative_key_query',
                                           False)])
def test_config_layer_norm_eps_and_positions(tmp_path, key, value, ok):
  p = str(tmp_path / 'config.json')
  d = json.load(open(os.path.join(HF, 'config.json')))
  d[key] = value
  json.dump(d, open(p, 'w'))
  if ok:
    assert tfrbert.BertEncoderConfig.from_json(p).hidden_size == 32
  else:
    with pytest.raises(ValueError, match=key):
      tfrbert.BertEncoderConfig.from_json(p)
  # Google's bert_config.json has neither key: the encoder's values are assumed
  del d[key]
  json.dump(d, open(p, 'w'))
  assert tfrbert.BertEncoderConfig.from_json(p).hidden_size == 32


def test_config_heads_must_divide(tmp_path):
  p = str(tmp_path / 'config.json')
  d = json.load(open(os.path.join(HF, 'config.json')))
  d['num_attention_heads'] = 3
  json.dump(d, open(p, 'w'))
  with pytest.raises(ValueError, match='num_attention_heads'):
    tfrbert.BertEncoderConfig.from_json(p)


def test_hf_fixture_matches_transformers_fp64():
  c = tfrbert.BertEncoderConfig.from_json(os.path.join(HF, 'config.json'))
  w = bc.read_bert_weights(HF, c)
  assert list(w) == _names(c)
  out = _hf_outputs()
  ids = torch.tensor(out['input_ids'])
  mask = torch.tensor(out['attention_mask'])
  tid = torch.tensor(out['token_type_ids'])
  want = torch.tensor(out['pooler_output'], dtype=torch.float64)
  e = c.hidden_size
  got = torch.stack([
      R.forward(ids, mask, tid, _flat64(w, c, (torch.eye(e)[j], torch.zeros(1))),
                H=c.num_attention_heads, **_sizes(c))
      for j in range(e)], 1)
  err = float((got - want).abs().max() / want.abs().max())
  assert err < 1e-10, err


def _write_safetensors(path, tensors):
  """A minimal safetensors writer (header length, JSON header, raw little-endian data).  A
  value may also be (dtype name, shape, raw bytes), for dtypes torch cannot hold."""
  names = {torch.float32: 'F32', torch.float16: 'F16', torch.bfloat16: 'BF16',
           torch.float64: 'F64', torch.int64: 'I64', torch.int32: 'I32', torch.uint8: 'U8'}
  header, blobs, off = {}, [], 0
  for k, t in tensors.items():
    if isinstance(t, tuple):
      dtype, shape, raw = t
    else:
      dtype, shape = names[t.dtype], list(t.shape)
      raw = t.contiguous().view(torch.uint8).numpy().tobytes() if t.numel() else b''
    header[k] = {'dtype': dtype, 'shape': list(shape), 'data_offsets': [off, off + len(raw)]}
    blobs.append(raw)
    off += len(raw)
  h = json.dumps(header).encode()
  with open(path, 'wb') as f:
    f.write(struct.pack('<Q', len(h)) + h + b''.join(blobs))


def test_hf_variants_import_to_the_same_weights(tmp_path):
  c = tfrbert.BertEncoderConfig.from_json(os.path.join(HF, 'config.json'))
  base = bc.read_bert_weights(HF, c)
  state = bc.read_safetensors(os.path.join(HF, 'model.safetensors'))
  # BertFor* names: `bert.` prefix, legacy gamma / beta, heads and buffers that are ignored
  renamed = {}
  for k, t in state.items():
    k = re.sub(r'LayerNorm\.weight$', 'LayerNorm.gamma', k)
    k = re.sub(r'LayerNorm\.bias$', 'LayerNorm.beta', k)
    renamed['bert.' + k] = t
  renamed['cls.predictions.bias'] = torch.zeros(64)
  renamed['classifier.weight'] = torch.zeros(2, 32)
  # the persistent buffer older transformers saved, I64 in safetensors files
  renamed['bert.embeddings.position_ids'] = torch.arange(16, dtype=torch.int64)[None]
  p = str(tmp_path / 'renamed.safetensors')
  _write_safetensors(p, dict(renamed, **{'cls.fp8_scale': ('F8_E4M3', (4,), bytes(4))}))
  st = bc.read_safetensors(p)
  assert isinstance(st['bert.embeddings.position_ids'], bc.UndecodedTensor)
  assert st['bert.embeddings.position_ids'].dtype == 'I64'
  got = bc.read_bert_weights(p, c)
  assert list(got) == list(base) and all(torch.equal(got[k], base[k]) for k in base)
  # the same without the prefix, as a bare BertModel would be saved
  plain = dict(state, **{'embeddings.position_ids': torch.arange(16, dtype=torch.int64)[None]})
  _write_safetensors(p, plain)
  got = bc.read_bert_weights(p, c)
  assert all(torch.equal(got[k], base[k]) for k in base)
  # pytorch_model.bin in a directory
  d = tmp_path / 'bin'
  d.mkdir()
  torch.save(renamed, str(d / 'pytorch_model.bin'))
  got = bc.read_bert_weights(str(d), c)
  assert all(torch.equal(got[k], base[k]) for k in base)
  # bf16 and fp16 storage: the same weights, rounded
  for dt in (torch.bfloat16, torch.float16):
    p = str(tmp_path / ('low_%s.safetensors' % str(dt)[6:]))
    _write_safetensors(p, {k: t.to(dt) for k, t in state.items()})
    got = bc.read_bert_weights(p, c)
    for k in base:
      assert torch.equal(got[k], base[k].to(dt).float()), k


def test_hf_missing_and_mismatched_tensors(tmp_path):
  c = tfrbert.BertEncoderConfig.from_json(os.path.join(HF, 'config.json'))
  state = bc.read_safetensors(os.path.join(HF, 'model.safetensors'))
  drop = dict(state)
  del drop['encoder.layer.1.output.dense.weight']
  p = str(tmp_path / 'drop.safetensors')
  _write_safetensors(p, drop)
  with pytest.raises(ValueError, match=r'encoder\.layer\.1\.output\.dense\.weight'):
    bc.read_bert_weights(p, c)
  bad = tfrbert.BertEncoderConfig(**dict(vars(c), intermediate_size=128))
  with pytest.raises(ValueError, match=r'intermediate\.dense\.weight'):
    bc.read_bert_weights(HF, bad)
  one = tfrbert.BertEncoderConfig(**dict(vars(c), num_layers=1))
  with pytest.raises(ValueError, match='more than'):
    bc.read_bert_weights(HF, one)
  wrong = dict(state)
  wrong['pooler.dense.bias'] = torch.zeros(3)
  _write_safetensors(p, wrong)
  with pytest.raises(ValueError, match=r'pooler\.dense\.bias'):
    bc.read_bert_weights(p, c)
  # a tensor the encoder needs, stored in a dtype the reader does not convert
  for dt in (torch.int64, torch.uint8):
    wrong = dict(state)
    wrong['pooler.dense.bias'] = torch.zeros(32, dtype=dt)
    _write_safetensors(p, wrong)
    with pytest.raises(ValueError, match=r'pooler\.dense\.bias has dtype (I64|U8)'):
      bc.read_bert_weights(p, c)
  wrong['pooler.dense.bias'] = torch.zeros(32, dtype=torch.int64)
  torch.save(wrong, str(tmp_path / 'wrong.bin'))
  with pytest.raises(ValueError, match=r'pooler\.dense\.bias has dtype torch\.int64'):
    bc.read_bert_weights(str(tmp_path / 'wrong.bin'), c)
  raw = open(os.path.join(HF, 'model.safetensors'), 'rb').read()
  open(p, 'wb').write(raw[:len(raw) // 2])
  with pytest.raises(ValueError):
    bc.read_bert_weights(p, c)
  with pytest.raises(ValueError, match='not a checkpoint'):
    bc.read_bert_weights(str(tmp_path / 'nothing'), c)


def _hf_as_tf_encoder(state, c, prefix='encoder/'):
  """hf_tiny's weights under tf-models' functional BertEncoder keys and shapes, written from
  the two layouts' definitions: Keras kernels are the transposed torch Linear weights, the
  attention's query / key / value kernels are [E, H, dh] and its output kernel [H, dh, E]
  (EinsumDense), each head's slice of a row or column contiguous, as in HF's view(H, dh)."""
  e, nh = c.hidden_size, c.num_attention_heads
  dh = e // nh
  out = {}

  def put(k, name, t):
    out['%slayer_with_weights-%d/%s/.ATTRIBUTES/VARIABLE_VALUE' % (prefix, k, name)] = t

  put(0, 'embeddings', state['embeddings.word_embeddings.weight'])
  put(1, 'embeddings', state['embeddings.position_embeddings.weight'])
  put(2, 'embeddings', state['embeddings.token_type_embeddings.weight'])
  put(3, 'gamma', state['embeddings.LayerNorm.weight'])
  put(3, 'beta', state['embeddings.LayerNorm.bias'])
  for l in range(c.num_layers):
    h, k = 'encoder.layer.%d.' % l, 4 + l
    for n in ('query', 'key', 'value'):
      w = state[h + 'attention.self.%s.weight' % n]          # [out = (H, dh), in = E]
      put(k, '_attention_layer/_%s_dense/kernel' % n,
          torch.stack([w[i * dh:(i + 1) * dh].t() for i in range(nh)], 1))   # [E, H, dh]
      b = state[h + 'attention.self.%s.bias' % n]
      put(k, '_attention_layer/_%s_dense/bias' % n,
          torch.stack([b[i * dh:(i + 1) * dh] for i in range(nh)]))          # [H, dh]
    wo = state[h + 'attention.output.dense.weight']           # [out = E, in = (H, dh)]
    put(k, '_attention_output_dense/kernel',
        torch.stack([wo[:, i * dh:(i + 1) * dh].t() for i in range(nh)]))    # [H, dh, E]
    put(k, '_attention_output_dense/bias', state[h + 'attention.output.dense.bias'])
    put(k, '_attention_layer_norm/gamma', state[h + 'attention.output.LayerNorm.weight'])
    put(k, '_attention_layer_norm/beta', state[h + 'attention.output.LayerNorm.bias'])
    put(k, '_intermediate_dense/kernel', state[h + 'intermediate.dense.weight'].t())
    put(k, '_intermediate_dense/bias', state[h + 'intermediate.dense.bias'])
    put(k, '_output_dense/kernel', state[h + 'output.dense.weight'].t())
    put(k, '_output_dense/bias', state[h + 'output.dense.bias'])
    put(k, '_output_layer_norm/gamma', state[h + 'output.LayerNorm.weight'])
    put(k, '_output_layer_norm/beta', state[h + 'output.LayerNorm.bias'])
  put(4 + c.num_layers, 'kernel', state['pooler.dense.weight'].t())
  put(4 + c.num_layers, 'bias', state['pooler.dense.bias'])
  return out


def test_tf_layout_of_a_multi_head_model_matches_transformers():
  """The TF2 mapping on a 2-head model: hf_tiny rewritten in tf-models' layout imports to
  the weights that reproduce transformers' outputs, so the head order of the [E, H, dh] and
  [H, dh, E] reshapes is pinned (bert_lite has one head)."""
  c = tfrbert.BertEncoderConfig.from_json(os.path.join(HF, 'config.json'))
  assert c.num_attention_heads == 2
  state = bc.read_safetensors(os.path.join(HF, 'model.safetensors'))
  got = bc._from_tf_encoder(_hf_as_tf_encoder(state, c), c)
  assert list(got) == _names(c)
  out = _hf_outputs()
  ids = torch.tensor(out['input_ids'])
  mask = torch.tensor(out['attention_mask'])
  tid = torch.tensor(out['token_type_ids'])
  want = torch.tensor(out['pooler_output'], dtype=torch.float64)
  e = c.hidden_size
  pooled = torch.stack([
      R.forward(ids, mask, tid, _flat64(got, c, (torch.eye(e)[j], torch.zeros(1))),
                H=c.num_attention_heads, **_sizes(c))
      for j in range(e)], 1)
  err = float((pooled - want).abs().max() / want.abs().max())
  assert err < 1e-10, err
  # the heads swapped inside the query kernel: a different model
  swapped = _hf_as_tf_encoder(state, c)
  key = ('encoder/layer_with_weights-4/_attention_layer/_query_dense/kernel/'
         '.ATTRIBUTES/VARIABLE_VALUE')
  swapped[key] = swapped[key].flip(1)
  bad = bc._from_tf_encoder(swapped, c)
  pooled = torch.stack([
      R.forward(ids, mask, tid, _flat64(bad, c, (torch.eye(e)[j], torch.zeros(1))),
                H=c.num_attention_heads, **_sizes(c))
      for j in range(e)], 1)
  assert float((pooled - want).abs().max() / want.abs().max()) > 1e-3


# --- clipping: argument errors -------------------------------------------------------


class _Tower(object):
  def __init__(self, n=8):
    self.flat = torch.nn.Parameter(torch.zeros(n))


def test_trainer_clip_argument_errors():
  loss = klosses.SoftmaxLoss()
  for opt in ('sgd', 'adagrad'):
    with pytest.raises(ValueError, match="gradient_clip_norm needs optimizer 'adamw'"):
      train_lib.RankingTrainer(_Tower(), loss, optimizer=opt, gradient_clip_norm=1.0)
  for bad in (0.0, -1.0, float('inf'), float('nan')):
    with pytest.raises(ValueError, match='finite and > 0'):
      train_lib.RankingTrainer(_Tower(), loss, optimizer='adamw', gradient_clip_norm=bad)


def test_trainer_clip_rejects_several_ranks(monkeypatch):
  monkeypatch.setattr(train_lib.dp, 'world_size', lambda group=None: 2)
  with pytest.raises(ValueError, match='one rank'):
    train_lib.RankingTrainer(_Tower(), klosses.SoftmaxLoss(), optimizer='adamw',
                             collective='nccl', gradient_clip_norm=1.0)


def test_clip_c_abi_argument_errors():
  """Rejected before any CUDA call: host pointers that a kernel would fault on are never
  touched."""
  buf = (ctypes.c_float * 4)()
  p = ctypes.cast(buf, ctypes.c_void_p)
  L = _C.lib
  assert L.tfr_global_norm_workspace_bytes(0) == 8
  assert L.tfr_global_norm_workspace_bytes(1) == 8
  assert L.tfr_global_norm_workspace_bytes(4096) == 8
  assert L.tfr_global_norm_workspace_bytes(4097) == 16
  assert L.tfr_global_norm_workspace_bytes(110_000_000) == 2048 * 8
  assert L.tfr_global_norm(p, 4, None, p, 8, None) == 1 and 'NULL' in _C.last_error()
  assert L.tfr_global_norm(None, 4, p, p, 8, None) == 1
  assert L.tfr_global_norm(p, 4, p, None, 8, None) == 1
  assert L.tfr_global_norm(p, 5000, p, p, 8, None) == 1 and 'workspace' in _C.last_error()
  args = [p, p, p, p, None, 4, 0.1, 0.9, 0.999, 1e-6, 0.01, 1, 1.0]
  assert L.tfr_adamw_step_clipped(*args, 1.0, None, None) == 1
  assert 'NULL' in _C.last_error()
  for clip in (0.0, -1.0, math.inf, math.nan):
    assert L.tfr_adamw_step_clipped(*args, clip, p, None) == 1
    assert 'clip_norm' in _C.last_error()
  bad_step = list(args)
  bad_step[11] = 0
  assert L.tfr_adamw_step_clipped(*bad_step, 1.0, p, None) == 1
  bad_beta = list(args)
  bad_beta[7] = 1.0
  assert L.tfr_adamw_step_clipped(*bad_beta, 1.0, p, None) == 1


def test_clip_symbols_declared_and_bound():
  hdr = open(os.path.join(os.path.dirname(GOLDEN), '..', '..', 'include',
                          'tfr_b200.h')).read()
  for name in ('tfr_global_norm', 'tfr_global_norm_workspace_bytes', 'tfr_adamw_step_clipped'):
    assert re.search(r'\b%s\s*\(' % name, hdr), name
    assert name in _C.EXPORTED_SYMBOLS
    assert hasattr(_C.lib, name)
