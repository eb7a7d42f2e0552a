"""Pretrained BERT weights for TFR-BERT's encoder (K15), read on the host without TensorFlow
or transformers, as `TFRBertTask.initialize` restores `init_checkpoint` into the encoder
(extension/premade/tfrbert_task.py:346-361).

    read_bert_weights(path, config)   {name: fp32 CPU tensor} in `weight_names()` order, the
                                      score head (`score/kernel`, `score/bias`) excluded

Formats:
  * a TensorFlow 2 tensor bundle (`<prefix>.index` + `<prefix>.data-NNNNN-of-NNNNN`) written
    from tf-models-official's functional BertEncoder (`TFRBertTask` saves it under `encoder/`,
    a bare Keras model under `model/`; the object prefix is detected).  The index is a
    LevelDB-format table whose blocks may be snappy-compressed; every numeric tensor's masked
    crc32c is checked.  Only DT_FLOAT variables are returned; `save_counter` (checksum checked)
    and the object graph are skipped.
  * a Hugging Face BERT: `model.safetensors` (weights in F32, F16 or BF16; entries of other
    dtypes stay undecoded and fail only an import that needs them, so an I64 `position_ids`
    buffer is ignored) or `pytorch_model.bin`
    (read with `torch.load(weights_only=True)`), names with or without the `bert.` prefix,
    LayerNorm `weight / bias` or the legacy `gamma / beta`.  Heads (`cls.*`, `classifier.*`)
    and buffers such as `position_ids` are ignored.

Every inconsistency (corrupt bytes, a shape that disagrees with the config, a missing tensor
or layer, a layout this module does not know, such as TF1 Google BERT's `bert/...` names or
tf-models' BertEncoderV2) raises ValueError naming what failed.
"""
import collections
import json
import os
import re
import struct

import torch

from ranking_b200 import _C

# --- TensorFlow tensor bundle ------------------------------------------------------------

_TABLE_MAGIC = 0xdb4775248b80fb57
_FOOTER_LEN = 48
_DT_FLOAT = 1
_OBJECT_GRAPH = '_CHECKPOINTABLE_OBJECT_GRAPH'   # DT_STRING, its checksum composed differently
_SAVE_COUNTER = 'save_counter/.ATTRIBUTES/VARIABLE_VALUE'   # DT_INT64: checked, then skipped
_DTYPE_NAMES = {1: 'DT_FLOAT', 2: 'DT_DOUBLE', 3: 'DT_INT32', 7: 'DT_STRING', 9: 'DT_INT64',
                14: 'DT_BFLOAT16', 19: 'DT_HALF'}


def _masked_crc32c(data):
  return _C.lib.tfr_masked_crc32c(bytes(data), len(data))


def _varint(buf, i, what):
  r = s = 0
  while True:
    if i >= len(buf) or s > 63:
      raise ValueError('%s: truncated varint' % what)
    c = buf[i]
    i += 1
    r |= (c & 0x7f) << s
    s += 7
    if c < 0x80:
      return r, i


def snappy_decompress(buf, what='snappy block'):
  """Raw snappy (the block format TensorFlow's table writer uses), in Python."""
  n, i = _varint(buf, 0, what)
  out = bytearray()
  while i < len(buf):
    tag = buf[i]
    i += 1
    kind = tag & 3
    if kind == 0:   # literal
      ln = tag >> 2
      if ln >= 60:
        nb = ln - 59
        if i + nb > len(buf):
          raise ValueError('%s: truncated literal length' % what)
        ln = int.from_bytes(buf[i:i + nb], 'little')
        i += nb
      ln += 1
      if i + ln > len(buf):
        raise ValueError('%s: literal runs past the input' % what)
      out += buf[i:i + ln]
      i += ln
      continue
    if kind == 1:
      ln, nb = ((tag >> 2) & 7) + 4, 1
      if i >= len(buf):
        raise ValueError('%s: truncated copy' % what)
      off = ((tag >> 5) << 8) | buf[i]
    else:
      ln, nb = (tag >> 2) + 1, (2 if kind == 2 else 4)
      if i + nb > len(buf):
        raise ValueError('%s: truncated copy' % what)
      off = int.from_bytes(buf[i:i + nb], 'little')
    i += 1 if kind == 1 else nb
    if off == 0 or off > len(out):
      raise ValueError('%s: copy offset %d outside the %d bytes written' % (what, off, len(out)))
    for _ in range(ln):   # overlapping copies repeat the pattern
      out.append(out[-off])
  if len(out) != n:
    raise ValueError('%s: %d bytes decoded, header says %d' % (what, len(out), n))
  return bytes(out)


def _read_block(data, offset, size, what):
  """Block contents at a handle, trailer (type byte + masked crc32c) checked."""
  if offset + size + 5 > len(data):
    raise ValueError('%s: block [%d, +%d) runs past the %d-byte index (truncated?)' %
                     (what, offset, size, len(data)))
  raw = data[offset:offset + size + 1]
  kind = raw[-1]
  crc = struct.unpack('<I', data[offset + size + 1:offset + size + 5])[0]
  if _masked_crc32c(raw) != crc:
    raise ValueError('%s: block at offset %d fails its crc32c' % (what, offset))
  if kind == 0:
    return raw[:-1]
  if kind == 1:
    return snappy_decompress(raw[:-1], what)
  raise ValueError('%s: block compression type %d unsupported (0 none, 1 snappy)' %
                   (what, kind))


def _block_entries(block, what):
  """(key, value) pairs of a table block: prefix-compressed keys, restart array at the end."""
  if len(block) < 4:
    raise ValueError('%s: block too short' % what)
  nres = struct.unpack('<I', block[-4:])[0]
  end = len(block) - 4 - 4 * nres
  if nres < 1 or end < 0:
    raise ValueError('%s: bad restart array (%d restarts)' % (what, nres))
  restarts = set(struct.unpack('<%dI' % nres, block[end:end + 4 * nres]))
  out, i, key = [], 0, b''
  while i < end:
    start = i
    shared, i = _varint(block, i, what)
    nonshared, i = _varint(block, i, what)
    vlen, i = _varint(block, i, what)
    if shared > len(key) or (start in restarts and shared) or i + nonshared + vlen > end:
      raise ValueError('%s: corrupt entry at byte %d' % (what, start))
    key = key[:shared] + block[i:i + nonshared]
    i += nonshared
    out.append((key, block[i:i + vlen]))
    i += vlen
  return out


def _proto_fields(buf, what):
  """{field number: [values]} of a protobuf message (varint, fixed32/64, length-delimited)."""
  f, i = collections.defaultdict(list), 0
  while i < len(buf):
    tag, i = _varint(buf, i, what)
    num, wt = tag >> 3, tag & 7
    if wt == 0:
      x, i = _varint(buf, i, what)
    elif wt == 1:
      x, i = buf[i:i + 8], i + 8
    elif wt == 2:
      ln, i = _varint(buf, i, what)
      x, i = buf[i:i + ln], i + ln
    elif wt == 5:
      x, i = struct.unpack('<I', buf[i:i + 4])[0] if i + 4 <= len(buf) else None, i + 4
    else:
      raise ValueError('%s: wire type %d unsupported' % (what, wt))
    if i > len(buf):
      raise ValueError('%s: truncated protobuf' % what)
    f[num].append(x)
  return f


def _bundle_entry(key, value):
  """BundleEntryProto -> dict(dtype, shape, shard, offset, size, crc)."""
  what = 'checkpoint entry %r' % key
  f = _proto_fields(value, what)
  if f.get(7):
    raise ValueError('%s is sliced / partitioned; only whole tensors are supported' % key)
  shape = []
  for s in f.get(2, []):
    sf = _proto_fields(s, what)
    if sf.get(3) and sf[3][-1]:
      raise ValueError('%s has an unknown rank' % key)
    shape += [_proto_fields(d, what).get(1, [0])[-1] for d in sf.get(2, [])]
  crc = f.get(6, [None])[-1]
  return dict(dtype=f.get(1, [0])[-1], shape=tuple(shape), shard=f.get(3, [0])[-1],
              offset=f.get(4, [0])[-1], size=f.get(5, [0])[-1], crc=crc)


def read_tf_bundle(prefix):
  """{variable key: fp32 CPU tensor} of a TF2 tensor bundle (`<prefix>.index` and its data
  shards); DT_FLOAT only, every tensor's masked crc32c checked."""
  index_path = prefix + '.index'
  with open(index_path, 'rb') as fh:
    data = fh.read()
  what = index_path
  if len(data) < _FOOTER_LEN or struct.unpack('<Q', data[-8:])[0] != _TABLE_MAGIC:
    raise ValueError('%s: not a TensorFlow checkpoint index (footer magic missing; '
                     'truncated?)' % what)
  footer = data[-_FOOTER_LEN:]
  _, j = _varint(footer, 0, what)   # metaindex handle: unused by tensor bundles
  _, j = _varint(footer, j, what)
  idx_off, j = _varint(footer, j, what)
  idx_size, j = _varint(footer, j, what)
  entries = []
  for _, handle in _block_entries(_read_block(data, idx_off, idx_size, what), what):
    off, k = _varint(handle, 0, what)
    size, _ = _varint(handle, k, what)
    entries += _block_entries(_read_block(data, off, size, what), what)
  if not entries or entries[0][0] != b'':
    raise ValueError('%s: the bundle header entry is missing' % what)
  header = _proto_fields(entries[0][1], what)
  num_shards = header.get(1, [1])[-1]
  if header.get(2, [0])[-1] != 0:
    raise ValueError('%s: big-endian bundles are not supported' % what)
  out, files = collections.OrderedDict(), {}
  try:
    for raw_key, value in entries[1:]:
      key = raw_key.decode('utf-8')
      if key == _OBJECT_GRAPH:
        continue
      e = _bundle_entry(key, value)
      if key != _SAVE_COUNTER:
        if e['dtype'] != _DT_FLOAT:
          raise ValueError('%s: dtype %s unsupported (DT_FLOAT only)' %
                           (key, _DTYPE_NAMES.get(e['dtype'], e['dtype'])))
        numel = 1
        for d in e['shape']:
          numel *= d
        if e['size'] != 4 * numel:
          raise ValueError('%s: %d bytes for shape %s' % (key, e['size'], e['shape']))
      if not 0 <= e['shard'] < num_shards:
        raise ValueError('%s: shard %d of %d' % (key, e['shard'], num_shards))
      if e['shard'] not in files:
        files[e['shard']] = open('%s.data-%05d-of-%05d' % (prefix, e['shard'], num_shards),
                                 'rb')
      fh = files[e['shard']]
      fh.seek(e['offset'])
      buf = fh.read(e['size'])
      if len(buf) != e['size']:
        raise ValueError('%s: data shard ends before the tensor (truncated?)' % key)
      if e['crc'] is None or _masked_crc32c(buf) != e['crc']:
        raise ValueError('%s: data fails its crc32c check (corrupt checkpoint)' % key)
      if key == _SAVE_COUNTER:
        continue
      out[key] = torch.frombuffer(bytearray(buf), dtype=torch.float32).reshape(e['shape'])
  finally:
    for fh in files.values():
      fh.close()
  return out


_TF_LAYER = re.compile(r'^(.*?)layer_with_weights-(\d+)/(.*)/\.ATTRIBUTES/VARIABLE_VALUE$')


def _from_tf_encoder(tensors, config):
  """tf-models' functional BertEncoder (layer_with_weights-k) -> K15 names."""
  if any(k.startswith('bert/') for k in tensors):
    raise ValueError('TF1 Google BERT checkpoints (bert/...) are not supported; convert it '
                     'to a TF2 BertEncoder or Hugging Face checkpoint')
  layers, prefixes = collections.defaultdict(dict), set()
  for key, t in tensors.items():
    m = _TF_LAYER.match(key)
    if m:
      prefixes.add(m.group(1))
      layers[int(m.group(2))][m.group(3)] = (key, t)
  if not layers:
    raise ValueError('unrecognised checkpoint layout: no tf-models BertEncoder '
                     '(layer_with_weights-k) variables among %s' % sorted(tensors)[:8])
  if len(prefixes) != 1:
    raise ValueError('checkpoint holds several objects with encoder layers: %s' %
                     sorted(prefixes))
  prefix = prefixes.pop()
  c = config
  e, nh, nl = c.hidden_size, c.num_attention_heads, c.num_layers
  dh = e // nh
  expected = 5 + nl
  extra = sorted(k for k in layers if k >= expected)
  if extra:
    raise ValueError('%slayer_with_weights-%d: the checkpoint has more layers than the '
                     'config (%d transformer layers)' % (prefix, extra[0], nl))

  def get(k, name, shape):
    layer = '%slayer_with_weights-%d' % (prefix, k)
    if k not in layers:
      raise ValueError('%s: layer missing from the checkpoint' % layer)
    if name not in layers[k]:
      raise ValueError('%s/%s: unrecognised layout (the layer has %s)' %
                       (layer, name, sorted(layers[k])))
    key, t = layers[k][name]
    if tuple(t.shape) != tuple(shape):
      raise ValueError('%s: shape %s disagrees with the config (expected %s)' %
                       (key, tuple(t.shape), tuple(shape)))
    return t

  out = collections.OrderedDict()
  out['word_embeddings'] = get(0, 'embeddings', (c.vocab_size, e))
  out['position_embeddings'] = get(1, 'embeddings', (c.max_position_embeddings, e))
  out['type_embeddings'] = get(2, 'embeddings', (c.type_vocab_size, e))
  out['embeddings/layer_norm/gamma'] = get(3, 'gamma', (e,))
  out['embeddings/layer_norm/beta'] = get(3, 'beta', (e,))
  for l in range(nl):
    k, p = 4 + l, 'transformer/layer_%d/' % l
    qkv = ['_attention_layer/_%s_dense/' % n for n in ('query', 'key', 'value')]
    out[p + 'attention/qkv/kernel'] = torch.cat(
        [get(k, a + 'kernel', (e, nh, dh)).reshape(e, e) for a in qkv], 1)
    out[p + 'attention/qkv/bias'] = torch.cat(
        [get(k, a + 'bias', (nh, dh)).reshape(e) for a in qkv])
    out[p + 'attention/output/kernel'] = get(k, '_attention_output_dense/kernel',
                                             (nh, dh, e)).reshape(e, e)
    out[p + 'attention/output/bias'] = get(k, '_attention_output_dense/bias', (e,))
    out[p + 'attention_layer_norm/gamma'] = get(k, '_attention_layer_norm/gamma', (e,))
    out[p + 'attention_layer_norm/beta'] = get(k, '_attention_layer_norm/beta', (e,))
    out[p + 'intermediate/kernel'] = get(k, '_intermediate_dense/kernel',
                                         (e, c.intermediate_size))
    out[p + 'intermediate/bias'] = get(k, '_intermediate_dense/bias', (c.intermediate_size,))
    out[p + 'output/kernel'] = get(k, '_output_dense/kernel', (c.intermediate_size, e))
    out[p + 'output/bias'] = get(k, '_output_dense/bias', (e,))
    out[p + 'output_layer_norm/gamma'] = get(k, '_output_layer_norm/gamma', (e,))
    out[p + 'output_layer_norm/beta'] = get(k, '_output_layer_norm/beta', (e,))
  out['pooler/kernel'] = get(4 + nl, 'kernel', (e, e))
  out['pooler/bias'] = get(4 + nl, 'bias', (e,))
  return out


# --- Hugging Face ------------------------------------------------------------------------

_SAFETENSORS_DTYPES = {'F32': torch.float32, 'F16': torch.float16, 'BF16': torch.bfloat16}


class UndecodedTensor(object):
  """A safetensors entry of a dtype other than F32 / F16 / BF16 (such as the I64
  `embeddings.position_ids` buffer older transformers saved): kept undecoded, so that it
  only fails an import that needs it."""

  def __init__(self, dtype, shape):
    self.dtype, self.shape = dtype, shape

  def __repr__(self):
    return 'UndecodedTensor(%s, %s)' % (self.dtype, self.shape)


def read_safetensors(path):
  """{name: tensor} of a .safetensors file (8-byte header length, JSON header, raw
  little-endian data): F32, F16 and BF16 tensors converted to fp32, entries of any other
  dtype as `UndecodedTensor`."""
  with open(path, 'rb') as fh:
    data = fh.read()
  if len(data) < 8:
    raise ValueError('%s: not a safetensors file (too short)' % path)
  hlen = struct.unpack('<Q', data[:8])[0]
  if 8 + hlen > len(data):
    raise ValueError('%s: header length %d runs past the file (truncated?)' % (path, hlen))
  try:
    header = json.loads(data[8:8 + hlen].decode('utf-8'))
  except (UnicodeDecodeError, json.JSONDecodeError) as err:
    raise ValueError('%s: unreadable safetensors header (%s)' % (path, err))
  body = memoryview(data)[8 + hlen:]
  out = collections.OrderedDict()
  for name, info in header.items():
    if name == '__metadata__':
      continue
    shape = tuple(int(s) for s in info['shape'])
    begin, end = (int(x) for x in info['data_offsets'])
    if not 0 <= begin <= end <= len(body):
      raise ValueError('%s: %s has data [%d, %d) outside the %d-byte body (truncated?)' %
                       (path, name, begin, end, len(body)))
    dtype = _SAFETENSORS_DTYPES.get(info.get('dtype'))
    if dtype is None:
      out[name] = UndecodedTensor(info.get('dtype'), shape)
      continue
    numel = 1
    for s in shape:
      numel *= s
    if end - begin != numel * dtype.itemsize:
      raise ValueError('%s: %s has %d bytes for %s of shape %s' %
                       (path, name, end - begin, info['dtype'], shape))
    t = torch.frombuffer(bytearray(body[begin:end]), dtype=dtype) if numel else \
        torch.empty(0, dtype=dtype)
    out[name] = t.reshape(shape).float()
  return out


def _from_hf(state, config, source):
  """Hugging Face BertModel / BertFor* names -> K15 names ([out, in] Linear weights become
  Keras [in, out] kernels)."""
  names = {}
  for k, t in state.items():
    n = k[5:] if k.startswith('bert.') else k
    n = re.sub(r'LayerNorm\.gamma$', 'LayerNorm.weight', n)
    n = re.sub(r'LayerNorm\.beta$', 'LayerNorm.bias', n)
    names[n] = (k, t)
  c = config
  e, i = c.hidden_size, c.intermediate_size

  def get(name, shape, linear=False):
    if name not in names:
      raise ValueError('%s: tensor %s (or bert.%s) missing' % (source, name, name))
    key, t = names[name]
    if isinstance(t, UndecodedTensor) or not t.is_floating_point():
      raise ValueError('%s: %s has dtype %s (F32, F16 or BF16 only)' %
                       (source, key, t.dtype))
    want = (shape[1], shape[0]) if linear else shape
    if tuple(t.shape) != tuple(want):
      raise ValueError('%s: %s has shape %s, the config needs %s' %
                       (source, key, tuple(t.shape), tuple(want)))
    t = t.detach().to(torch.float32)
    return t.t().contiguous() if linear else t

  out = collections.OrderedDict()
  out['word_embeddings'] = get('embeddings.word_embeddings.weight', (c.vocab_size, e))
  out['position_embeddings'] = get('embeddings.position_embeddings.weight',
                                   (c.max_position_embeddings, e))
  out['type_embeddings'] = get('embeddings.token_type_embeddings.weight',
                               (c.type_vocab_size, e))
  out['embeddings/layer_norm/gamma'] = get('embeddings.LayerNorm.weight', (e,))
  out['embeddings/layer_norm/beta'] = get('embeddings.LayerNorm.bias', (e,))
  for l in range(c.num_layers):
    h, p = 'encoder.layer.%d.' % l, 'transformer/layer_%d/' % l
    qkv = [h + 'attention.self.%s.' % n for n in ('query', 'key', 'value')]
    out[p + 'attention/qkv/kernel'] = torch.cat(
        [get(a + 'weight', (e, e), True) for a in qkv], 1)
    out[p + 'attention/qkv/bias'] = torch.cat([get(a + 'bias', (e,)) for a in qkv])
    out[p + 'attention/output/kernel'] = get(h + 'attention.output.dense.weight', (e, e), True)
    out[p + 'attention/output/bias'] = get(h + 'attention.output.dense.bias', (e,))
    out[p + 'attention_layer_norm/gamma'] = get(h + 'attention.output.LayerNorm.weight', (e,))
    out[p + 'attention_layer_norm/beta'] = get(h + 'attention.output.LayerNorm.bias', (e,))
    out[p + 'intermediate/kernel'] = get(h + 'intermediate.dense.weight', (e, i), True)
    out[p + 'intermediate/bias'] = get(h + 'intermediate.dense.bias', (i,))
    out[p + 'output/kernel'] = get(h + 'output.dense.weight', (i, e), True)
    out[p + 'output/bias'] = get(h + 'output.dense.bias', (e,))
    out[p + 'output_layer_norm/gamma'] = get(h + 'output.LayerNorm.weight', (e,))
    out[p + 'output_layer_norm/beta'] = get(h + 'output.LayerNorm.bias', (e,))
  if 'encoder.layer.%d.attention.self.query.weight' % c.num_layers in names:
    raise ValueError('%s: the checkpoint has more than the config\'s %d layers' %
                     (source, c.num_layers))
  out['pooler/kernel'] = get('pooler.dense.weight', (e, e), True)
  out['pooler/bias'] = get('pooler.dense.bias', (e,))
  return out


# --- entry point -------------------------------------------------------------------------


def _resolve(path):
  """(kind, file or prefix): 'safetensors', 'bin' or 'tf'."""
  if os.path.isdir(path):
    for name, kind in (('model.safetensors', 'safetensors'), ('pytorch_model.bin', 'bin')):
      if os.path.isfile(os.path.join(path, name)):
        return kind, os.path.join(path, name)
    idx = sorted(f for f in os.listdir(path) if f.endswith('.index'))
    if len(idx) == 1:
      return 'tf', os.path.join(path, idx[0])[:-len('.index')]
    raise ValueError('%s: no model.safetensors, pytorch_model.bin or single TF checkpoint '
                     '(.index) in the directory (found %d .index files)' % (path, len(idx)))
  if path.endswith('.safetensors'):
    return 'safetensors', path
  if path.endswith('.bin'):
    return 'bin', path
  prefix = path[:-len('.index')] if path.endswith('.index') else path
  if os.path.isfile(prefix + '.index'):
    return 'tf', prefix
  raise ValueError('%s: not a checkpoint (no such file, and no %s.index)' % (path, prefix))


def read_bert_weights(path, config):
  """{name: fp32 CPU tensor} for every encoder weight of `config` (a BertEncoderConfig) in
  `weight_names()` order, without the score head, from a TF2 BertEncoder checkpoint prefix
  (or its `.index`), a Hugging Face `model.safetensors` / `pytorch_model.bin`, or a directory
  holding one of them.  No encoder is built, so any size works."""
  kind, f = _resolve(path)
  if kind == 'tf':
    return _from_tf_encoder(read_tf_bundle(f), config)
  if kind == 'safetensors':
    state = read_safetensors(f)
  else:
    state = torch.load(f, map_location='cpu', weights_only=True)
    if not isinstance(state, dict):
      raise ValueError('%s: expected a state dict, got %s' % (f, type(state).__name__))
  return _from_hf(state, config, f)
