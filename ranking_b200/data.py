"""Input side of the hot path: LibSVM ranking files -> dense [num_queries, list_size, D]
features + labels (the format of examples/tf_ranking_libsvm.py:137-195), and
pinned-memory batch iteration for `HostBatchPipeline`.
"""
import numpy as np
import torch


def load_libsvm_data(path, list_size, num_features):
  """examples/tf_ranking_libsvm.py:137-195: one line per document,
  `label qid:<id> <feature>:<value> ... [# comment]`; feature ids are 1-based.

  Queries keep the order of first appearance; only the first `list_size` documents
  of a query are kept; missing features are 0; padded slots have label -1.
  Returns (features float32 [Q, list_size, num_features], labels float32 [Q, list_size]).
  """
  qid_to_index = {}
  qid_to_ndoc = []
  feats, labels = [], []
  total_docs = discarded_docs = 0
  with open(path, 'rt') as f:
    for line in f:
      tokens = line.split('#')[0].split()
      if not tokens:
        continue
      assert len(tokens) >= 2, 'Ill-formatted line: {}'.format(line)
      label = float(tokens[0])
      qid = tokens[1]
      idx = qid_to_index.get(qid)
      if idx is None:
        idx = qid_to_index[qid] = len(qid_to_index)
        qid_to_ndoc.append(0)
        feats.append(np.zeros([list_size, num_features], dtype=np.float32))
        labels.append(np.full([list_size], -1., dtype=np.float32))
      total_docs += 1
      doc_idx = qid_to_ndoc[idx]
      qid_to_ndoc[idx] += 1
      if doc_idx >= list_size:      # keep the first `list_size` docs only
        discarded_docs += 1
        continue
      row = feats[idx][doc_idx]
      for kv in tokens[2:]:
        k, v = kv.split(':')
        k = int(k)
        assert 1 <= k <= num_features, 'Key {} not found in features.'.format(k)
        row[k - 1] = float(v)
      labels[idx][doc_idx] = label
  info = {'num_queries': len(qid_to_index), 'num_docs': total_docs,
          'num_discarded': discarded_docs}
  if not feats:
    return (np.zeros([0, list_size, num_features], np.float32),
            np.zeros([0, list_size], np.float32), info)
  return np.stack(feats), np.stack(labels), info


def batch_iterator(features, labels, batch_size, shuffle=False, seed=0,
                   drop_remainder=True, repeat=False, pin_memory=True):
  """Yields (x [B, N, D], y [B, N]) CPU tensors (pinned when CUDA is there) in the
  order tf.data's from_tensor_slices -> shuffle -> batch would (the shuffle here is a
  full permutation per epoch)."""
  x_all = torch.as_tensor(np.ascontiguousarray(features), dtype=torch.float32)
  y_all = torch.as_tensor(np.ascontiguousarray(labels), dtype=torch.float32)
  q = x_all.shape[0]
  pin = pin_memory and torch.cuda.is_available()
  gen = torch.Generator().manual_seed(seed)
  while True:
    order = torch.randperm(q, generator=gen) if shuffle else torch.arange(q)
    for lo in range(0, q, batch_size):
      idx = order[lo:lo + batch_size]
      if idx.numel() < batch_size and drop_remainder:
        break
      x, y = x_all[idx].contiguous(), y_all[idx].contiguous()
      if pin:
        x, y = x.pin_memory(), y.pin_memory()
      yield x, y
    if not repeat:
      return


# ----------------------------------------------------------------------------
# TFRecord files of ExampleListWithContext protos (the reference's training format:
# data.py:80-208, 391-540).  Decoding runs in the native parser behind
# tfr_elwc_parse (csrc/elwc_parser.cu, host code).
# ----------------------------------------------------------------------------
import ctypes
import struct


def _masked_crc(data):
  from ranking_b200 import _C
  return int(_C.lib.tfr_masked_crc32c(data, len(data)))


def read_tfrecords(path, verify_crc=True):
  """Yields the payload bytes of every record of a TFRecord file
  (uint64 length, uint32 masked crc32c(length), data, uint32 masked crc32c(data))."""
  with open(path, 'rb') as f:
    while True:
      head = f.read(12)
      if not head:
        return
      if len(head) < 12:
        raise ValueError('truncated TFRecord header in %s' % path)
      length, len_crc = struct.unpack('<QI', head)
      if verify_crc and _masked_crc(head[:8]) != len_crc:
        raise ValueError('corrupted TFRecord length in %s' % path)
      data = f.read(length)
      tail = f.read(4)
      if len(data) < length or len(tail) < 4:
        raise ValueError('truncated TFRecord in %s' % path)
      if verify_crc and _masked_crc(data) != struct.unpack('<I', tail)[0]:
        raise ValueError('corrupted TFRecord data in %s' % path)
      yield data


def write_tfrecords(path, records):
  with open(path, 'wb') as f:
    for data in records:
      head = struct.pack('<Q', len(data))
      f.write(head)
      f.write(struct.pack('<I', _masked_crc(head)))
      f.write(data)
      f.write(struct.pack('<I', _masked_crc(data)))


# -- a small protobuf writer for tf.Example / ExampleListWithContext (tests, data prep) --
def _varint(v):
  out = bytearray()
  v &= (1 << 64) - 1
  while True:
    b = v & 0x7f
    v >>= 7
    if v:
      out.append(b | 0x80)
    else:
      out.append(b)
      return bytes(out)


def _ld(field, payload):
  return _varint((field << 3) | 2) + _varint(len(payload)) + payload


def encode_example(features):
  """{name: list of float | list of int | list of bytes} -> serialized tf.Example."""
  entries = b''
  for name, values in features.items():
    values = list(values)
    if values and isinstance(values[0], (bytes, str)):
      body = b''.join(_ld(1, v if isinstance(v, bytes) else v.encode()) for v in values)
      feat = _ld(1, body)
    elif values and isinstance(values[0], int) and not isinstance(values[0], bool):
      feat = _ld(3, _ld(1, b''.join(_varint(int(v)) for v in values)))
    else:
      feat = _ld(2, _ld(1, struct.pack('<%df' % len(values), *[float(v) for v in values])))
    entries += _ld(1, _ld(1, name.encode()) + _ld(2, feat))
  return _ld(1, entries)


def encode_elwc(context, examples):
  """ExampleListWithContext{examples = 1 (repeated), context = 2}."""
  out = b''.join(_ld(1, encode_example(e)) for e in examples)
  if context is not None:
    out += _ld(2, encode_example(context))
  return out


def _spec_array(spec):
  from ranking_b200 import _C
  items = list(spec.items()) if spec else []
  arr = (_C.FeatureSpec * max(len(items), 1))()
  keep = []
  for i, (name, (dim, default)) in enumerate(items):
    key = name.encode()
    keep.append(key)
    arr[i].name = key
    arr[i].dim = int(dim)
    arr[i].default_value = float(default)
  return arr, len(items), sum(int(d) for _, (d, _) in items), keep


EXAMPLE_LIST_WITH_CONTEXT = 'example_list_with_context'   # data.py:45-51 data formats
EXAMPLE_IN_EXAMPLE = 'example_in_example'
SEQUENCE_EXAMPLE = 'sequence_example'
_FORMATS = {EXAMPLE_LIST_WITH_CONTEXT: 0, EXAMPLE_IN_EXAMPLE: 1, SEQUENCE_EXAMPLE: 2}


def parse_from_example_in_example(serialized, list_size, context_feature_spec=None,
                                  example_feature_spec=None, **kwargs):
  """data.py:211-380 (dense features): outer Examples with `serialized_context` /
  `serialized_examples` bytes features."""
  return parse_from_example_list(serialized, list_size, context_feature_spec,
                                 example_feature_spec, data_format=EXAMPLE_IN_EXAMPLE,
                                 **kwargs)


def parse_from_sequence_example(serialized, list_size, context_feature_spec=None,
                                example_feature_spec=None, **kwargs):
  """data.py:713-855 (dense features): SequenceExamples, item i = frame i."""
  return parse_from_example_list(serialized, list_size, context_feature_spec,
                                 example_feature_spec, data_format=SEQUENCE_EXAMPLE,
                                 **kwargs)


def make_parsing_fn(data_format, list_size, context_feature_spec=None,
                    example_feature_spec=None, **kwargs):
  """data.py:857-911: serialized records -> feature dict, for any of the three formats."""
  if data_format not in _FORMATS:
    raise ValueError('Data format {} is not supported.'.format(data_format))
  return lambda serialized: parse_from_example_list(
      serialized, list_size, context_feature_spec, example_feature_spec,
      data_format=data_format, **kwargs)


def encode_example_in_example(context, examples):
  """The EIE record for `context` / `examples` feature dicts (see encode_example)."""
  return encode_example({
      'serialized_context': [encode_example(context or {})],
      'serialized_examples': [encode_example(e) for e in examples]})


def _encode_feature(values):
  """One Feature message (oneof bytes / float / int64 list)."""
  values = list(values)
  if values and isinstance(values[0], (bytes, str)):
    return _ld(1, b''.join(_ld(1, v if isinstance(v, bytes) else v.encode()) for v in values))
  if values and isinstance(values[0], int) and not isinstance(values[0], bool):
    return _ld(3, _ld(1, b''.join(_varint(int(v)) for v in values)))
  return _ld(2, _ld(1, struct.pack('<%df' % len(values), *[float(v) for v in values])))


def encode_sequence_example(context, examples, feature_names=None):
  """SequenceExample{context = 1, feature_lists = 2}: one feature list per example
  feature, one frame per item (items that lack a feature get an empty Feature)."""
  names = feature_names or sorted({k for e in examples for k in e})
  lists = b''
  for name in names:
    frames = b''.join(_ld(1, _encode_feature(e[name]) if name in e else b'') for e in examples)
    lists += _ld(1, _ld(1, name.encode()) + _ld(2, frames))
  ctx_features = b''.join(_ld(1, _ld(1, k.encode()) + _ld(2, _encode_feature(v)))
                          for k, v in (context or {}).items())
  return _ld(1, ctx_features) + _ld(2, lists)


class Vocabulary(object):
  """Token -> id map of `tf.feature_column.categorical_column_with_vocabulary_file` /
  `_list`: ids 0 .. V-1 in list (file line) order.  `num_oov_buckets=0`: an unknown token
  gets id -1, which embedding lookups ignore; `num_oov_buckets=1`: it gets id V, so its
  embedding table needs V + 1 rows (`num_ids`).  More buckets (TF hashes them with
  Fingerprint64) and duplicate tokens raise ValueError.  The map lives in the native
  decoder (tfr_vocab_create), which looks tokens up while it parses records."""

  def __init__(self, tokens, num_oov_buckets=0):
    from ranking_b200 import _C
    toks = [t.encode() if isinstance(t, str) else bytes(t) for t in tokens]
    n = len(toks)
    arr = (ctypes.c_char_p * max(n, 1))(*toks)
    lens = (ctypes.c_int64 * max(n, 1))(*[len(t) for t in toks])
    handle = ctypes.c_void_p()
    self._handle = None
    _C.check(_C.lib.tfr_vocab_create(arr, lens, n, int(num_oov_buckets), ctypes.byref(handle)))
    self._handle = handle
    self.tokens = toks
    self.vocabulary_size = n
    self.num_oov_buckets = int(num_oov_buckets)

  @classmethod
  def from_list(cls, vocabulary_list, num_oov_buckets=0):
    return cls(vocabulary_list, num_oov_buckets)

  @classmethod
  def from_file(cls, path, vocabulary_size=None, num_oov_buckets=0):
    """One token per line (the line without its line break); `vocabulary_size` keeps the
    first lines only and must not exceed the line count."""
    with open(path, 'rb') as f:
      lines = f.read().split(b'\n')
    if lines and lines[-1] == b'':
      lines.pop()
    lines = [l[:-1] if l.endswith(b'\r') else l for l in lines]
    if vocabulary_size is not None:
      if vocabulary_size < 1 or vocabulary_size > len(lines):
        raise ValueError('vocabulary_size %d: %s has %d tokens' %
                         (vocabulary_size, path, len(lines)))
      lines = lines[:vocabulary_size]
    return cls(lines, num_oov_buckets)

  @property
  def num_ids(self):
    """Rows an embedding table over this vocabulary needs."""
    return self.vocabulary_size + self.num_oov_buckets

  def lookup(self, tokens):
    """ids (int32 tensor) of a sequence of str / bytes tokens."""
    from ranking_b200 import _C
    toks = [t.encode() if isinstance(t, str) else bytes(t) for t in tokens]
    n = len(toks)
    out = torch.empty(n, dtype=torch.int32)
    arr = (ctypes.c_char_p * max(n, 1))(*toks)
    lens = (ctypes.c_int64 * max(n, 1))(*[len(t) for t in toks])
    _C.check(_C.lib.tfr_vocab_lookup(self._handle, arr, lens, n,
                                     ctypes.c_void_p(out.data_ptr())))
    return out

  def __len__(self):
    return self.vocabulary_size

  def __del__(self):
    if getattr(self, '_handle', None) is not None:
      try:
        from ranking_b200 import _C
        _C.lib.tfr_vocab_destroy(self._handle)
      except Exception:   # noqa: BLE001  (interpreter shutdown)
        pass
      self._handle = None


def _token_specs(token_feature_spec):
  """{'context': {name: (max_tokens, vocab)}, 'example': {...}} -> two (names, TokenSpec
  array, keep-alive) triples, in the given order."""
  from ranking_b200 import _C
  spec = dict(token_feature_spec or {})
  extra = set(spec) - {'context', 'example'}
  if extra:
    raise ValueError("token_feature_spec takes the keys 'context' and 'example', got %s" %
                     sorted(extra))
  out = []
  for kind in ('context', 'example'):
    items = list((spec.get(kind) or {}).items())
    arr = (_C.TokenSpec * max(len(items), 1))()
    keep = []
    for i, (name, (max_tokens, vocab)) in enumerate(items):
      if not isinstance(vocab, Vocabulary):
        raise ValueError('token feature %r: the vocabulary must be a data.Vocabulary' % name)
      if int(max_tokens) < 1:
        raise ValueError('token feature %r: max_tokens must be >= 1' % name)
      key = name.encode()
      keep += [key, vocab]
      arr[i].name = key
      arr[i].max_tokens = int(max_tokens)
      arr[i].vocab = vocab._handle
    out.append(([n for n, _ in items], [int(t) for _, (t, _) in items], arr, keep))
  return out


def parse_from_example_list(serialized, list_size, context_feature_spec=None,
                            example_feature_spec=None, pin_memory=False, num_threads=0,
                            data_format=EXAMPLE_LIST_WITH_CONTEXT, out=None,
                            token_feature_spec=None):
  """data.py:391-540 for dense float / int64 features.  `serialized`: a sequence of
  serialized ELWC protos; the specs map feature name -> (dim, default_value), in the
  column order wanted.  Returns dict(context [B, Dc], examples [B, list_size, De],
  sizes [B] int32, mask [B, list_size] bool) of CPU tensors.  Pass a previous result as
  `out` to decode into the same (e.g. pinned) buffers: fresh allocations are first touched
  inside the decoder threads and the page faults serialise them.

  Token (bytes_list) features: `token_feature_spec = {'context': {name: (max_tokens,
  vocab)}, 'example': {name: (max_tokens, vocab)}}` with `vocab` a `Vocabulary`.  The
  result then also holds `context_tokens` {name: int32 [B, max_tokens]}, `example_tokens`
  {name: int32 [B, list_size, max_tokens]} (a bag's first max_tokens ids in record order,
  -1 in the other slots, in missing features and in padded items) and `dropped_tokens`
  {name: number of tokens cut by max_tokens}."""
  from ranking_b200 import _C
  if data_format not in _FORMATS:
    raise ValueError('Data format {} is not supported.'.format(data_format))
  if token_feature_spec is not None:
    return _parse_with_tokens(serialized, list_size, context_feature_spec,
                              example_feature_spec, token_feature_spec, pin_memory,
                              num_threads, data_format)
  records = [r if isinstance(r, bytes) else bytes(r) for r in serialized]
  b = len(records)
  carr, nc, dc, keep_c = _spec_array(context_feature_spec)
  earr, ne, de, keep_e = _spec_array(example_feature_spec)
  ptrs = (ctypes.c_char_p * max(b, 1))(*records)
  lens = (ctypes.c_int64 * max(b, 1))(*[len(r) for r in records])

  def alloc(*shape, dtype=torch.float32):
    t = torch.empty(*shape, dtype=dtype)
    return t.pin_memory() if pin_memory and torch.cuda.is_available() else t

  if out is not None and tuple(out['examples'].shape) == (b, list_size, de) and \
      tuple(out['context'].shape) == (b, dc):
    ctx, ex, sizes = out['context'], out['examples'], out['sizes']
    mask = out['mask'].view(torch.uint8)
  else:
    ctx = alloc(b, dc)
    ex = alloc(b, list_size, de)
    sizes = torch.empty(b, dtype=torch.int32)
    mask = torch.empty(b, list_size, dtype=torch.uint8)
  _C.check(_C.lib.tfr_ranking_parse(
      _FORMATS[data_format], ptrs, lens, b, int(list_size), carr, nc, earr, ne,
      ctypes.c_void_p(ctx.data_ptr()) if dc else None,
      ctypes.c_void_p(ex.data_ptr()) if de else None,
      ctypes.c_void_p(sizes.data_ptr()), ctypes.c_void_p(mask.data_ptr()),
      int(num_threads)))
  del keep_c, keep_e
  return {'context': ctx, 'examples': ex, 'sizes': sizes, 'mask': mask.view(torch.bool)}


def _parse_with_tokens(serialized, list_size, context_feature_spec, example_feature_spec,
                       token_feature_spec, pin_memory, num_threads, data_format):
  from ranking_b200 import _C
  records = [r if isinstance(r, bytes) else bytes(r) for r in serialized]
  b = len(records)
  carr, nc, dc, keep_c = _spec_array(context_feature_spec)
  earr, ne, de, keep_e = _spec_array(example_feature_spec)
  (cnames, ct, ctarr, keep_ct), (enames, et, etarr, keep_et) = _token_specs(token_feature_spec)
  ptrs = (ctypes.c_char_p * max(b, 1))(*records)
  lens = (ctypes.c_int64 * max(b, 1))(*[len(r) for r in records])
  pin = pin_memory and torch.cuda.is_available()

  def alloc(*shape, dtype=torch.float32):
    t = torch.empty(*shape, dtype=dtype)
    return t.pin_memory() if pin else t

  ctx, ex = alloc(b, dc), alloc(b, list_size, de)
  sizes = torch.empty(b, dtype=torch.int32)
  mask = torch.empty(b, list_size, dtype=torch.uint8)
  ctok = [alloc(b, t, dtype=torch.int32) for t in ct]
  etok = [alloc(b, list_size, t, dtype=torch.int32) for t in et]
  cptr = (ctypes.c_void_p * max(len(ctok), 1))(*[t.data_ptr() for t in ctok])
  eptr = (ctypes.c_void_p * max(len(etok), 1))(*[t.data_ptr() for t in etok])
  dropped = torch.zeros(max(len(ctok) + len(etok), 1), dtype=torch.int64)
  _C.check(_C.lib.tfr_ranking_parse_tokens(
      _FORMATS[data_format], ptrs, lens, b, int(list_size), carr, nc, earr, ne,
      ctarr, len(ctok), etarr, len(etok),
      ctypes.c_void_p(ctx.data_ptr()) if dc else None,
      ctypes.c_void_p(ex.data_ptr()) if de else None, cptr, eptr,
      ctypes.c_void_p(dropped.data_ptr()), ctypes.c_void_p(sizes.data_ptr()),
      ctypes.c_void_p(mask.data_ptr()), int(num_threads)))
  del keep_c, keep_e, keep_ct, keep_et
  drops = dropped.tolist()
  return {'context': ctx, 'examples': ex, 'sizes': sizes, 'mask': mask.view(torch.bool),
          'context_tokens': dict(zip(cnames, ctok)),
          'example_tokens': dict(zip(enames, etok)),
          'dropped_tokens': dict(zip(cnames + enames, drops))}


def elwc_batches(paths, batch_size, list_size, context_feature_spec, example_feature_spec,
                 label_feature, drop_remainder=True, pin_memory=True, token_feature_spec=None):
  """Yields (x [B, list_size, Dc + De], y [B, list_size]) from TFRecord files of ELWC
  protos: context features first (repeated over the list), then the example features —
  the layout `DNNScorer` builds (keras/model.py:800-817).  `label_feature` names the
  example feature that holds the relevance label (give it the default -1 so that padded
  slots are invalid); it is removed from x.

  With `token_feature_spec` (see `parse_from_example_list`) it yields (x, y, tokens)
  instead, tokens = {'context': {name: int32 [B, T]}, 'example': {name: int32
  [B, list_size, T]}}: the batches `EmbeddingRankingTrainer` and `pipeline.fit` take."""
  ex_spec = dict(example_feature_spec)
  if label_feature not in ex_spec:
    raise ValueError('label feature %r is not in example_feature_spec' % label_feature)
  names = list(ex_spec)
  off = 0
  cols = []
  for name in names:
    dim = int(ex_spec[name][0])
    if name == label_feature:
      label_col = off
      if dim != 1:
        raise ValueError('the label feature must have dim 1')
    else:
      cols.extend(range(off, off + dim))
    off += dim
  buf = []

  def flush():
    out = parse_from_example_list(buf, list_size, context_feature_spec, ex_spec,
                                  token_feature_spec=token_feature_spec,
                                  pin_memory=pin_memory and token_feature_spec is not None)
    ex = out['examples']
    y = ex[:, :, label_col].clone()
    y = torch.where(out['mask'], y, torch.full_like(y, -1.))
    feats = ex[:, :, cols]
    if out['context'].shape[1]:
      ctx = out['context'].unsqueeze(1).expand(-1, list_size, -1)
      feats = torch.cat([ctx, feats], 2)
    x = feats.contiguous()
    if pin_memory and torch.cuda.is_available():
      x, y = x.pin_memory(), y.pin_memory()
    if token_feature_spec is None:
      return x, y
    return x, y, {'context': out['context_tokens'], 'example': out['example_tokens']}

  for path in ([paths] if isinstance(paths, str) else paths):
    for rec in read_tfrecords(path):
      buf.append(rec)
      if len(buf) == batch_size:
        yield flush()
        buf = []
  if buf and not drop_remainder:
    yield flush()


def elwc_multilabel_batches(paths, batch_size, list_size, context_feature_spec,
                            example_feature_spec, label_spec, sample_weight_feature=None,
                            drop_remainder=True, pin_memory=True):
  """Multi-task batches (the reference's `MultiLabelDatasetBuilder._features_and_labels`,
  keras/pipeline.py:1196-1221): yields (x [B, list_size, Dc + De], labels {task: [B,
  list_size]}, mask [B, list_size] bool, weights [B, list_size] or None).

  `label_spec` maps each task to the example feature holding its label (dim 1); give those
  features the default -1 so that an item without a task's label is invalid for that task.
  Padded slots are -1 in every task.  `sample_weight_feature` names an example feature (dim 1)
  holding the per-item weight shared by the tasks.  Label and weight columns are removed from
  x; `mask` is the decoder's list mask (real items, whatever their labels)."""
  ex_spec = dict(example_feature_spec)
  label_spec = dict(label_spec)
  if not label_spec:
    raise ValueError('label_spec must map at least one task to a label feature')
  special = {}
  for task, name in label_spec.items():
    special.setdefault(name, []).append(task)
  if sample_weight_feature is not None:
    if sample_weight_feature in special:
      raise ValueError('%r is both a label and the sample weight' % sample_weight_feature)
    special[sample_weight_feature] = []
  off, cols, where = 0, [], {}
  for name in ex_spec:
    dim = int(ex_spec[name][0])
    if name in special:
      if dim != 1:
        raise ValueError('label and weight features must have dim 1 (%r has %d)' % (name, dim))
      where[name] = off
    else:
      cols.extend(range(off, off + dim))
    off += dim
  missing = sorted(set(special) - set(where))
  if missing:
    raise ValueError('features %s are not in example_feature_spec' % missing)
  buf = []

  def flush():
    out = parse_from_example_list(buf, list_size, context_feature_spec, ex_spec,
                                  pin_memory=False)
    ex, mask = out['examples'], out['mask']
    pin = pin_memory and torch.cuda.is_available()
    labels = {}
    for task, name in label_spec.items():
      y = torch.where(mask, ex[:, :, where[name]], torch.full_like(ex[:, :, 0], -1.))
      labels[task] = y.pin_memory() if pin else y
    weights = None
    if sample_weight_feature is not None:
      weights = ex[:, :, where[sample_weight_feature]].contiguous()
      weights = weights.pin_memory() if pin else weights
    feats = ex[:, :, cols]
    if out['context'].shape[1]:
      ctx = out['context'].unsqueeze(1).expand(-1, list_size, -1)
      feats = torch.cat([ctx, feats], 2)
    x = feats.contiguous()
    if pin:
      x, mask = x.pin_memory(), mask.pin_memory()
    return x, labels, mask, weights

  for path in ([paths] if isinstance(paths, str) else paths):
    for rec in read_tfrecords(path):
      buf.append(rec)
      if len(buf) == batch_size:
        yield flush()
        buf = []
  if buf and not drop_remainder:
    yield flush()


class Prefetcher(object):
  """Runs a batch iterator (e.g. `elwc_batches(..., pin_memory=True)`: TFRecord read +
  native ELWC decode into pinned buffers) in a background thread, `depth` batches ahead, so
  that the host-side input work overlaps the device step.  `HostBatchPipeline.run` takes any
  iterable of (x_pinned, y_pinned), so

      pipe.run(Prefetcher(elwc_batches(paths, B, N, ctx_spec, ex_spec, 'label'), depth=4))

  is the whole input path of the reference's `make_dataset` -> `model.fit`
  (keras/pipeline.py:505-632) for dense features.  The decoder releases the GIL (it is a C
  call), so one thread here plus the decoder's own threads keep the cores busy.  Exceptions of
  the producer are re-raised at the consumer; `close()` (or exhausting / deleting the
  iterator) stops the thread."""

  _END = object()

  def __init__(self, batches, depth=2):
    import queue
    import threading
    if depth < 1:
      raise ValueError('depth must be >= 1')
    self._q = queue.Queue(maxsize=int(depth))
    self._stop = threading.Event()
    self._exc = None
    self._thread = threading.Thread(target=self._run, args=(iter(batches),), daemon=True)
    self._thread.start()

  def _put(self, item):
    import queue
    while not self._stop.is_set():
      try:
        self._q.put(item, timeout=0.1)
        return True
      except queue.Full:
        continue
    return False

  def _run(self, it):
    try:
      for batch in it:
        if not self._put(batch):
          return
    except BaseException as e:   # noqa: BLE001  (handed to the consumer)
      self._exc = e
    self._put(self._END)

  def __iter__(self):
    return self

  def __next__(self):
    if self._stop.is_set():
      raise StopIteration
    item = self._q.get()
    if item is self._END:
      self._stop.set()
      if self._exc is not None:
        raise self._exc
      raise StopIteration
    return item

  def close(self):
    self._stop.set()
    self._thread.join(timeout=5.0)

  def __del__(self):
    self._stop.set()
