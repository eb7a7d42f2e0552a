"""Token features without a GPU: the embedding oracle on the reference's feature-column
expectations, the vocabulary rules, and the native decoder's id tensors (ANTIQUE fixture and
records written by data.encode_*), checked against a pure-Python protobuf walk."""
import os
import struct

import pytest
import torch

import __graft_entry__

__graft_entry__.build()

from oracle import embedding as oemb  # noqa: E402
from ranking_b200 import data  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ANTIQUE = os.path.join(ROOT, 'tests', 'golden', 'antique')
TABLE = torch.tensor([[1., 2.], [3., 5.], [7., 11.], [9., 13.]], dtype=torch.float64)


# ---- oracle: python/feature_test.py:100-239 and keras/feature_test.py:28-145 ----------------
def test_encode_features_mean_combiner():
  """feature_test.py:100-168: ids of -1 are ignored, an empty bag is a zero vector."""
  a = torch.tensor([[3, -1, -1], [0, 1, -1]])
  b = torch.tensor([[0, -1, -1], [-1, -1, -1]])
  assert oemb.pool(a, TABLE).tolist() == [[9., 13.], [2., 3.5]]
  assert oemb.pool(b, TABLE).tolist() == [[1., 2.], [0., 0.]]


def test_combiners_and_repeated_ids():
  ids = torch.tensor([[0, 1, -1, -1], [2, 2, 3, -1], [-1, -1, -1, -1]])
  s = oemb.pool(ids, TABLE, 'sum')
  assert s.tolist() == [[4., 7.], [23., 35.], [0., 0.]]
  m = oemb.pool(ids, TABLE, 'mean')
  assert torch.allclose(m, torch.tensor([[2., 3.5], [23 / 3, 35 / 3], [0., 0.]],
                                        dtype=torch.float64))
  q = oemb.pool(ids, TABLE, 'sqrtn')
  assert torch.allclose(q[1], torch.tensor([23., 35.], dtype=torch.float64) / 3 ** 0.5)
  assert q[2].tolist() == [0., 0.]


def test_sequence_embedding():
  """feature_test.py:170-239."""
  ids = torch.tensor([[3, -1, -1], [0, 1, -1]])
  assert oemb.sequence_embedding(ids, TABLE).tolist() == [
      [[9., 13.], [0., 0.], [0., 0.]], [[1., 2.], [3., 5.], [0., 0.]]]


def test_table_gradient_counts_every_occurrence():
  table = TABLE.clone().requires_grad_()
  ids = torch.tensor([[2, 2, 0, -1], [-1, -1, -1, -1]])
  oemb.pool(ids, table, 'mean').sum().backward()
  want = torch.zeros(4, 2, dtype=torch.float64)
  want[2] = 2 / 3
  want[0] = 1 / 3
  assert torch.allclose(table.grad, want)


def test_vocabulary_list_embedding_in_listwise_features():
  """keras/feature_test.py:28-145: `unigrams` over the vocabulary list ['ranking',
  'regression', 'classification', 'ordinal'], one token per item of a [2, 2] batch,
  embeds to [2, 2, dimension]."""
  vocab = data.Vocabulary.from_list(['ranking', 'regression', 'classification', 'ordinal'])
  ids = vocab.lookup(['ranking', 'regression', 'classification', 'ordinal']).reshape(2, 2, 1)
  assert ids.tolist() == [[[0], [1]], [[2], [3]]]
  table = torch.randn(4, 10, dtype=torch.float64, generator=torch.Generator().manual_seed(0))
  out = oemb.pool(ids, table)
  assert list(out.shape) == [2, 2, 10]
  assert torch.equal(out.reshape(4, 10), table)


# ---- vocabulary rules ------------------------------------------------------------------
def test_vocabulary_file_order_and_oov(tmp_path):
  p = tmp_path / 'vocab.txt'
  p.write_bytes(b'b\na\nc\r\nd\n')
  v = data.Vocabulary.from_file(str(p))
  assert v.tokens == [b'b', b'a', b'c', b'd'] and len(v) == 4 and v.num_ids == 4
  assert v.lookup(['a', 'b', 'c', 'd', 'zzz', '']).tolist() == [1, 0, 2, 3, -1, -1]
  v1 = data.Vocabulary.from_file(str(p), num_oov_buckets=1)
  assert v1.num_ids == 5
  assert v1.lookup(['zzz', 'd']).tolist() == [4, 3]
  v2 = data.Vocabulary.from_file(str(p), vocabulary_size=2)
  assert v2.lookup(['b', 'a', 'c']).tolist() == [0, 1, -1]
  with pytest.raises(ValueError):
    data.Vocabulary.from_file(str(p), vocabulary_size=5)


def test_vocabulary_rejects_duplicates_and_hash_buckets():
  with pytest.raises(ValueError, match='duplicate'):
    data.Vocabulary.from_list(['a', 'b', 'a'])
  with pytest.raises(ValueError, match='num_oov_buckets'):
    data.Vocabulary.from_list(['a', 'b'], num_oov_buckets=2)


def test_antique_vocabulary():
  v = data.Vocabulary.from_file(os.path.join(ANTIQUE, 'vocab.txt'))
  assert [t.decode() for t in v.tokens] == ['relevant', 'question', 'answer', 'irrelevant',
                                            'data']


# ---- a pure-Python protobuf walk (the checker of the native decoder) -------------------
def _fields(buf):
  i = 0
  while i < len(buf):
    tag, i = _varint(buf, i)
    f, w = tag >> 3, tag & 7
    if w == 0:
      v, i = _varint(buf, i)
    elif w == 2:
      n, i = _varint(buf, i)
      v, i = buf[i:i + n], i + n
    elif w == 5:
      v, i = buf[i:i + 4], i + 4
    elif w == 1:
      v, i = buf[i:i + 8], i + 8
    else:
      raise ValueError(w)
    yield f, w, v


def _varint(buf, i):
  v, s = 0, 0
  while True:
    b = buf[i]
    i += 1
    v |= (b & 0x7f) << s
    s += 7
    if not b & 0x80:
      return v, i


def _features(example):
  """Serialized tf.Example -> {name: ('bytes', [..]) | ('int64', [..]) | ('float', [..])}."""
  out = {}
  for f, _, features in _fields(example):
    if f != 1:
      continue
    for f2, _, entry in _fields(features):
      key = value = None
      for f3, _, v in _fields(entry):
        if f3 == 1:
          key = v.decode()
        elif f3 == 2:
          value = v
      out[key] = _feature(value)
  return out


def _feature(value):
  for f, _, lst in _fields(value):
    if f == 1:
      return 'bytes', [v for g, _, v in _fields(lst) if g == 1]
    if f == 3:
      vals = []
      for g, w, v in _fields(lst):
        if w == 2:
          j = 0
          while j < len(v):
            x, j = _varint(v, j)
            vals.append(x)
        else:
          vals.append(v)
      return 'int64', vals
    if f == 2:
      vals = []
      for g, w, v in _fields(lst):
        vals += list(struct.unpack('<%df' % (len(v) // 4), v)) if w == 2 else \
            [struct.unpack('<f', v)[0]]
      return 'float', vals
  return 'bytes', []


def _elwc(record):
  examples, context = [], {}
  for f, _, v in _fields(record):
    if f == 1:
      examples.append(_features(v))
    elif f == 2:
      context = _features(v)
  return context, examples


def _bag(feats, name, vocab, t):
  toks = feats.get(name, ('bytes', []))[1]
  oov = len(vocab.tokens) if vocab.num_oov_buckets else -1
  ids = [{tok: i for i, tok in enumerate(vocab.tokens)}.get(tok, oov) for tok in toks]
  return (ids[:t] + [-1] * t)[:t], max(0, len(ids) - t)


def _check_against_walk(records, vocab, list_size, tq, td, data_format=data.EXAMPLE_LIST_WITH_CONTEXT,
                        walked=None):
  spec = {'context': {'query_tokens': (tq, vocab)}, 'example': {'document_tokens': (td, vocab)}}
  out = data.parse_from_example_list(records, list_size, None, {'relevance': (1, -1)},
                                     data_format=data_format, token_feature_spec=spec,
                                     num_threads=3)
  q = out['context_tokens']['query_tokens']
  d = out['example_tokens']['document_tokens']
  assert q.dtype == torch.int32 and list(q.shape) == [len(records), tq]
  assert list(d.shape) == [len(records), list_size, td]
  dropped_q = dropped_d = 0
  for b, rec in enumerate(records):
    ctx, examples = walked[b] if walked else _elwc(rec)
    want, drop = _bag(ctx, 'query_tokens', vocab, tq)
    dropped_q += drop
    assert q[b].tolist() == want, b
    assert int(out['sizes'][b]) == len(examples)
    for i in range(list_size):
      if i < len(examples):
        want, drop = _bag(examples[i], 'document_tokens', vocab, td)
        dropped_d += drop
        assert d[b, i].tolist() == want, (b, i)
        rel = examples[i].get('relevance', ('int64', []))[1]
        assert float(out['examples'][b, i, 0]) == (float(rel[0]) if rel else -1.0)
      else:
        assert d[b, i].tolist() == [-1] * td
  assert out['dropped_tokens'] == {'query_tokens': dropped_q, 'document_tokens': dropped_d}
  return out


def _fixture_records():
  return list(data.read_tfrecords(os.path.join(ANTIQUE, 'train_elwc.tfrecord')))


def test_antique_fixture_ids_match_protobuf_walk():
  records = _fixture_records()
  assert len(records) == 10
  vocab = data.Vocabulary.from_file(os.path.join(ANTIQUE, 'vocab.txt'))
  walked = [_elwc(r) for r in records]
  longest_q = max(len(c.get('query_tokens', ('', []))[1]) for c, _ in walked)
  longest_d = max(len(e.get('document_tokens', ('', []))[1]) for _, ex in walked for e in ex)
  assert longest_q >= 1 and longest_d >= 1
  # every bag whole, then truncated to 1 token; list_size 50 (the example's) pads
  out = _check_against_walk(records, vocab, 50, longest_q, longest_d)
  assert out['dropped_tokens'] == {'query_tokens': 0, 'document_tokens': 0}
  _check_against_walk(records, vocab, 50, 1, 1)
  _check_against_walk(records, vocab, 1, longest_q + 3, longest_d + 4)


def test_antique_fixture_batches():
  vocab = data.Vocabulary.from_file(os.path.join(ANTIQUE, 'vocab.txt'))
  spec = {'context': {'query_tokens': (8, vocab)}, 'example': {'document_tokens': (8, vocab)}}
  path = os.path.join(ANTIQUE, 'train_elwc.tfrecord')
  batches = list(data.elwc_batches(path, 4, 50, None, {'relevance': (1, -1)}, 'relevance',
                                   drop_remainder=False, pin_memory=False,
                                   token_feature_spec=spec))
  assert [b[0].shape[0] for b in batches] == [4, 4, 2]
  for x, y, tokens in batches:
    assert list(x.shape[1:]) == [50, 0]
    assert list(tokens['context']['query_tokens'].shape) == [x.shape[0], 8]
    assert list(tokens['example']['document_tokens'].shape) == [x.shape[0], 50, 8]
    assert bool((y[:, 2:] == -1).all())
  # without token features the batches are (x, y) pairs, as before
  pairs = list(data.elwc_batches(path, 4, 50, None, {'relevance': (1, -1)}, 'relevance',
                                 pin_memory=False))
  assert all(len(p) == 2 for p in pairs) and len(pairs) == 2


def _lists():
  """Lists with truncation, empty bags, missing features, OOV tokens and a padded tail."""
  return [
      ({'q': ['a', 'b', 'zzz', 'c', 'a']},
       [{'d': ['a', 'a', 'b'], 'rel': [2]}, {'d': [], 'rel': [0]},
        {'rel': [1]}, {'d': ['c', 'b', 'a', 'zzz', 'c', 'c', 'b'], 'rel': [1]}]),
      ({}, [{'d': ['zzz'], 'rel': [0]}]),
      ({'q': []}, []),
      ({'q': ['c']}, [{'d': ['b', 'c'], 'rel': [3]}, {'d': ['a'], 'rel': [1]},
                      {'d': ['a', 'b'], 'rel': [0]}]),
  ]


def _walk_lists(lists):
  out = []
  for ctx, examples in lists:
    c = {k: ('bytes', [t.encode() for t in v]) for k, v in ctx.items()}
    ex = []
    for e in examples:
      ex.append({k: ('bytes', [t.encode() for t in v]) if k != 'rel' else ('int64', v)
                 for k, v in e.items()})
    out.append((c, ex))
  return out


def _rename(walked):
  """q / d -> the names _check_against_walk reads."""
  ren = {'q': 'query_tokens', 'd': 'document_tokens', 'rel': 'relevance'}
  return [({ren[k]: v for k, v in c.items()},
           [{ren[k]: v for k, v in e.items()} for e in ex]) for c, ex in walked]


@pytest.mark.parametrize('fmt', [data.EXAMPLE_LIST_WITH_CONTEXT, data.EXAMPLE_IN_EXAMPLE,
                                 data.SEQUENCE_EXAMPLE])
@pytest.mark.parametrize('oov', [0, 1])
def test_encoded_records_every_format(fmt, oov):
  vocab = data.Vocabulary.from_list(['a', 'b', 'c'], num_oov_buckets=oov)
  ren = {'q': 'query_tokens', 'd': 'document_tokens', 'rel': 'relevance'}
  lists = [({ren[k]: v for k, v in c.items()}, [{ren[k]: v for k, v in e.items()} for e in ex])
           for c, ex in _lists()]
  if fmt == data.EXAMPLE_LIST_WITH_CONTEXT:
    records = [data.encode_elwc(c, ex) for c, ex in lists]
  elif fmt == data.EXAMPLE_IN_EXAMPLE:
    records = [data.encode_example_in_example(c, ex) for c, ex in lists]
  else:
    records = [data.encode_sequence_example(c, ex, ['document_tokens', 'relevance'])
               for c, ex in lists]
  walked = _rename(_walk_lists(_lists()))
  for list_size, tq, td in [(4, 5, 7), (3, 2, 2), (5, 8, 8)]:
    _check_against_walk(records, vocab, list_size, tq, td, data_format=fmt, walked=walked)
  out = data.parse_from_example_list(
      records, 4, None, None, data_format=fmt,
      token_feature_spec={'context': {'query_tokens': (4, vocab)},
                          'example': {'document_tokens': (4, vocab)}})
  q = out['context_tokens']['query_tokens']
  oov_id = 3 if oov else -1
  assert q[0].tolist() == [0, 1, oov_id, 2]
  assert out['dropped_tokens'] == {'query_tokens': 1, 'document_tokens': 3}


def test_token_feature_errors():
  vocab = data.Vocabulary.from_list(['a'])
  rec = data.encode_elwc({}, [{'d': [1.5, 2.5]}])
  with pytest.raises(ValueError, match='float_list'):
    data.parse_from_example_list([rec], 2, token_feature_spec={'example': {'d': (4, vocab)}})
  with pytest.raises(ValueError, match='context'):
    data.parse_from_example_list([rec], 2, token_feature_spec={'examples': {'d': (4, vocab)}})
  with pytest.raises(ValueError, match='max_tokens'):
    data.parse_from_example_list([rec], 2, token_feature_spec={'example': {'d': (0, vocab)}})
  # an empty float list is an empty bag, not an error
  rec = data.encode_elwc({}, [{'d': []}])
  out = data.parse_from_example_list([rec], 2, token_feature_spec={'example': {'d': (4, vocab)}})
  assert out['example_tokens']['d'].tolist() == [[[-1] * 4, [-1] * 4]]
