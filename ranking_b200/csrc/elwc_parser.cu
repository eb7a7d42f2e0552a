// Input side of the hot path (host code, no device work): decoding batches of serialized
// `ExampleListWithContext` protos — the reference's training data format — straight into
// the dense [B, N, D] / [B, Dc] float buffers the scorer consumes, with the padding /
// truncation semantics of data.py:133-208 (`_ExampleInExampleParser.parse`) and
// data.py:391-540 (`parse_from_example_list`) for FixedLen float / int64 features.
//
// Wire format handled here (protobuf, proto3 encodings):
//   ExampleListWithContext { repeated Example examples = 1; Example context = 2; }
//   Example  { Features features = 1; }
//   Features { map<string, Feature> feature = 1; }   entry { string key = 1; Feature value = 2; }
//   Feature  { oneof { BytesList bytes_list = 1; FloatList float_list = 2; Int64List int64_list = 3; } }
//   FloatList { repeated float value = 1; }  Int64List { repeated int64 value = 1; }   (packed or not)
//
// Token features (bytes_list, e.g. `query_tokens` / `document_tokens` of the reference's ANTIQUE
// examples) decode through a vocabulary into int32 id slots: [B, T] for context features,
// [B, list_size, T] for example features, -1 in unused slots (tfr_ranking_parse_tokens).
#include <algorithm>
#include <atomic>
#include <cstring>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "common.cuh"

namespace tfr {
namespace {

struct Span {
  const uint8_t* p;
  const uint8_t* end;
  bool ok() const { return p <= end; }
  bool done() const { return p >= end; }
};

bool read_varint(Span& s, uint64_t* out) {
  uint64_t v = 0;
  for (int shift = 0; shift < 64 && s.p < s.end; shift += 7) {
    const uint8_t b = *s.p++;
    v |= static_cast<uint64_t>(b & 0x7f) << shift;
    if (!(b & 0x80)) {
      *out = v;
      return true;
    }
  }
  return false;
}

// Reads a tag; for length-delimited fields returns the payload span.
bool read_field(Span& s, uint32_t* field, uint32_t* wire, Span* payload, uint64_t* scalar) {
  uint64_t tag;
  if (!read_varint(s, &tag)) return false;
  *field = static_cast<uint32_t>(tag >> 3);
  *wire = static_cast<uint32_t>(tag & 7);
  switch (*wire) {
    case 0:
      return read_varint(s, scalar);
    case 1:
      if (s.end - s.p < 8) return false;
      std::memcpy(scalar, s.p, 8);
      s.p += 8;
      return true;
    case 2: {
      uint64_t len;
      if (!read_varint(s, &len) || len > static_cast<uint64_t>(s.end - s.p)) return false;
      payload->p = s.p;
      payload->end = s.p + len;
      s.p += len;
      return true;
    }
    case 5: {
      if (s.end - s.p < 4) return false;
      uint32_t v;
      std::memcpy(&v, s.p, 4);
      *scalar = v;
      s.p += 4;
      return true;
    }
    default:
      return false;
  }
}

struct Spec {
  std::string name;
  int dim;
  float default_value;
  int offset;   // column offset in the output row
};

// Parses a FloatList / Int64List payload into dst[0..dim); returns the value count.
int parse_values(Span list, bool is_float, float* dst, int dim) {
  int n = 0;
  while (!list.done()) {
    uint32_t f, w;
    Span pl{nullptr, nullptr};
    uint64_t sc = 0;
    if (!read_field(list, &f, &w, &pl, &sc)) return -1;
    if (f != 1) continue;
    if (is_float) {
      if (w == 2) {               // packed
        const size_t cnt = static_cast<size_t>(pl.end - pl.p) / 4;
        for (size_t i = 0; i < cnt; ++i, ++n)
          if (n < dim) std::memcpy(dst + n, pl.p + 4 * i, 4);
      } else if (w == 5) {
        const uint32_t bits = static_cast<uint32_t>(sc);
        if (n < dim) std::memcpy(dst + n, &bits, 4);
        ++n;
      } else {
        return -1;
      }
    } else {
      if (w == 2) {               // packed varints
        while (!pl.done()) {
          uint64_t v;
          if (!read_varint(pl, &v)) return -1;
          if (n < dim) dst[n] = static_cast<float>(static_cast<int64_t>(v));
          ++n;
        }
      } else if (w == 0) {
        if (n < dim) dst[n] = static_cast<float>(static_cast<int64_t>(sc));
        ++n;
      } else {
        return -1;
      }
    }
  }
  return n;
}

}  // namespace
}  // namespace tfr

// Token vocabulary (categorical_column_with_vocabulary_file / _list): token -> id in
// [0, size); an unknown token maps to `size` with one OOV bucket, to -1 without.
struct tfr_vocab_impl {
  std::unordered_map<std::string, int32_t> ids;
  int32_t size = 0;
  int32_t num_oov_buckets = 0;
  int32_t lookup(const uint8_t* p, size_t n) const {
    auto it = ids.find(std::string(reinterpret_cast<const char*>(p), n));
    if (it != ids.end()) return it->second;
    return num_oov_buckets ? size : -1;
  }
};

namespace tfr {
namespace {

// A bytes_list feature decoded into `max_tokens` id slots.
struct TokSpec {
  std::string name;
  int max_tokens;
  const tfr_vocab_impl* vocab;
};

// Where one Example (or one SequenceExample frame / context) lands: the dense row and, for
// token feature k, the slots base[k] + row_index * max_tokens[k].
struct Dest {
  const std::vector<Spec>* specs;
  float* row;
  const std::vector<TokSpec>* toks;
  int32_t* const* base;
  int64_t row_index;
  int64_t* dropped;   // per token feature: tokens past max_tokens
  int32_t* ids(int k) const {
    return base[k] + row_index * (*toks)[k].max_tokens;
  }
};

// One Feature message (oneof bytes / float / int64 list) -> row[spec.offset ..].
int parse_feature_value(Span value, const Spec& spec, float* row) {
  while (!value.done()) {
    uint32_t f, w;
    Span list{nullptr, nullptr};
    uint64_t sc;
    if (!read_field(value, &f, &w, &list, &sc)) return TFR_INVALID_ARGUMENT;
    if (w != 2) continue;
    if (f == 1) {
      set_error("feature '%s' is a bytes_list; only float_list / int64_list features can "
                "be decoded into the dense scorer input", spec.name.c_str());
      return TFR_UNSUPPORTED;
    }
    const int n = parse_values(list, f == 2, row + spec.offset, spec.dim);
    if (n < 0) return TFR_INVALID_ARGUMENT;
    if (n != spec.dim && n != 0) {   // tf.io.FixedLenFeature: exact length or missing
      set_error("feature '%s' has %d values, the spec says %d", spec.name.c_str(), n, spec.dim);
      return TFR_INVALID_ARGUMENT;
    }
  }
  return TFR_OK;
}

const Spec* find_spec(const std::vector<Spec>& specs, Span key) {
  const size_t klen = static_cast<size_t>(key.end - key.p);
  for (const Spec& s : specs)
    if (s.name.size() == klen && std::memcmp(s.name.data(), key.p, klen) == 0) return &s;
  return nullptr;
}

// Splits one map entry { key = 1; value = 2 } of Features / FeatureLists.
bool read_entry(Span entry, Span* key, Span* value) {
  key->p = value->p = nullptr;
  while (!entry.done()) {
    uint32_t f, w;
    Span pl{nullptr, nullptr};
    uint64_t sc;
    if (!read_field(entry, &f, &w, &pl, &sc)) return false;
    if (w != 2) continue;
    if (f == 1) *key = pl;
    if (f == 2) *value = pl;
  }
  return true;
}

int find_tok(const std::vector<TokSpec>* toks, Span key) {
  if (!toks) return -1;
  const size_t klen = static_cast<size_t>(key.end - key.p);
  for (size_t k = 0; k < toks->size(); ++k) {
    const std::string& n = (*toks)[k].name;
    if (n.size() == klen && std::memcmp(n.data(), key.p, klen) == 0) return static_cast<int>(k);
  }
  return -1;
}

// One Feature message of a token feature -> ids[0 .. max_tokens) (pre-filled with -1).  The
// first max_tokens tokens are kept; the rest are counted in *dropped.  An empty float / int64
// list is an empty bag; a non-empty one is an error.
int parse_token_value(Span value, const TokSpec& spec, int32_t* ids, int64_t* dropped) {
  int n = 0;
  while (!value.done()) {
    uint32_t f, w;
    Span list{nullptr, nullptr};
    uint64_t sc;
    if (!read_field(value, &f, &w, &list, &sc)) return TFR_INVALID_ARGUMENT;
    if (w != 2) continue;
    if (f == 2 || f == 3) {
      const int cnt = parse_values(list, f == 2, nullptr, 0);
      if (cnt < 0) return TFR_INVALID_ARGUMENT;
      if (cnt > 0) {
        set_error("token feature '%s' is a %s; token features must be bytes_list",
                  spec.name.c_str(), f == 2 ? "float_list" : "int64_list");
        return TFR_UNSUPPORTED;
      }
      continue;
    }
    if (f != 1) continue;
    while (!list.done()) {
      Span v{nullptr, nullptr};
      if (!read_field(list, &f, &w, &v, &sc)) return TFR_INVALID_ARGUMENT;
      if (f != 1 || w != 2) continue;
      if (n < spec.max_tokens)
        ids[n] = spec.vocab->lookup(v.p, static_cast<size_t>(v.end - v.p));
      else
        ++*dropped;
      ++n;
    }
  }
  return TFR_OK;
}

// A Features message -> dest (already filled with the defaults).
int parse_features(Span features, const Dest& d) {
  while (!features.done()) {
    uint32_t f, w;
    Span entry{nullptr, nullptr};
    uint64_t sc;
    if (!read_field(features, &f, &w, &entry, &sc)) return TFR_INVALID_ARGUMENT;
    if (f != 1 || w != 2) continue;
    Span key, value;
    if (!read_entry(entry, &key, &value)) return TFR_INVALID_ARGUMENT;
    if (!key.p || !value.p) continue;
    const Spec* spec = find_spec(*d.specs, key);
    if (spec) {
      const int rc = parse_feature_value(value, *spec, d.row);
      if (rc) return rc;
      continue;
    }
    const int k = find_tok(d.toks, key);
    if (k < 0) continue;            // feature not requested
    const int rc = parse_token_value(value, (*d.toks)[k], d.ids(k), d.dropped + k);
    if (rc) return rc;
  }
  return TFR_OK;
}

// One serialized tf.Example { Features features = 1 } -> dest.
int parse_example(Span ex, const Dest& d) {
  while (!ex.done()) {
    uint32_t f, w;
    Span features{nullptr, nullptr};
    uint64_t sc;
    if (!read_field(ex, &f, &w, &features, &sc)) return TFR_INVALID_ARGUMENT;
    if (f != 1 || w != 2) continue;
    const int rc = parse_features(features, d);
    if (rc) return rc;
  }
  return TFR_OK;
}

// Visits the values of a bytes_list Feature.
template <typename Fn>
int for_each_bytes(Span feature, Fn fn) {
  while (!feature.done()) {
    uint32_t f, w;
    Span list{nullptr, nullptr};
    uint64_t sc;
    if (!read_field(feature, &f, &w, &list, &sc)) return TFR_INVALID_ARGUMENT;
    if (f != 1 || w != 2) continue;       // bytes_list
    while (!list.done()) {
      Span v{nullptr, nullptr};
      if (!read_field(list, &f, &w, &v, &sc)) return TFR_INVALID_ARGUMENT;
      if (f != 1 || w != 2) continue;
      const int rc = fn(v);
      if (rc) return rc;
    }
  }
  return TFR_OK;
}

std::vector<Spec> make_specs(const tfr_feature_spec* in, int n, int* total) {
  std::vector<Spec> out;
  int off = 0;
  for (int i = 0; i < n; ++i) {
    out.push_back(Spec{in[i].name ? in[i].name : "", in[i].dim, in[i].default_value, off});
    off += in[i].dim;
  }
  *total = off;
  return out;
}

void fill_defaults(const std::vector<Spec>& specs, float* row) {
  for (const Spec& s : specs)
    for (int j = 0; j < s.dim; ++j) row[s.offset + j] = s.default_value;
}

// CRC-32C (Castagnoli), the checksum of the TFRecord framing.
uint32_t crc32c(const uint8_t* p, size_t n) {
  static uint32_t table[256];
  static bool init = false;
  if (!init) {
    for (uint32_t i = 0; i < 256; ++i) {
      uint32_t c = i;
      for (int k = 0; k < 8; ++k) c = (c & 1) ? (c >> 1) ^ 0x82F63B78u : c >> 1;
      table[i] = c;
    }
    init = true;
  }
  uint32_t c = 0xFFFFFFFFu;
  for (size_t i = 0; i < n; ++i) c = table[(c ^ p[i]) & 0xFF] ^ (c >> 8);
  return c ^ 0xFFFFFFFFu;
}

}  // namespace
}  // namespace tfr

using namespace tfr;

extern "C" uint32_t tfr_masked_crc32c(const uint8_t* data, size_t n) {
  const uint32_t c = crc32c(data, n);
  return ((c >> 15) | (c << 17)) + 0xa282ead8u;   // TFRecord's masking
}

extern "C" int tfr_vocab_create(const char* const* tokens, const int64_t* token_sizes, int n,
                                int num_oov_buckets, void** vocab_out) {
  TFR_REQUIRE(vocab_out && n >= 0 && (n == 0 || (tokens && token_sizes)), "bad arguments");
  TFR_REQUIRE(num_oov_buckets == 0 || num_oov_buckets == 1,
              "num_oov_buckets=%d: only 0 (unknown tokens are ignored) or 1 (one OOV row) are "
              "supported; more buckets need TF's Fingerprint64 hashing", num_oov_buckets);
  *vocab_out = nullptr;
  tfr_vocab_impl* v = new tfr_vocab_impl();
  v->num_oov_buckets = num_oov_buckets;
  v->ids.reserve(static_cast<size_t>(n));
  for (int i = 0; i < n; ++i) {
    std::string tok(tokens[i], static_cast<size_t>(token_sizes[i]));
    if (!v->ids.emplace(tok, i).second) {
      set_error("duplicate vocabulary token '%s' (lines %d and %d)", tok.c_str(),
                v->ids[tok] + 1, i + 1);
      delete v;
      return TFR_INVALID_ARGUMENT;
    }
  }
  v->size = n;
  *vocab_out = v;
  return TFR_OK;
}

extern "C" int tfr_vocab_destroy(void* vocab) {
  delete static_cast<tfr_vocab_impl*>(vocab);
  return TFR_OK;
}

extern "C" int tfr_vocab_lookup(const void* vocab, const char* const* tokens,
                                const int64_t* token_sizes, int n, int32_t* ids_out) {
  TFR_REQUIRE(vocab && n >= 0 && (n == 0 || (tokens && token_sizes && ids_out)), "bad arguments");
  const tfr_vocab_impl* v = static_cast<const tfr_vocab_impl*>(vocab);
  for (int i = 0; i < n; ++i)
    ids_out[i] = v->lookup(reinterpret_cast<const uint8_t*>(tokens[i]),
                           static_cast<size_t>(token_sizes[i]));
  return TFR_OK;
}

static int parse_batch(int format, const uint8_t* const* records, const int64_t* record_sizes,
                       int B, int list_size, const tfr_feature_spec* context_spec, int n_context,
                       const tfr_feature_spec* example_spec, int n_example,
                       const tfr_token_spec* context_tokens, int n_context_tokens,
                       const tfr_token_spec* example_tokens, int n_example_tokens,
                       float* context_out, float* example_out, int32_t* const* context_ids_out,
                       int32_t* const* example_ids_out, int64_t* dropped_out,
                       int32_t* sizes_out, uint8_t* mask_out, int n_threads) {
  TFR_REQUIRE(format >= TFR_FORMAT_ELWC && format <= TFR_FORMAT_SEQUENCE_EXAMPLE,
              "format %d is not a tfr_data_format", format);
  TFR_REQUIRE(records && record_sizes && B >= 0 && list_size >= 1, "bad arguments");
  TFR_REQUIRE(n_context >= 0 && n_example >= 0, "bad feature counts");
  TFR_REQUIRE(n_example == 0 || example_out, "example_out must not be NULL");
  TFR_REQUIRE(n_context == 0 || context_out, "context_out must not be NULL");
  TFR_REQUIRE(n_context == 0 || context_spec, "context_spec must not be NULL");
  TFR_REQUIRE(n_example == 0 || example_spec, "example_spec must not be NULL");
  {   // every dim >= 1 and the row widths fit an int: the offsets below index the outputs
    long long wc = 0, we = 0;
    for (int i = 0; i < n_context; ++i) {
      TFR_REQUIRE(context_spec[i].dim >= 1, "context feature %d has dim %d", i, context_spec[i].dim);
      wc += context_spec[i].dim;
    }
    for (int i = 0; i < n_example; ++i) {
      TFR_REQUIRE(example_spec[i].dim >= 1, "example feature %d has dim %d", i, example_spec[i].dim);
      we += example_spec[i].dim;
    }
    TFR_REQUIRE(wc < (1ll << 30) && we < (1ll << 30), "feature rows are too wide");
  }
  int dc = 0, de = 0;
  const std::vector<Spec> cspec = make_specs(context_spec, n_context, &dc);
  const std::vector<Spec> espec = make_specs(example_spec, n_example, &de);
  TFR_REQUIRE(n_context_tokens >= 0 && n_example_tokens >= 0, "bad token feature counts");
  TFR_REQUIRE(n_context_tokens == 0 || (context_tokens && context_ids_out),
              "context token specs / outputs must not be NULL");
  TFR_REQUIRE(n_example_tokens == 0 || (example_tokens && example_ids_out),
              "example token specs / outputs must not be NULL");
  auto make_toks = [](const tfr_token_spec* in, int n, int32_t* const* outs,
                      std::vector<TokSpec>* out) -> int {
    for (int i = 0; i < n; ++i) {
      TFR_REQUIRE(in[i].max_tokens >= 1, "token feature %d has max_tokens %d", i,
                  in[i].max_tokens);
      TFR_REQUIRE(in[i].vocab && outs[i], "token feature %d: NULL vocabulary or output", i);
      out->push_back(TokSpec{in[i].name ? in[i].name : "", in[i].max_tokens,
                             static_cast<const tfr_vocab_impl*>(in[i].vocab)});
    }
    return TFR_OK;
  };
  std::vector<TokSpec> ctoks, etoks;
  if (int rc = make_toks(context_tokens, n_context_tokens, context_ids_out, &ctoks)) return rc;
  if (int rc = make_toks(example_tokens, n_example_tokens, example_ids_out, &etoks)) return rc;
  const int nct = n_context_tokens, nk = n_context_tokens + n_example_tokens;
  const bool has_ctx = dc || nct, has_ex = de || n_example_tokens;
  // tokens dropped by truncation, per list and token feature (summed after the threads join)
  std::vector<int64_t> dropped(static_cast<size_t>(B) * (nk ? nk : 1), 0);

  // one list = one independent unit of work
  auto parse_one = [&](int b) -> int {
    Span rec{records[b], records[b] + record_sizes[b]};
    float* crow = dc ? context_out + static_cast<size_t>(b) * dc : nullptr;
    if (crow) fill_defaults(cspec, crow);
    // padded slots are parsed from an empty Example in the reference: every feature takes
    // its default (data.py:170-183); token slots hold -1 (an empty bag)
    for (int i = 0; i < list_size && de; ++i)
      fill_defaults(espec, example_out + (static_cast<size_t>(b) * list_size + i) * de);
    for (int k = 0; k < nct; ++k)
      std::fill_n(context_ids_out[k] + static_cast<size_t>(b) * ctoks[k].max_tokens,
                  ctoks[k].max_tokens, -1);
    for (int k = 0; k < n_example_tokens; ++k)
      std::fill_n(example_ids_out[k] + static_cast<size_t>(b) * list_size * etoks[k].max_tokens,
                  static_cast<size_t>(list_size) * etoks[k].max_tokens, -1);
    int64_t* drop = dropped.data() + static_cast<size_t>(b) * nk;
    const Dest cdest{&cspec, crow, &ctoks, context_ids_out, b, drop};
    int count = 0;
    auto example_row = [&](int i) {
      const int64_t r = static_cast<int64_t>(b) * list_size + i;
      return Dest{&espec, de ? example_out + r * de : nullptr, &etoks, example_ids_out, r,
                  drop + nct};
    };
    auto bad_record = [&]() {
      set_error("record %d is not a valid %s", b,
                format == TFR_FORMAT_ELWC ? "ExampleListWithContext"
                : format == TFR_FORMAT_EXAMPLE_IN_EXAMPLE ? "Example-in-Example record"
                                                          : "SequenceExample");
      return TFR_INVALID_ARGUMENT;
    };
    if (format == TFR_FORMAT_ELWC) {
      // ExampleListWithContext { repeated Example examples = 1; Example context = 2; }
      while (!rec.done()) {
        uint32_t f, w;
        Span pl{nullptr, nullptr};
        uint64_t sc;
        if (!read_field(rec, &f, &w, &pl, &sc)) return bad_record();
        if (w != 2) continue;
        if (f == 1) {                 // one example of the list; extra ones are truncated
          if (count < list_size && has_ex) {
            const int rc = parse_example(pl, example_row(count));
            if (rc) return rc;
          }
          ++count;
        } else if (f == 2 && has_ctx) {
          const int rc = parse_example(pl, cdest);
          if (rc) return rc;
        }
      }
    } else if (format == TFR_FORMAT_EXAMPLE_IN_EXAMPLE) {
      // an outer Example whose bytes features `serialized_context` [1] and
      // `serialized_examples` [n] hold serialized Examples (data.py:136-150)
      while (!rec.done()) {
        uint32_t f, w;
        Span features{nullptr, nullptr};
        uint64_t sc;
        if (!read_field(rec, &f, &w, &features, &sc)) return bad_record();
        if (f != 1 || w != 2) continue;
        while (!features.done()) {
          Span entry{nullptr, nullptr};
          if (!read_field(features, &f, &w, &entry, &sc)) return bad_record();
          if (f != 1 || w != 2) continue;
          Span key, value;
          if (!read_entry(entry, &key, &value)) return bad_record();
          if (!key.p || !value.p) continue;
          const std::string k(reinterpret_cast<const char*>(key.p),
                              static_cast<size_t>(key.end - key.p));
          int rc = TFR_OK;
          if (k == "serialized_context") {
            rc = for_each_bytes(value, [&](Span v) {
              return has_ctx ? parse_example(v, cdest) : TFR_OK;
            });
          } else if (k == "serialized_examples") {
            rc = for_each_bytes(value, [&](Span v) {
              int r = TFR_OK;
              if (count < list_size && has_ex) r = parse_example(v, example_row(count));
              ++count;
              return r;
            });
          }
          if (rc) return rc;
        }
      }
    } else {
      // SequenceExample { Features context = 1; FeatureLists feature_lists = 2; }
      // FeatureLists { map<string, FeatureList> = 1 }, FeatureList { repeated Feature = 1 }:
      // frame i of a feature list is item i (data.py:572-711)
      while (!rec.done()) {
        uint32_t f, w;
        Span pl{nullptr, nullptr};
        uint64_t sc;
        if (!read_field(rec, &f, &w, &pl, &sc)) return bad_record();
        if (w != 2) continue;
        if (f == 1 && has_ctx) {
          const int rc = parse_features(pl, cdest);
          if (rc) return rc;
        } else if (f == 2) {
          while (!pl.done()) {
            Span entry{nullptr, nullptr};
            if (!read_field(pl, &f, &w, &entry, &sc)) return bad_record();
            if (f != 1 || w != 2) continue;
            Span key, value;
            if (!read_entry(entry, &key, &value)) return bad_record();
            if (!key.p || !value.p) continue;
            const Spec* spec = find_spec(espec, key);
            const int tk = spec ? -1 : find_tok(&etoks, key);
            int frame = 0;
            while (!value.done()) {           // FeatureList.feature
              Span feat{nullptr, nullptr};
              if (!read_field(value, &f, &w, &feat, &sc)) return bad_record();
              if (f != 1 || w != 2) continue;
              if (spec && frame < list_size) {
                const int rc = parse_feature_value(feat, *spec, example_row(frame).row);
                if (rc) return rc;
              } else if (tk >= 0 && frame < list_size) {
                const Dest d = example_row(frame);
                const int rc = parse_token_value(feat, etoks[tk], d.ids(tk), d.dropped + tk);
                if (rc) return rc;
              }
              ++frame;
            }
            if ((spec || tk >= 0) && frame > count) count = frame;
          }
        }
      }
    }
    if (sizes_out) sizes_out[b] = count;      // the untruncated list length (data.py:148)
    if (mask_out)
      for (int i = 0; i < list_size; ++i)
        mask_out[static_cast<size_t>(b) * list_size + i] = i < count ? 1 : 0;
    return TFR_OK;
  };

  auto report_dropped = [&]() {
    if (!dropped_out) return;
    for (int k = 0; k < nk; ++k) {
      int64_t s = 0;
      for (int b = 0; b < B; ++b) s += dropped[static_cast<size_t>(b) * nk + k];
      dropped_out[k] = s;
    }
  };
  int threads = n_threads > 0 ? n_threads : static_cast<int>(std::thread::hardware_concurrency());
  if (threads < 1) threads = 1;
  if (threads > B) threads = B;
  if (threads <= 1) {
    for (int b = 0; b < B; ++b) {
      const int rc = parse_one(b);
      if (rc) return rc;
    }
    report_dropped();
    return TFR_OK;
  }
  // lists are handed out by an atomic counter; the first failure wins and its message
  // (thread-local in the worker) is re-raised on the calling thread
  std::atomic<int> next{0}, status{TFR_OK};
  std::vector<std::string> messages(threads);
  std::vector<std::thread> pool;
  for (int t = 0; t < threads; ++t)
    pool.emplace_back([&, t] {
      for (int b = next.fetch_add(1); b < B && status.load() == TFR_OK; b = next.fetch_add(1)) {
        const int rc = parse_one(b);
        if (rc) {
          int expected = TFR_OK;
          if (status.compare_exchange_strong(expected, rc)) messages[t] = tfr_last_error();
        }
      }
    });
  for (std::thread& th : pool) th.join();
  if (status.load() != TFR_OK) {
    for (const std::string& m : messages)
      if (!m.empty()) set_error("%s", m.c_str());
    return status.load();
  }
  report_dropped();
  return TFR_OK;
}

extern "C" int tfr_ranking_parse(int format, const uint8_t* const* records,
                                 const int64_t* record_sizes, int B, int list_size,
                                 const tfr_feature_spec* context_spec, int n_context,
                                 const tfr_feature_spec* example_spec, int n_example,
                                 float* context_out, float* example_out, int32_t* sizes_out,
                                 uint8_t* mask_out, int n_threads) {
  return parse_batch(format, records, record_sizes, B, list_size, context_spec, n_context,
                     example_spec, n_example, nullptr, 0, nullptr, 0, context_out, example_out,
                     nullptr, nullptr, nullptr, sizes_out, mask_out, n_threads);
}

extern "C" int tfr_ranking_parse_tokens(
    int format, const uint8_t* const* records, const int64_t* record_sizes, int B,
    int list_size, const tfr_feature_spec* context_spec, int n_context,
    const tfr_feature_spec* example_spec, int n_example, const tfr_token_spec* context_tokens,
    int n_context_tokens, const tfr_token_spec* example_tokens, int n_example_tokens,
    float* context_out, float* example_out, int32_t* const* context_ids_out,
    int32_t* const* example_ids_out, int64_t* dropped_out, int32_t* sizes_out,
    uint8_t* mask_out, int n_threads) {
  return parse_batch(format, records, record_sizes, B, list_size, context_spec, n_context,
                     example_spec, n_example, context_tokens, n_context_tokens, example_tokens,
                     n_example_tokens, context_out, example_out, context_ids_out,
                     example_ids_out, dropped_out, sizes_out, mask_out, n_threads);
}

extern "C" int tfr_elwc_parse(const uint8_t* const* records, const int64_t* record_sizes, int B,
                              int list_size, const tfr_feature_spec* context_spec, int n_context,
                              const tfr_feature_spec* example_spec, int n_example,
                              float* context_out, float* example_out, int32_t* sizes_out,
                              uint8_t* mask_out, int n_threads) {
  return tfr_ranking_parse(TFR_FORMAT_ELWC, records, record_sizes, B, list_size, context_spec,
                           n_context, example_spec, n_example, context_out, example_out,
                           sizes_out, mask_out, n_threads);
}
