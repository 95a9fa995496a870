// ipc_out.hpp — Arrow IPC stream assembly for the product (host side, C++17, no CUDA here).
//
// Writes what ipc.NewWriter(buf, WithSchema, WithAllocator).Write(record)+Close() emits in the
// reference's offline V2 path (reporter/parca_reporter.go:1779-1790): schema message, dictionary
// batches (inner dictionaries first), one record batch, end-of-stream marker; uncompressed.
//
// Unlike a builder-based writer this one never owns column data: every Arrow buffer is a
// BufRef that points at device memory, host memory, or "zeros", and the writer only *plans*
// where each buffer lands in the final stream. The caller then copies device buffers straight
// into the pinned output at those offsets (cudaMemcpyAsync D2H) — the record body is never
// staged or re-copied on the host.
//
// The flatbuffer metadata is built back-to-front as the format requires; the order in which
// tables are created (children, then key/values, then the type table, then the name) fixes the
// byte layout and is kept identical to the repo's test oracle so streams compare bit-exactly.
#pragma once
#include <cstdint>
#include <cstring>
#include <memory>
#include <string>
#include <utility>
#include <vector>

namespace pa {

struct BufRef {
  enum Kind : uint8_t { NONE, HOST, DEVICE, ZEROS, SLICED /* spread over the shards of a merged batch; ptr is a tag */ } kind = NONE;
  const void* ptr = nullptr;
  uint64_t len = 0;
  static BufRef none() { return BufRef{}; }
  static BufRef host(const void* p, uint64_t n) { return BufRef{HOST, p, n}; }
  static BufRef dev(const void* p, uint64_t n) { return BufRef{DEVICE, p, n}; }
  static BufRef zeros(uint64_t n) { return BufRef{ZEROS, nullptr, n}; }
};

enum class Ty : uint8_t { Int, Utf8, Utf8View, FixedBinary, TimestampNsUtc, Struct, ListView, RunEnd, DictU32, Binary, List, Bool };

// One node = one Arrow field + its array. For Ty::DictU32 the node itself carries the uint32
// indices and `dict` is the dictionary *value* node (whose type becomes the field's type).
struct Node {
  Ty ty = Ty::Int;
  std::string name;
  bool nullable = false;
  int bits = 0;
  bool is_signed = false;
  int byte_width = 0;
  std::vector<std::pair<std::string, std::string>> metadata;
  int64_t length = 0;
  int64_t null_count = 0;
  BufRef validity;            // ignored (zero-length) when null_count == 0
  std::vector<BufRef> bufs;   // type-specific data buffers, in IPC order
  std::vector<Node> kids;
  std::unique_ptr<Node> dict;
};

// Where one planned buffer lands in the output stream.
struct Placement {
  BufRef src;
  uint64_t at;  // absolute byte offset in the stream
};

class FlatBuilder {  // minimal flatbuffers encoder
 public:
  FlatBuilder() : buf_(2048), head_(2048) {}
  uint32_t size() const { return (uint32_t)(buf_.size() - head_); }
  const uint8_t* data() const { return buf_.data() + head_; }
  uint32_t str(const std::string& s) {
    align(4, s.size() + 1);
    put_zero(1);
    put_raw(s.data(), s.size());
    put<uint32_t>((uint32_t)s.size());
    return size();
  }
  uint32_t offsets(const std::vector<uint32_t>& v) {
    align(4, v.size() * 4);
    for (size_t i = v.size(); i-- > 0;) put<uint32_t>(rel(v[i]));
    put<uint32_t>((uint32_t)v.size());
    return size();
  }
  uint32_t longs(const std::vector<int64_t>& v, size_t per_elem) {
    align(4, v.size() * 8);
    align(8, v.size() * 8);
    for (size_t i = v.size(); i-- > 0;) put<int64_t>(v[i]);
    put<uint32_t>((uint32_t)(v.size() / per_elem));
    return size();
  }
  void begin(int nslots) { slot_.assign((size_t)nslots, 0u); start_ = size(); }
  template <class T>
  void field(int s, T v, T dflt) {
    if (v == dflt) return;
    align(sizeof(T), 0);
    put<T>(v);
    slot_[(size_t)s] = size();
  }
  void ref(int s, uint32_t target) {
    if (!target) return;
    align(4, 0);
    put<uint32_t>(rel(target));
    slot_[(size_t)s] = size();
  }
  uint32_t end() {
    align(4, 0);
    put<int32_t>(0);
    uint32_t table = size();
    size_t n = slot_.size();
    while (n > 0 && slot_[n - 1] == 0) n--;
    for (size_t i = n; i-- > 0;) put<uint16_t>(slot_[i] ? (uint16_t)(table - slot_[i]) : (uint16_t)0);
    put<uint16_t>((uint16_t)(table - start_));
    put<uint16_t>((uint16_t)((n + 2) * 2));
    int32_t soff = (int32_t)size() - (int32_t)table;
    memcpy(buf_.data() + buf_.size() - table, &soff, 4);
    return table;
  }
  void finish(uint32_t root) {
    align(maxalign_, 4);
    put<uint32_t>(rel(root));
  }

 private:
  std::vector<uint8_t> buf_;
  size_t head_;
  size_t maxalign_ = 1;
  std::vector<uint32_t> slot_;
  uint32_t start_ = 0;
  void room(size_t need) {
    while (head_ < need) {
      size_t old = buf_.size();
      std::vector<uint8_t> bigger(old * 2);
      memcpy(bigger.data() + old + head_, buf_.data() + head_, old - head_);
      head_ += old;
      buf_.swap(bigger);
    }
  }
  void align(size_t a, size_t upcoming) {
    if (a > maxalign_) maxalign_ = a;
    size_t pad = (~(size() + upcoming) + 1) & (a - 1);
    room(pad + upcoming + a + 8);
    put_zero(pad);
  }
  void put_zero(size_t n) { room(n); head_ -= n; memset(buf_.data() + head_, 0, n); }
  void put_raw(const void* p, size_t n) { room(n); head_ -= n; if (n) memcpy(buf_.data() + head_, p, n); }
  template <class T>
  void put(T v) { put_raw(&v, sizeof(T)); }
  uint32_t rel(uint32_t target) { align(4, 0); return size() - target + 4; }
};

// Plans a whole stream. Metadata bytes are produced immediately (they are tiny); bodies are
// described by `placements` and filled in by the caller.
class StreamPlan {
 public:
  std::vector<Placement> placements;
  uint64_t total = 0;
  // One entry per message, in stream order: its encapsulated metadata (continuation marker and padding included) sits at
  // `at`, its body at `body_at`, and its buffers are placements[p0 .. p1).
  struct Message { uint64_t at, body_at, body_len; size_t p0, p1; };
  std::vector<Message> messages;
  const std::vector<uint8_t>& message_meta(size_t i) const { return meta_[i].second; }

  // pass 1: compute the layout. `meta` receives (offset, bytes) blobs to memcpy into the output.
  void build(const std::vector<Node>& columns, const std::vector<std::pair<std::string, std::string>>& schema_md, int64_t n_rows) {
    placements.clear();
    messages.clear();
    meta_.clear();
    total = 0;
    next_dict_id_ = 0;
    {  // schema
      FlatBuilder b;
      std::vector<uint32_t> f;
      for (auto& c : columns) f.push_back(field(b, c));
      uint32_t fv = b.offsets(f);
      uint32_t md = key_values(b, schema_md);
      b.begin(4);
      b.ref(1, fv);
      b.ref(2, md);
      uint32_t schema = b.end();
      message(b, 1, schema, 0);
      emit(b, Body{});
    }
    int64_t id = 0;
    for (auto& c : columns) dictionaries(c, id);
    {
      Body body;
      for (auto& c : columns) walk(c, body);
      FlatBuilder b;
      uint32_t rb = record_batch(b, n_rows, body);
      message(b, 3, rb, (int64_t)body.size);
      emit(b, body);
    }
    static const uint32_t eos[2] = {0xFFFFFFFFu, 0u};
    meta_.push_back({total, std::vector<uint8_t>((const uint8_t*)eos, (const uint8_t*)eos + 8)});
    total += 8;
  }
  // `tail` = the LAST columns of a record. Returns, per buffer of those columns in IPC order, its source and the distance from
  // its first byte to the END of the stream (nothing but the 8-byte end-of-stream marker follows the record batch body).
  static std::vector<std::pair<BufRef, uint64_t>> tail_distances(const Node* tail, size_t n) {
    Body body;
    for (size_t c = 0; c < n; c++) walk(tail[c], body);
    std::vector<std::pair<BufRef, uint64_t>> out;
    for (size_t i = 0; i < body.srcs.size(); i++) out.emplace_back(body.srcs[i], body.size - (uint64_t)body.buffers[2 * i] + 8);
    return out;
  }
  // pass 2 (host part): write metadata blobs and every padding gap's zeros; HOST/ZEROS buffers too.
  void write_host_parts(uint8_t* out) const {
    for (auto& m : meta_) memcpy(out + m.first, m.second.data(), m.second.size());
    for (auto& p : placements) {
      if (p.src.kind == BufRef::HOST && p.src.len) memcpy(out + p.at, p.src.ptr, p.src.len);
      if (p.src.kind == BufRef::ZEROS && p.src.len) memset(out + p.at, 0, p.src.len);
      uint64_t pad = ((p.src.len + 7) & ~7ull) - p.src.len;
      if (pad) memset(out + p.at + p.src.len, 0, pad);
    }
  }

 private:
  struct Body {
    std::vector<int64_t> nodes, buffers, variadic;
    std::vector<BufRef> srcs;
    uint64_t size = 0;
  };
  std::vector<std::pair<uint64_t, std::vector<uint8_t>>> meta_;
  int64_t next_dict_id_ = 0;

  static uint32_t key_values(FlatBuilder& b, const std::vector<std::pair<std::string, std::string>>& md) {
    if (md.empty()) return 0;
    std::vector<uint32_t> v;
    for (auto& e : md) {
      uint32_t k = b.str(e.first), val = b.str(e.second);
      b.begin(2);
      b.ref(0, k);
      b.ref(1, val);
      v.push_back(b.end());
    }
    return b.offsets(v);
  }
  static void type_of(FlatBuilder& b, const Node& n, uint8_t* tag, uint32_t* tab) {
    switch (n.ty) {
      case Ty::Int: b.begin(2); b.field<int32_t>(0, n.bits, 0); b.field<uint8_t>(1, n.is_signed ? 1 : 0, 0); *tab = b.end(); *tag = 2; break;
      case Ty::Utf8: b.begin(0); *tab = b.end(); *tag = 5; break;
      case Ty::Binary: b.begin(0); *tab = b.end(); *tag = 4; break;
      case Ty::Utf8View: b.begin(0); *tab = b.end(); *tag = 24; break;
      case Ty::FixedBinary: b.begin(1); b.field<int32_t>(0, n.byte_width, 0); *tab = b.end(); *tag = 15; break;
      case Ty::TimestampNsUtc: { uint32_t tz = b.str("UTC"); b.begin(2); b.field<int16_t>(0, 3, 0); b.ref(1, tz); *tab = b.end(); *tag = 10; break; }
      case Ty::Struct: b.begin(0); *tab = b.end(); *tag = 13; break;
      case Ty::ListView: b.begin(0); *tab = b.end(); *tag = 25; break;
      case Ty::List: b.begin(0); *tab = b.end(); *tag = 12; break;
      case Ty::Bool: b.begin(0); *tab = b.end(); *tag = 6; break;
      case Ty::RunEnd: b.begin(0); *tab = b.end(); *tag = 22; break;
      case Ty::DictU32: break;
    }
  }
  uint32_t field(FlatBuilder& b, const Node& n) {
    const Node* t = &n;
    uint32_t enc = 0;
    if (n.ty == Ty::DictU32) {
      int64_t id = next_dict_id_++;
      b.begin(2); b.field<int32_t>(0, 32, 0); uint32_t idx = b.end();
      b.begin(4); b.field<int64_t>(0, id, 0); b.ref(1, idx); enc = b.end();
      t = n.dict.get();
    }
    std::vector<uint32_t> ch;
    for (auto& k : t->kids) ch.push_back(field(b, k));
    uint32_t chv = b.offsets(ch);
    uint32_t md = key_values(b, n.metadata);
    uint8_t tag = 0; uint32_t tab = 0;
    type_of(b, *t, &tag, &tab);
    uint32_t name = b.str(n.name);
    b.begin(7);
    b.ref(0, name);
    b.field<uint8_t>(1, n.nullable ? 1 : 0, 0);
    b.field<uint8_t>(2, tag, 0);
    b.ref(3, tab);
    b.ref(4, enc);
    b.ref(5, chv);
    b.ref(6, md);
    return b.end();
  }
  static void message(FlatBuilder& b, uint8_t header_type, uint32_t header, int64_t body_len) {
    b.begin(5);
    b.field<int16_t>(0, 4, 0);  // MetadataVersion V5
    b.field<uint8_t>(1, header_type, 0);
    b.ref(2, header);
    b.field<int64_t>(3, body_len, 0);
    uint32_t m = b.end();
    b.finish(m);
  }
  void emit(const FlatBuilder& b, const Body& body) {
    uint32_t n = b.size();
    uint32_t padded = ((n + 8 + 7) & ~7u) - 8;
    std::vector<uint8_t> blob(8 + padded, 0);
    uint32_t pre[2] = {0xFFFFFFFFu, padded};
    memcpy(blob.data(), pre, 8);
    memcpy(blob.data() + 8, b.data(), n);
    meta_.push_back({total, std::move(blob)});
    messages.push_back(Message{total, total + 8 + padded, body.size, placements.size(), placements.size() + body.srcs.size()});
    total += 8 + padded;
    for (size_t i = 0; i < body.srcs.size(); i++) placements.push_back(Placement{body.srcs[i], total + (uint64_t)body.buffers[2 * i]});
    total += body.size;
  }
  static void add(Body& body, const BufRef& r) {
    body.buffers.push_back((int64_t)body.size);
    body.buffers.push_back((int64_t)r.len);
    body.srcs.push_back(r);
    body.size += (r.len + 7) & ~7ull;
  }
  static void walk(const Node& n, Body& body) {
    body.nodes.push_back(n.length);
    body.nodes.push_back(n.null_count);
    if (n.ty != Ty::RunEnd) add(body, n.null_count ? n.validity : BufRef::none());
    for (auto& r : n.bufs) add(body, r);
    if (n.ty == Ty::Utf8View) body.variadic.push_back((int64_t)n.bufs.size() - 1);
    for (auto& k : n.kids) walk(k, body);
  }
  static uint32_t record_batch(FlatBuilder& b, int64_t length, const Body& body) {
    uint32_t var = body.variadic.empty() ? 0 : b.longs(body.variadic, 1);
    uint32_t bufs = b.longs(body.buffers, 2);
    uint32_t nodes = b.longs(body.nodes, 2);
    b.begin(5);
    b.field<int64_t>(0, length, 0);
    b.ref(1, nodes);
    b.ref(2, bufs);
    b.ref(4, var);
    return b.end();
  }
  void dictionaries(const Node& n, int64_t& id) {
    const Node* v = &n;
    int64_t mine = -1;
    if (n.ty == Ty::DictU32) { mine = id++; v = n.dict.get(); }
    for (auto& k : v->kids) dictionaries(k, id);
    if (mine >= 0) {
      Body body;
      walk(*n.dict, body);
      FlatBuilder b;
      uint32_t rb = record_batch(b, n.dict->length, body);
      b.begin(3);
      b.field<int64_t>(0, mine, 0);
      b.ref(1, rb);
      uint32_t db = b.end();
      message(b, 2, db, (int64_t)body.size);
      emit(b, body);
    }
  }
};

}  // namespace pa
