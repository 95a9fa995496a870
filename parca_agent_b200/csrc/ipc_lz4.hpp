// ipc_lz4.hpp — optional LZ4_FRAME body compression of a finished Arrow IPC stream (host side, C++17).
//
// The reference's network path wraps record bodies with ipc.WithLZ4() (reporter/parca_reporter.go:1851; offline mode
// writes them uncompressed, :1779-1790). Its compressor is github.com/pierrec/lz4/v4 v4.1.25 (go.mod:143), which is not
// available here, so this mode CANNOT be byte-identical to the Go output and is flagged as such: it produces a valid
// Arrow stream with BodyCompression{LZ4_FRAME, BUFFER} (every non-empty buffer = int64 uncompressed length, then one LZ4
// frame; -1 = stored raw) that decodes to exactly the same record. The LZ4 frame encoder is the system's liblz4.so.1,
// bound at run time with dlopen (no headers ship in this image); without it the call fails, nothing falls back.
//
// Input: any uncompressed stream this library wrote (schema, dictionary batches, one record batch, end marker).
// The flatbuffer metadata is re-read with a few lines of table walking and rebuilt with pa::FlatBuilder, in the same
// construction order as ipc_out.hpp (plus the `compression` field), so a stream compressed here and the oracle's stream
// compressed by the same function stay comparable. The metadata rewrite (read_batch_meta + lz4_batch_message) is shared with
// PA_IPC_LZ4_FRAME_GPU, which compresses the bodies on the device (k_lz4_* in kernels.cuh, lz4_gpu_stream in agg.cu).
#pragma once
#include <dlfcn.h>

#include <atomic>
#include <cstdint>
#include <cstring>
#include <string>
#include <thread>
#include <vector>

#include "ipc_out.hpp"

namespace pa {

struct Lz4Api {
  void* handle = nullptr;
  size_t (*bound)(size_t, const void*) = nullptr;                                   // LZ4F_compressFrameBound
  size_t (*compress)(void*, size_t, const void*, size_t, const void*) = nullptr;    // LZ4F_compressFrame (NULL prefs = defaults)
  unsigned (*is_error)(size_t) = nullptr;                                           // LZ4F_isError
  bool load(std::string* err) {
    if (handle) return true;
    handle = dlopen("liblz4.so.1", RTLD_NOW | RTLD_LOCAL);
    if (!handle) { *err = "liblz4.so.1 not found (dlopen)"; return false; }
    bound = (size_t(*)(size_t, const void*))dlsym(handle, "LZ4F_compressFrameBound");
    compress = (size_t(*)(void*, size_t, const void*, size_t, const void*))dlsym(handle, "LZ4F_compressFrame");
    is_error = (unsigned (*)(size_t))dlsym(handle, "LZ4F_isError");
    if (!bound || !compress || !is_error) { *err = "liblz4.so.1 lacks the LZ4F frame API"; return false; }
    return true;
  }
};

namespace fbread {  // just enough flatbuffer reading for Message / RecordBatch / DictionaryBatch, every access bounds-checked
inline uint32_t u32(const uint8_t* p) { uint32_t v; memcpy(&v, p, 4); return v; }
inline int32_t i32(const uint8_t* p) { int32_t v; memcpy(&v, p, 4); return v; }
inline int64_t i64(const uint8_t* p) { int64_t v; memcpy(&v, p, 8); return v; }
inline uint16_t u16(const uint8_t* p) { uint16_t v; memcpy(&v, p, 2); return v; }
struct Buf {  // one metadata flatbuffer; positions are byte offsets (0 = "absent"), `bad` latches on the first out-of-range access
  const uint8_t* base;
  uint32_t len;
  bool bad = false;
  bool ok(int64_t pos, uint64_t n) {
    if (pos < 0 || (uint64_t)pos > len || (uint64_t)len - (uint64_t)pos < n) { bad = true; return false; }
    return true;
  }
  int64_t root() { if (!ok(0, 4)) return 0; int64_t t = u32(base); return ok(t, 4) && t ? t : 0; }
  int64_t field(int64_t table, int slot) {  // 0 = absent (default) or malformed (then bad is set)
    if (!table || !ok(table, 4)) return 0;
    int64_t vt = table - (int64_t)i32(base + table);
    if (!ok(vt, 4)) return 0;
    uint16_t vts = u16(base + vt);
    if (vts < 4 || !ok(vt, vts)) { bad = true; return 0; }
    if (4 + 2 * slot + 2 > (int)vts) return 0;
    uint16_t off = u16(base + vt + 4 + 2 * slot);
    if (!off) return 0;
    int64_t f = table + off;
    return ok(f, 1) ? f : 0;
  }
  int64_t indirect(int64_t p) {  // offset field -> target
    if (!p || !ok(p, 4)) return 0;
    int64_t t = p + (int64_t)u32(base + p);
    return ok(t, 4) ? t : 0;
  }
  uint8_t byte(int64_t f) { return f && ok(f, 1) ? base[f] : (uint8_t)0; }
  int64_t scalar64(int64_t f) { return f && ok(f, 8) ? i64(base + f) : 0; }
  bool longs(int64_t vec_field, int per_elem, std::vector<int64_t>* out) {  // vectors of int64 / of 16-byte structs
    out->clear();
    if (!vec_field) return !bad;
    int64_t v = indirect(vec_field);
    if (!v) return false;
    uint64_t n = u32(base + v), bytes = n * (uint64_t)per_elem * 8;
    if (!ok(v + 4, bytes)) return false;
    out->resize((size_t)(n * per_elem));
    if (bytes) memcpy(out->data(), base + v + 4, (size_t)bytes);
    return true;
  }
};
}  // namespace fbread

// Metadata of one record batch (type 3) or dictionary batch (type 2) message.
struct BatchMeta {
  uint8_t type = 0;
  int64_t length = 0, dict_id = 0;
  std::vector<int64_t> nodes, buffers, variadic;  // buffers: (offset, length) pairs of the uncompressed body
};

// Reads the Message flatbuffer `meta` of a record or dictionary batch. False (and *err) on malformed or compressed metadata.
inline bool read_batch_meta(const uint8_t* meta, uint32_t meta_len, BatchMeta* p, std::string* err) {
  fbread::Buf fb{meta, meta_len};
  int64_t m = fb.root();
  p->type = fb.byte(fb.field(m, 1));
  int64_t rb = fb.indirect(fb.field(m, 2));
  if (!m || fb.bad || !rb || (p->type != 2 && p->type != 3)) { *err = "message without header"; return false; }
  if (p->type == 2) {  // DictionaryBatch{id, data}
    p->dict_id = fb.scalar64(fb.field(rb, 0));
    rb = fb.indirect(fb.field(rb, 1));
    if (!rb) { *err = "dictionary batch without data"; return false; }
  }
  p->length = fb.scalar64(fb.field(rb, 0));
  bool vec_ok = fb.longs(fb.field(rb, 1), 2, &p->nodes) && fb.longs(fb.field(rb, 2), 2, &p->buffers) && fb.longs(fb.field(rb, 4), 1, &p->variadic);
  if (!vec_ok || fb.bad) { *err = "malformed record batch metadata"; return false; }
  if (fb.field(rb, 3)) { *err = "stream is already compressed"; return false; }
  return true;
}

// The encapsulated metadata (continuation marker, length, flatbuffer, zero padding to 8 bytes) of `p` with
// BodyCompression{LZ4_FRAME, BUFFER}, whose buffers hold sizes[b] bytes each (0 = empty), back to back at 8-byte aligned
// offsets. *offs receives each buffer's offset in the new body and *body_len the body's length.
inline std::vector<uint8_t> lz4_batch_message(const BatchMeta& p, const std::vector<int64_t>& sizes, std::vector<int64_t>* offs, int64_t* body_len) {
  std::vector<int64_t> nb(p.buffers.size());
  offs->assign(sizes.size(), 0);
  int64_t at = 0;
  for (size_t b = 0; b < sizes.size(); b++) {
    (*offs)[b] = nb[2 * b] = at;
    nb[2 * b + 1] = sizes[b];
    at = (at + sizes[b] + 7) & ~(int64_t)7;
  }
  *body_len = at;
  FlatBuilder fb;
  uint32_t var = p.variadic.empty() ? 0 : fb.longs(p.variadic, 1);
  fb.begin(2);                      // BodyCompression{codec = LZ4_FRAME (0), method = BUFFER (0)}: all defaults
  uint32_t comp = fb.end();
  uint32_t bufs = fb.longs(nb, 2);
  uint32_t nodes = fb.longs(p.nodes, 2);
  fb.begin(5);
  fb.field<int64_t>(0, p.length, 0);
  fb.ref(1, nodes);
  fb.ref(2, bufs);
  fb.ref(3, comp);
  fb.ref(4, var);
  uint32_t rb = fb.end();
  uint32_t header = rb;
  if (p.type == 2) {
    fb.begin(3);
    fb.field<int64_t>(0, p.dict_id, 0);
    fb.ref(1, rb);
    header = fb.end();
  }
  fb.begin(5);
  fb.field<int16_t>(0, 4, 0);  // MetadataVersion V5
  fb.field<uint8_t>(1, p.type, 0);
  fb.ref(2, header);
  fb.field<int64_t>(3, at, 0);
  uint32_t m = fb.end();
  fb.finish(m);
  uint32_t n = fb.size(), padded = ((n + 8 + 7) & ~7u) - 8;
  std::vector<uint8_t> out(8 + (size_t)padded, 0);
  uint32_t pre[2] = {0xFFFFFFFFu, padded};
  memcpy(out.data(), pre, 8);
  memcpy(out.data() + 8, fb.data(), n);
  return out;
}

// Re-encodes `in` with LZ4_FRAME body compression into `out`. Returns false and sets *err on malformed input / missing liblz4.
inline bool ipc_compress_lz4(const uint8_t* in, uint64_t len, std::vector<uint8_t>& out, std::string* err, unsigned threads = 0) {
  static Lz4Api api;
  if (!api.load(err)) return false;
  struct Msg { uint8_t type; const uint8_t* meta; uint32_t meta_len; const uint8_t* body; int64_t body_len; };
  std::vector<Msg> msgs;
  uint64_t pos = 0;
  bool eos = false;
  while (pos + 8 <= len) {
    uint32_t cont = fbread::u32(in + pos), mlen = fbread::u32(in + pos + 4);
    if (cont != 0xFFFFFFFFu) { *err = "not an encapsulated IPC message"; return false; }
    pos += 8;
    if (mlen == 0) { eos = true; break; }
    if (pos + mlen > len) { *err = "truncated metadata"; return false; }
    const uint8_t* meta = in + pos;
    fbread::Buf fb{meta, mlen};
    int64_t m = fb.root();
    uint8_t type = fb.byte(fb.field(m, 1));
    int64_t body_len = fb.scalar64(fb.field(m, 3));
    if (!m || fb.bad || body_len < 0) { *err = "malformed message metadata"; return false; }
    Msg x{type, meta, mlen, in + pos + mlen, body_len};
    if (pos + mlen + (uint64_t)x.body_len > len) { *err = "truncated body"; return false; }
    msgs.push_back(x);
    pos += mlen + (uint64_t)x.body_len;
  }
  if (!eos) { *err = "missing end-of-stream marker"; return false; }

  // one task per non-empty buffer
  struct Task { const uint8_t* src; int64_t n; std::vector<uint8_t> dst; };
  struct Plan { BatchMeta meta; std::vector<int> task_of_buffer; };
  std::vector<Task> tasks;
  std::vector<Plan> plans(msgs.size());
  for (size_t i = 0; i < msgs.size(); i++) {
    if (msgs[i].type != 2 && msgs[i].type != 3) continue;
    Plan& p = plans[i];
    if (!read_batch_meta(msgs[i].meta, msgs[i].meta_len, &p.meta, err)) return false;
    for (size_t b = 0; b + 1 < p.meta.buffers.size(); b += 2) {
      int64_t off = p.meta.buffers[b], n = p.meta.buffers[b + 1];
      if (off < 0 || n < 0 || off > msgs[i].body_len || n > msgs[i].body_len - off) { *err = "buffer outside its body"; return false; }
      if (n == 0) { p.task_of_buffer.push_back(-1); continue; }
      p.task_of_buffer.push_back((int)tasks.size());
      tasks.push_back(Task{msgs[i].body + off, n, {}});
    }
  }
  std::atomic<size_t> next{0};
  std::atomic<bool> failed{false};
  auto work = [&] {
    for (size_t t; (t = next.fetch_add(1)) < tasks.size();) {
      Task& k = tasks[t];
      size_t cap = api.bound((size_t)k.n, nullptr);
      k.dst.resize(8 + cap);
      size_t w = api.compress(k.dst.data() + 8, cap, k.src, (size_t)k.n, nullptr);
      if (api.is_error(w)) { failed = true; continue; }
      int64_t prefix = k.n;
      if (w >= (size_t)k.n) { prefix = -1; w = (size_t)k.n; memcpy(k.dst.data() + 8, k.src, w); }  // incompressible: stored raw
      memcpy(k.dst.data(), &prefix, 8);
      k.dst.resize(8 + w);
    }
  };
  if (!threads) threads = std::min<unsigned>(std::max(1u, std::thread::hardware_concurrency()), 32u);
  threads = (unsigned)std::min<size_t>(threads, std::max<size_t>(tasks.size(), 1));
  std::vector<std::thread> pool;
  for (unsigned t = 1; t < threads; t++) pool.emplace_back(work);
  work();
  for (auto& th : pool) th.join();
  if (failed) { *err = "LZ4F_compressFrame failed"; return false; }

  out.clear();
  auto append = [&out](const void* p, size_t n) { const uint8_t* q = (const uint8_t*)p; out.insert(out.end(), q, q + n); };
  for (size_t i = 0; i < msgs.size(); i++) {
    if (msgs[i].type != 2 && msgs[i].type != 3) {  // schema: verbatim
      uint32_t pre[2] = {0xFFFFFFFFu, msgs[i].meta_len};
      append(pre, 8);
      append(msgs[i].meta, msgs[i].meta_len);
      continue;
    }
    Plan& p = plans[i];
    std::vector<int64_t> sizes(p.task_of_buffer.size()), offs;
    for (size_t b = 0; b < sizes.size(); b++) sizes[b] = p.task_of_buffer[b] < 0 ? 0 : (int64_t)tasks[p.task_of_buffer[b]].dst.size();
    int64_t body_len = 0;
    std::vector<uint8_t> meta = lz4_batch_message(p.meta, sizes, &offs, &body_len);
    append(meta.data(), meta.size());
    size_t body = out.size();
    out.resize(body + (size_t)body_len, 0);
    for (size_t b = 0; b < sizes.size(); b++)
      if (sizes[b]) memcpy(out.data() + body + offs[b], tasks[p.task_of_buffer[b]].dst.data(), (size_t)sizes[b]);
  }
  uint32_t eos_mark[2] = {0xFFFFFFFFu, 0u};
  append(eos_mark, 8);
  return true;
}

}  // namespace pa
