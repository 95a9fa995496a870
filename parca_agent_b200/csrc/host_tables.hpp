// host_tables.hpp — registration-time state of the aggregator (host side, off the hot path).
//
// Everything the reference resolves per distinct frame *per interval* inside appendLocationV2
// (reporter/parca_reporter.go:418-555) is resolved here ONCE per registered frame into plain
// integer attributes (canonical string ids, function ids), so that the per-interval GPU path
// only ranks and gathers integers. Strings are canonicalised by content (equal bytes <=> equal
// canonical id), which is what makes id equality equivalent to the reference's byte-wise
// comparisons (bytes.Equal in reporter/arrow.go:99, the arrow-go memo tables).
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../include/parcaagg.h"

namespace pa {

constexpr uint32_t kNoId = 0xFFFFFFFFu;

struct StringPool {
  std::vector<uint8_t> bytes;
  std::vector<uint64_t> off{0};                    // canonical id -> byte range [off[i], off[i+1])
  std::unordered_map<std::string, uint32_t> index; // content -> canonical id
  std::vector<uint32_t> sid2cid;                   // caller's string id -> canonical id

  StringPool() { intern("", 0); sid2cid.push_back(0); }  // id 0 == "" on both sides
  uint32_t intern(const char* p, size_t n) {
    std::string key(p, n);
    auto it = index.find(key);
    if (it != index.end()) return it->second;
    uint32_t id = (uint32_t)(off.size() - 1);
    bytes.insert(bytes.end(), (const uint8_t*)p, (const uint8_t*)p + n);
    off.push_back(bytes.size());
    index.emplace(std::move(key), id);
    return id;
  }
  uint32_t intern(const char* z) { return intern(z, strlen(z)); }
  uint32_t count() const { return (uint32_t)(off.size() - 1); }
  uint32_t len(uint32_t cid) const { return (uint32_t)(off[cid + 1] - off[cid]); }
  const uint8_t* ptr(uint32_t cid) const { return bytes.data() + off[cid]; }
};

// frames after resolution: one entry per registered libpf.Frame value
struct FrameTableHost {
  std::vector<uint64_t> addr;      // frame.AddressOrLineno (:429)
  std::vector<uint32_t> type_cid;  // location.frame_type
  std::vector<uint32_t> map_cid;   // location.mapping_file
  std::vector<uint32_t> bid_cid;   // location.mapping_build_id, kNoId = null
  std::vector<uint64_t> line;      // line.line (only meaningful when func != kNoId)
  std::vector<uint32_t> func;      // function id, kNoId = location has no line
  // functions: FunctionV2{SystemName, Filename, StartLine=0} keyed by (system_name cid, filename cid)
  std::vector<uint32_t> fn_sys_cid;   // kNoId never happens in practice ("" -> null system_name)
  std::vector<uint32_t> fn_file_cid;  // kNoId = null filename ("" in FunctionV2)
  std::unordered_map<uint64_t, uint32_t> fn_index;
  // v1 stacktrace record (buildStacktraceRecord, :1583-1735): the same frames resolved by the v1 rules
  std::vector<uint32_t> v1_map_cid;   // mapping_file
  std::vector<uint32_t> v1_bid_cid;   // mapping_build_id, kNoId = null
  std::vector<uint32_t> v1_fn_cid;    // line.function_name, kNoId = the location has no line (null lines entry)
  std::vector<uint32_t> v1_file_cid;  // line.function_filename, kNoId = null
  std::vector<uint64_t> v1_line;      // line.line (int64 bit pattern)
  std::vector<uint64_t> v1_col;       // line.column
  std::vector<uint8_t> v1_complete;   // 0 = this frame clears is_complete
  uint32_t count() const { return (uint32_t)addr.size(); }
  uint32_t n_funcs() const { return (uint32_t)fn_sys_cid.size(); }

  uint32_t function(uint32_t sys_cid, uint32_t file_cid) {  // arrow_v2.go:186-208 key
    uint64_t key = ((uint64_t)sys_cid << 32) | file_cid;
    auto it = fn_index.find(key);
    if (it != fn_index.end()) return it->second;
    uint32_t id = n_funcs();
    fn_index.emplace(key, id);
    fn_sys_cid.push_back(sys_cid == 0 ? kNoId : sys_cid);    // "" => AppendNull (:195-199)
    fn_file_cid.push_back(file_cid == 0 ? kNoId : file_cid);  // "" => AppendNull (:200-204)
    return id;
  }

  // appendLocationV2, branch by branch. `sp` maps caller string ids to canonical ids.
  bool resolve(const pa_frame_desc& f, StringPool& sp) {
    auto cid = [&sp](uint32_t sid, bool* ok) -> uint32_t {
      if (sid >= sp.sid2cid.size()) { *ok = false; return 0; }
      return sp.sid2cid[sid];
    };
    bool ok = true;
    uint32_t type = cid(f.type_name_sid, &ok), fn = cid(f.function_name_sid, &ok), file = cid(f.source_file_sid, &ok);
    uint32_t exec_file = cid(f.exec_file_name_sid, &ok), exec_bid = cid(f.exec_build_id_sid, &ok);
    uint32_t mfile = cid(f.mapping_file_name_sid, &ok), gnu = cid(f.gnu_build_id_sid, &ok);
    if (!ok) return false;
    bool exists = (f.flags & PA_FRAME_F_MAPPING_FILE) && (f.flags & PA_FRAME_F_EXEC_KNOWN);  // :456-462, :486-492
    uint32_t map = 0, bid = kNoId, func_id = kNoId;
    uint64_t line_no = 0;
    switch (f.kind) {
      case PA_FRAME_ABORT:  // :432-446
        map = sp.intern("agent-internal-error-frame");
        func_id = function(sp.intern("aborted"), 0);
        break;
      case PA_FRAME_NATIVE:  // :449-476
        if (exists) {
          map = exec_file;
          if (exec_bid != 0) {
            bid = exec_bid;
          } else {  // fid.StringNoQuotes() (:469)
            char hex[40];
            int n = snprintf(hex, sizeof hex, "%016llx%016llx", (unsigned long long)f.file_id_hi, (unsigned long long)f.file_id_lo);
            bid = sp.intern(hex, (size_t)n);
          }
        } else {
          map = sp.intern("UNKNOWN");
        }
        break;
      case PA_FRAME_KERNEL: {  // :478-514
        map = sp.intern("[kernel.kallsyms]");
        uint32_t module = exists ? exec_file : sp.intern("vmlinux");
        uint32_t sym;
        if (fn != 0) { sym = fn; line_no = f.source_line; } else sym = sp.intern("UNKNOWN");
        func_id = function(sym, module);
        break;
      }
      case PA_FRAME_OOMPROF:  // :516-520
        map = file;
        bid = fn;
        break;
      default: {  // :522-551 interpreted frames
        map = type;
        uint32_t name, path;
        if (fn != 0) { name = fn; path = file; line_no = f.source_line; } else { name = sp.intern("UNREPORTED"); path = name; }
        if (path == 0) path = sp.intern("UNKNOWN");  // "Empty path causes the backend to crash" (:540-543)
        func_id = function(name, path);
      }
    }
    {  // the v1 rules differ in the details (mapping file of interpreted frames, columns, plain function names)
      uint32_t m1 = 0, b1 = kNoId, fn1 = kNoId, file1 = kNoId;
      uint64_t ln1 = 0, col1 = 0;
      uint8_t complete = 1;
      switch (f.kind) {
        case PA_FRAME_ABORT:  // :1586-1604
          m1 = sp.intern("agent-internal-error-frame");
          fn1 = sp.intern("aborted");
          break;
        case PA_FRAME_NATIVE:  // :1606-1643
          m1 = map; b1 = bid;
          complete = exists ? 1 : 0;
          break;
        case PA_FRAME_KERNEL:  // :1644-1687
          m1 = map;
          file1 = exists ? exec_file : sp.intern("vmlinux");
          if (fn != 0) { fn1 = fn; ln1 = f.source_line; } else { fn1 = sp.intern("UNKNOWN"); complete = 0; }
          col1 = f.source_column;
          break;
        case PA_FRAME_OOMPROF:  // :1688-1694
          m1 = file; b1 = fn;
          complete = 0;
          break;
        default:  // :1695-1733
          if (fn != 0) { fn1 = fn; file1 = file; ln1 = f.source_line; } else { fn1 = sp.intern("UNREPORTED"); file1 = fn1; complete = 0; }
          if (file1 == 0) file1 = sp.intern("UNKNOWN");
          if (gnu != 0) { m1 = mfile; b1 = gnu; } else { m1 = type; }
          col1 = f.source_column;
      }
      v1_map_cid.push_back(m1); v1_bid_cid.push_back(b1); v1_fn_cid.push_back(fn1); v1_file_cid.push_back(file1);
      v1_line.push_back(ln1); v1_col.push_back(col1); v1_complete.push_back(complete);
    }
    addr.push_back(f.address_or_lineno);
    type_cid.push_back(type);
    map_cid.push_back(map);
    bid_cid.push_back(bid);
    line.push_back(line_no);
    func.push_back(func_id);
    return true;
  }
};

// per-PID cached labels (the content of the `labels` LRU, parca_reporter.go:569), append-only. Every distinct label name gets a
// lifetime ordinal, every (name, value) pair a value id in that name's dictionary, and a labelset is its run of (ordinal, value
// id) pairs in CSR form, which the device mirrors append-only. A batch's label column plan is a set of name ordinals.
struct LabelSets {
  std::vector<uint32_t> off{0};    // labelset -> its pairs [off[i], off[i + 1])
  std::vector<uint32_t> pairs;     // two words per pair: name ordinal, value id
  std::vector<uint32_t> name_cid;  // ordinal -> name canonical id
  std::vector<std::vector<uint32_t>> vals;  // ordinal -> value id -> value canonical id
  std::unordered_map<uint32_t, uint32_t> ord_of;              // name canonical id -> ordinal
  std::vector<std::unordered_map<uint32_t, uint32_t>> val_of;  // ordinal -> value canonical id -> value id
  uint32_t count() const { return (uint32_t)(off.size() - 1); }
  uint32_t n_names() const { return (uint32_t)name_cid.size(); }

  // one labelset of (name cid, value cid); a name that repeats keeps its last value
  void add(const std::vector<std::pair<uint32_t, uint32_t>>& set) {
    const size_t p0 = pairs.size();
    for (auto& kv : set) {
      auto it = ord_of.find(kv.first);
      if (it == ord_of.end()) {
        it = ord_of.emplace(kv.first, n_names()).first;
        name_cid.push_back(kv.first);
        vals.emplace_back();
        val_of.emplace_back();
      }
      const uint32_t ord = it->second;
      auto& vi = val_of[ord];
      auto jt = vi.find(kv.second);
      if (jt == vi.end()) { jt = vi.emplace(kv.second, (uint32_t)vals[ord].size()).first; vals[ord].push_back(kv.second); }
      size_t p = p0;
      while (p < pairs.size() && pairs[p] != ord) p += 2;
      if (p == pairs.size()) { pairs.push_back(ord); pairs.push_back(jt->second); }
      else pairs[p + 1] = jt->second;
    }
    off.push_back((uint32_t)(pairs.size() / 2));
  }
};

}  // namespace pa
