// reporter.cpp — see reporter.hpp. Host glue only: interning + the Origin switch; no aggregation.
#include "reporter.hpp"

#include <algorithm>
#include <chrono>
#include <cstring>
#include <random>

namespace parca {

// ---- production sink: straight onto the C ABI -------------------------------------------------
namespace {
struct AggSink final : Sink {
  pa_agg* a;
  uint32_t hash_mode;
  AggSink(pa_agg* agg, uint32_t mode) : a(agg), hash_mode(mode) {}
  uint32_t RegisterString(const std::string& s) override {
    uint32_t off[2] = {0, (uint32_t)s.size()}, id = PA_NO_STRING;
    if (pa_agg_register_strings(a, (const uint8_t*)s.data(), off, 1, &id) != PA_OK) return PA_NO_STRING;
    return id;
  }
  uint64_t RegisterFrame(const pa_frame_desc& d) override {
    uint64_t id = ~0ull;
    if (pa_agg_register_frames(a, &d, 1, &id) != PA_OK) return ~0ull;
    return id;
  }
  uint32_t RegisterLabelset(const std::vector<pa_label_pair>& pairs) override {
    uint32_t off[2] = {0, (uint32_t)pairs.size()}, id = PA_NO_STRING;
    if (pa_agg_register_labelsets(a, pairs.data(), off, 1, &id) != PA_OK) return PA_NO_STRING;
    return id;
  }
  // rows are handed to the ring kBatch at a time: one lock round-trip and one call across the ABI per batch instead of
  // per sample (what a cgo shim must do too: a cgo call costs ~100 ns). Callers are serialised by the reporter's mutex.
  static constexpr size_t kBatch = 256;
  std::vector<pa_sample_hdr> pend_h;
  std::vector<uint64_t> pend_f;
  int push() {
    if (pend_h.empty()) return PA_OK;
    int rc = pa_agg_submit(a, pend_h.data(), pend_f.data(), pend_h.size());
    pend_h.clear();
    pend_f.clear();
    return rc;
  }
  uint64_t RegisterStack(const TraceHash& h, const uint64_t* ids, uint32_t n) override {
    const uint64_t hash[2] = {h.hi, h.lo}, off[2] = {0, n};
    uint64_t id = ~0ull;
    // (the handle: the consecutive id on a plain registered aggregator, generation << 32 | slot with PA_CFG_RETIRE_STACKS)
    if (pa_agg_register_stack_handles(a, hash_mode == PA_HASH_PROVIDED ? hash : nullptr, ids, off, 1, &id) != PA_OK) return ~0ull;
    return id;
  }
  int RetireStacks(uint32_t idle, std::vector<uint64_t>* handles) override {
    std::vector<uint64_t> buf(1u << 16);
    for (;;) {  // a call retires at most buf.size() stacks; the next one finds the rest
      uint64_t n = 0;
      int rc = pa_agg_retire_stacks(a, idle, buf.data(), buf.size(), &n);
      if (rc != PA_OK) return rc;
      handles->insert(handles->end(), buf.begin(), buf.begin() + n);
      if (n < buf.size()) return PA_OK;
    }
  }
  int Submit(const pa_sample_hdr& hdr, const uint64_t* frame_ids) override {
    pend_h.push_back(hdr);
    if (frame_ids) pend_f.insert(pend_f.end(), frame_ids, frame_ids + hdr.nframes);  // (registered stacks: the row names its stack)
    return pend_h.size() >= kBatch ? push() : PA_OK;
  }
  int Publish() override { return push(); }
  int Flush(pa_agg_result* out) override { return pa_agg_flush(a, out); }
  void Release(pa_agg_result* res) override { pa_agg_release(a, res); }
  int LastStackIds(uint8_t* out, uint64_t n) override { return pa_agg_last_stack_ids(a, out, n); }
  int Stacktraces(const uint8_t* ids, uint64_t n, pa_agg_result* out) override { return pa_agg_stacktraces(a, ids, n, out); }
};
}  // namespace
Sink* NewAggSink(pa_agg* agg, uint32_t hash_mode) { return new AggSink(agg, hash_mode); }

// ---- maybeFixTruncation (reporter/parca_reporter.go:190-216) -------------------------------------
bool MaybeFixTruncation(std::string* s, size_t maxLen) {
  int64_t n = pa_fix_truncation((const uint8_t*)s->data(), s->size(), maxLen);
  if (n < 0) { s->clear(); return false; }
  s->resize((size_t)n);
  return true;
}
static bool validUtf8(const std::string& s) { return pa_fix_truncation((const uint8_t*)s.data(), s.size(), (uint64_t)-1) == (int64_t)s.size(); }

// ---- offline log framing ---------------------------------------------------------------------
void OfflineLog::header(uint16_t version) {
  const uint8_t h[8] = {0xA6, 0xE7, 0xCC, 0xCA, (uint8_t)(version >> 8), (uint8_t)version, 0, 0};  // setupOfflineModeLog :1109-1113
  buf_.assign(h, h + 8);
}
void OfflineLog::Append(const uint8_t* ipc, uint64_t len) {
  uint32_t sz = (uint32_t)len;  // binary.Write(BigEndian, uint32(buf.Len())) :1807-1810
  const uint8_t be[4] = {(uint8_t)(sz >> 24), (uint8_t)(sz >> 16), (uint8_t)(sz >> 8), (uint8_t)sz};
  buf_.insert(buf_.end(), be, be + 4);
  buf_.insert(buf_.end(), ipc, ipc + len);
  n_++;
  buf_[6] = (uint8_t)(n_ / 256);  // WriteAt([]byte{byte(n/256), byte(n)}, 6) :1829
  buf_[7] = (uint8_t)n_;
}

// ---- reporter -----------------------------------------------------------------------------------
ParcaReporter::ParcaReporter(Sink* sink, Config cfg) : sink_(sink), cfg_(std::move(cfg)) { strings_.emplace("", 0u); }
ParcaReporter::~ParcaReporter() { Stop(); }

uint32_t ParcaReporter::sid(const std::string& s) {
  auto it = strings_.find(s);
  if (it != strings_.end()) return it->second;
  uint32_t id = sink_->RegisterString(s);
  if (id != PA_NO_STRING) strings_.emplace(s, id);  // a failed registration is retried next time
  return id;
}

bool ParcaReporter::ExecutableKnown(FileID id) {
  std::lock_guard<std::mutex> g(mu_);
  return executables_.count(id) != 0;
}

void ParcaReporter::ReportExecutable(const ExecutableMetadata& md) {
  std::lock_guard<std::mutex> g(mu_);
  if (executables_.count(md.ID)) return;  // :673-675
  executables_.emplace(md.ID, md);
  // Frames interned while this executable was unknown resolved to "UNKNOWN"; the reference looks the
  // executable up again every interval (:460), so forget those ids: their next sighting re-interns
  // the same Frame value with the executable attached.
  auto it = unknown_by_file_.find(md.ID);
  if (it != unknown_by_file_.end()) {
    for (auto& key : it->second) frames_.erase(key);
    unknown_by_file_.erase(it);
    trace_cache_.clear();  // cached id lists may contain the forgotten ids
    trace_ids_.clear();
    stack_cache_.clear();  // and so may registered stacks: their next sighting registers them again
    zero_hash_stacks_.clear();
    hash_of_stack_.clear();  // (the old copies go idle and are retired; their handles are no longer in the caches)
    zero_key_of_stack_.clear();
  }
}

// Frame value -> dense frame id. The key is the whole Frame (as libpf.Frame is the map key at :421).
uint64_t ParcaReporter::frameId(const Frame& f) {
  if (f.Handle) {  // interned handle: value identity is pointer identity
    auto h = frames_by_handle_.find(f.Handle);
    if (h != frames_by_handle_.end()) return h->second;
  }
  std::string key;
  key.reserve(64 + f.FunctionName.size() + f.SourceFile.size());
  auto put = [&key](const void* p, size_t n) { key.append((const char*)p, n); };
  put(&f.Type.kind, 1); key += f.Type.name; key.push_back('\0');
  key += f.FunctionName; key.push_back('\0'); key += f.SourceFile; key.push_back('\0');
  put(&f.SourceLine, 4); put(&f.SourceColumn, 4); put(&f.AddressOrLineno, 8);
  key += f.MappingFileName; key.push_back('\0'); key += f.MappingGnuBuildID; key.push_back('\0');
  uint8_t mv = (uint8_t)((f.MappingValid ? 1 : 0) | (f.MappingHasFile ? 2 : 0));
  put(&mv, 1); put(&f.MappingFileID, sizeof(FileID));
  auto it = frames_.find(key);
  if (it != frames_.end()) { if (f.Handle) frames_by_handle_.emplace(f.Handle, it->second); return it->second; }

  pa_frame_desc d;
  memset(&d, 0, sizeof d);
  d.kind = f.Type.kind;
  d.type_name_sid = sid(f.Type.name);
  d.address_or_lineno = f.AddressOrLineno;
  d.function_name_sid = sid(f.FunctionName);
  d.source_file_sid = sid(f.SourceFile);
  d.source_line = f.SourceLine;
  d.source_column = f.SourceColumn;
  if (f.MappingValid && !f.MappingGnuBuildID.empty()) {  // :1716
    d.mapping_file_name_sid = sid(f.MappingFileName);
    d.gnu_build_id_sid = sid(f.MappingGnuBuildID);
  }
  d.file_id_hi = f.MappingFileID.hi;
  d.file_id_lo = f.MappingFileID.lo;
  const bool has_file = f.MappingValid && f.MappingHasFile;  // :456-462
  if (has_file) {
    d.flags |= PA_FRAME_F_MAPPING_FILE;
    auto e = executables_.find(f.MappingFileID);
    if (e != executables_.end()) {
      d.flags |= PA_FRAME_F_EXEC_KNOWN;
      d.exec_file_name_sid = sid(e->second.FileName);
      d.exec_build_id_sid = sid(e->second.GnuBuildID);
    } else if (f.Type.kind == PA_FRAME_NATIVE || f.Type.kind == PA_FRAME_KERNEL) {
      unknown_by_file_[f.MappingFileID].push_back(key);
    }
  }
  uint64_t id = sink_->RegisterFrame(d);
  frames_.emplace(std::move(key), id);
  if (f.Handle && !(has_file && !(d.flags & PA_FRAME_F_EXEC_KNOWN))) frames_by_handle_.emplace(f.Handle, id);  // frames of a still-unknown executable keep going through the value path (they are re-resolved once it is reported)
  return id;
}

uint32_t ParcaReporter::labelsetId(const Labels& l) {
  std::string key;
  for (auto& kv : l) { key += kv.first; key.push_back('\0'); key += kv.second; key.push_back('\1'); }
  auto it = labelsets_.find(key);
  if (it != labelsets_.end()) return it->second;
  std::vector<pa_label_pair> pairs;
  for (auto& kv : l) pairs.push_back(pa_label_pair{sid(kv.first), sid(kv.second)});
  uint32_t id = sink_->RegisterLabelset(pairs);
  labelsets_.emplace(std::move(key), id);
  return id;
}

// labelsForTID's per-PID half (:569-604): node label + provider labels, meta labels dropped, cached per PID.
// The per-sample cpu / thread_id / thread_name patch (:616-625) is applied on the GPU from the
// sample header (pa_agg_config.label_flags), so nothing is allocated per sample here.
bool ParcaReporter::labelsForPID(uint32_t pid, PidLabels** out) {
  auto it = labels_.find(pid);
  if (it == labels_.end()) {
    PidLabels pl;
    std::map<std::string, std::string> lb;  // labels.Builder: Set(name, "") deletes
    lb["node"] = cfg_.nodeName;
    if (cfg_.labelsForPID) {
      Labels extra;
      pl.keep = cfg_.labelsForPID(pid, &extra);
      for (auto& kv : extra) { if (kv.second.empty()) lb.erase(kv.first); else lb[kv.first] = kv.second; }
    }
    for (auto i = lb.begin(); i != lb.end();) {  // model.MetaLabelPrefix (:589-593)
      if (i->first.rfind("__meta_", 0) == 0 || i->second.empty()) i = lb.erase(i); else ++i;
    }
    pl.base.assign(lb.begin(), lb.end());
    pl.labelset = labelsetId(pl.base);
    it = labels_.emplace(pid, std::move(pl)).first;
  }
  *out = &it->second;
  return it->second.keep;
}

int ParcaReporter::writeSampleV2(const Trace* trace, const TraceEventMeta* meta, uint32_t labelset, uint8_t kind, int64_t value,
                                 const uint64_t* ids, size_t nids) {
  pa_sample_hdr h;
  memset(&h, 0, sizeof h);
  h.hash_hi = trace->Hash.hi;
  h.hash_lo = trace->Hash.lo;
  h.timestamp_ns = meta->Timestamp;
  h.value = value;
  h.pid = meta->PID;
  h.tid = meta->TID;
  if (!last_comm_valid_ || meta->Comm != last_comm_) {
    last_comm_sid_ = sid(meta->Comm);
    last_comm_ = meta->Comm;
    last_comm_valid_ = last_comm_sid_ != PA_NO_STRING;
  }
  h.comm_sid = last_comm_sid_;
  h.labelset_id = labelset;
  h.cpu = (uint32_t)meta->CPU;
  h.nframes = (uint16_t)nids;
  h.kind = kind;
  if (cfg_.registeredStacks) {  // `ids` is the stack id: the row carries no frame ids
    h.frame_off = *ids;
    return sink_->Submit(h, nullptr);
  }
  return sink_->Submit(h, ids);
}

uint64_t ParcaReporter::stackId(const Trace* trace) {
  const size_t nfr = trace->Frames.size();
  const bool by_hash = (trace->Hash.hi | trace->Hash.lo) != 0;  // oomprof traces share the zero hash with different frames
  if (by_hash) {
    const TraceSlot* tc = stack_cache_.find(trace->Hash);
    if (tc && tc->n == nfr) return tc->off;
  }
  scratch_ids_.clear();
  scratch_ids_.reserve(nfr);
  for (auto& f : trace->Frames) scratch_ids_.push_back(frameId(f));
  std::string key;
  if (!by_hash) {
    key.assign((const char*)scratch_ids_.data(), nfr * 8);
    auto it = zero_hash_stacks_.find(key);
    if (it != zero_hash_stacks_.end()) return it->second;
  }
  const uint64_t id = sink_->RegisterStack(trace->Hash, scratch_ids_.data(), (uint32_t)nfr);
  if (id == ~0ull) return id;
  const bool index = cfg_.retireIdleBatches != 0;
  if (by_hash) {
    if (stack_cache_.size() >= kTraceCacheEntries) { stack_cache_.clear(); hash_of_stack_.clear(); }
    stack_cache_.put(trace->Hash, id, (uint32_t)nfr);
    if (index) hash_of_stack_[id] = trace->Hash;
  } else {
    if (index) zero_key_of_stack_[id] = key;
    zero_hash_stacks_.emplace(std::move(key), id);
  }
  return id;
}

// Retired handles leave the caches under the ingest lock, before the next flush: a row that still names one was committed before
// this point and lands in the next batch, which resolves it exactly (the grace batch). A cache entry that has meanwhile been
// replaced by another handle for the same key stays.
int ParcaReporter::retireStacks() {
  std::vector<uint64_t> gone;
  int rc = sink_->RetireStacks(cfg_.retireIdleBatches, &gone);
  std::lock_guard<std::mutex> g(mu_);
  for (uint64_t h : gone) {
    auto k = hash_of_stack_.find(h);
    if (k != hash_of_stack_.end()) {
      const TraceSlot* s = stack_cache_.find(k->second);
      if (s && s->off == h) stack_cache_.erase(k->second);
      hash_of_stack_.erase(k);
    }
    auto z = zero_key_of_stack_.find(h);
    if (z != zero_key_of_stack_.end()) {
      auto e = zero_hash_stacks_.find(z->second);
      if (e != zero_hash_stacks_.end() && e->second == h) zero_hash_stacks_.erase(e);
      zero_key_of_stack_.erase(z);
    }
  }
  stacksRetired += gone.size();
  return rc;
}

int ParcaReporter::ReportTraceEvent(const Trace* trace, const TraceEventMeta* meta) {
  std::lock_guard<std::mutex> g(mu_);
  PidLabels* pl;
  if (!labelsForPID(meta->PID, &pl)) {  // :231-235
    skippedByRelabeling++;
    return 0;
  }
  if (trace->Frames.empty()) emptySamples++;  // :237-239 (the row is still written)
  uint32_t labelset = pl->labelset;
  if (!trace->CustomLabels.empty()) {  // :380-392: custom labels join the sample's label set
    std::map<std::string, std::string> lb(pl->base.begin(), pl->base.end());
    for (auto& kv : trace->CustomLabels) {
      if (!validUtf8(kv.first)) continue;  // "ignoring non-UTF8 label"
      std::string v = kv.second;
      if (!MaybeFixTruncation(&v, cfg_.customLabelMaxValLen - 1)) continue;  // "ignoring non-UTF8 value"
      if (v.empty()) continue;
      lb[kv.first] = v;
    }
    labelset = labelsetId(Labels(lb.begin(), lb.end()));
  }
  const size_t nfr = trace->Frames.size();
  uint64_t stack = 0;
  if (cfg_.registeredStacks) {  // every row of this trace names its registered stack (writeSampleV2 passes the id, not frames)
    if (nfr > 65535 || (stack = stackId(trace)) == ~0ull) { droppedBatches++; return 0; }
  }
  // frame ids of this trace: from the per-hash cache when the stack was seen before (one lookup), else per frame
  const uint64_t* idp = cfg_.registeredStacks ? &stack : nullptr;
  const bool cacheable = (trace->Hash.hi | trace->Hash.lo) != 0;  // oomprof traces share the zero hash with different frames
  if (cacheable && !idp) {
    const TraceSlot* tc = trace_cache_.find(trace->Hash);
    if (tc && tc->n == nfr) idp = trace_ids_.data() + tc->off;
  }
  if (!idp) {
    scratch_ids_.clear();
    scratch_ids_.reserve(nfr);
    for (auto& f : trace->Frames) scratch_ids_.push_back(frameId(f));
    if (cacheable) {
      if (trace_cache_.size() >= kTraceCacheEntries) { trace_cache_.clear(); trace_ids_.clear(); }
      trace_cache_.put(trace->Hash, (uint64_t)trace_ids_.size(), (uint32_t)nfr);
      trace_ids_.insert(trace_ids_.end(), scratch_ids_.begin(), scratch_ids_.end());
    }
    idp = scratch_ids_.data();
  }
  if (nfr > 65535) { droppedBatches++; return 0; }  // the row format carries a 16-bit depth; such a trace cannot come out of the unwinder
  const uint64_t* ids = idp;  // (registered stacks: the stack id)

  int rc = 0;
  switch (meta->Origin) {  // reportTraceEventV2 :338-363
    case TraceOriginSampling: rc = writeSampleV2(trace, meta, labelset, PA_KIND_CPU, 1, ids, nfr); cpuSamples++; break;
    case TraceOriginOffCPU: rc = writeSampleV2(trace, meta, labelset, PA_KIND_OFFCPU, meta->OffTime, ids, nfr); offcpuSamples++; break;
    case TraceOriginCuda: rc = writeSampleV2(trace, meta, labelset, PA_KIND_CUDA, meta->OffTime, ids, nfr); gpuSamples++; break;
    case TraceOriginMemory: {
      const MemorySample* m = meta->OriginData;
      if (!m) break;  // "memory trace event missing OriginData" :345-348
      if (m->Allocs != m->Frees) rc |= writeSampleV2(trace, meta, labelset, PA_KIND_MEM_INUSE_OBJECTS, (int64_t)(m->Allocs - m->Frees), ids, nfr);
      if (m->AllocBytes != m->FreeBytes) rc |= writeSampleV2(trace, meta, labelset, PA_KIND_MEM_INUSE_SPACE, (int64_t)(m->AllocBytes - m->FreeBytes), ids, nfr);
      if (cfg_.reportAllocs) {
        rc |= writeSampleV2(trace, meta, labelset, PA_KIND_MEM_ALLOC_OBJECTS, (int64_t)m->Allocs, ids, nfr);
        rc |= writeSampleV2(trace, meta, labelset, PA_KIND_MEM_ALLOC_SPACE, (int64_t)m->AllocBytes, ids, nfr);
      }
      memorySamples++;
      break;
    }
  }
  if (rc == PA_ENOSPC) droppedBatches++;  // ring full: the sample is dropped, like a failed interval drops its data (:1218-1220)
  return 0;                                // the reference returns nil in every V2 branch (:365)
}

int ParcaReporter::SampleEvents(const std::vector<MemorySample>& samples, const OomprofSampleMeta& meta) {
  TraceEventMeta m;
  m.Timestamp = meta.Timestamp;
  m.Comm = meta.Comm;
  m.Origin = TraceOriginMemory;
  m.PID = meta.PID;
  m.TID = meta.PID;  // "For oomprof, TID is same as PID" (:725)
  for (const MemorySample& sample : samples) {
    Trace t;  // Hash is never set on this path: all oomprof traces share the zero id, as in the reference
    for (uint64_t addr : sample.Addresses) {
      Frame f;
      f.Type = FrameType{PA_FRAME_OOMPROF, "native"};  // appendLocationV2 reports libpf.NativeFrame.String() for these (:518)
      f.AddressOrLineno = addr;
      f.FunctionName = meta.BuildID;
      f.SourceFile = meta.ExecutablePath;
      t.Frames.push_back(std::move(f));
    }
    t.CustomLabels = meta.CustomLabels;
    m.OriginData = &sample;
    int rc = ReportTraceEvent(&t, &m);
    if (rc) return rc;  // "failed to report oomprof trace event" (:753)
  }
  return 0;
}

int64_t ParcaReporter::FlushOnce() {
  pa_agg_result res;
  int rc;
  {
    // rows still buffered on the host side join this interval under the ingest lock; the ring swap itself is the
    // aggregator's (buildSampleRecordV2 holds sampleWriterV2Mu only for its writer swap, :1745-1748)
    std::lock_guard<std::mutex> g(mu_);
    rc = sink_->Publish();
  }
  if (rc == PA_ENOSPC) droppedBatches++;  // ring full: those rows are lost, the interval still goes out
  rc = sink_->Flush(&res);
  if (rc != PA_OK) { droppedBatches++; return rc; }  // flush error: logged, interval dropped (:1218-1220)
  int64_t rows = (int64_t)res.n_rows;
  if (res.n_rows) {  // empty intervals are skipped (:1842-1845)
    if (cfg_.onBatch) cfg_.onBatch(res.ipc, res.ipc_len, res.n_rows);
    sampleWrites += res.n_rows;               // :1869
    sampleWriteRequestBytes += res.ipc_len;   // :1870
  }
  const uint64_t n_unique = res.n_unique_stacks;
  sink_->Release(&res);
  if (cfg_.registeredStacks && cfg_.retireIdleBatches) retireStacks();  // (a failed call is retried after the next flush)
  if (rows && cfg_.offlineV1Stacktraces) {
    // :1300-1349 — walk the sample record's stacktrace_id dictionary in order, keep the ids this log has not
    // seen, and write their stacktrace record right behind the sample record (even when there are none)
    std::vector<uint8_t> ids(n_unique * 16), fresh;
    if ((rc = sink_->LastStackIds(ids.data(), n_unique)) != PA_OK) { droppedBatches++; return rc; }
    {
      std::lock_guard<std::mutex> g(mu_);  // ResetLoggedStacks (log rotation) may run on another thread
      for (uint64_t i = 0; i < n_unique; i++) {
        std::string key((const char*)ids.data() + 16 * i, 16);
        bool& seen = logged_stacks_[key];
        if (seen) continue;
        seen = true;
        fresh.insert(fresh.end(), key.begin(), key.end());
      }
    }
    pa_agg_result st;
    if ((rc = sink_->Stacktraces(fresh.data(), fresh.size() / 16, &st)) != PA_OK) { droppedBatches++; return rc; }
    if (cfg_.onBatch) cfg_.onBatch(st.ipc, st.ipc_len, st.n_rows);
    stacktraceWriteRequestBytes += st.ipc_len;  // :1351
    sink_->Release(&st);
  }
  return rows;
}

void ParcaReporter::ResetLoggedStacks() {
  std::lock_guard<std::mutex> g(mu_);
  logged_stacks_.clear();
}

int ParcaReporter::Start() {
  std::lock_guard<std::mutex> g(tick_mu_);
  if (started_) return 0;
  started_ = true;
  stop_ = false;
  ticker_ = std::thread([this] {
    std::mt19937_64 rng(0x5EED);
    std::unique_lock<std::mutex> lk(tick_mu_);
    double wait = cfg_.reportIntervalSeconds;
    while (!stop_) {
      if (tick_cv_.wait_for(lk, std::chrono::duration<double>(wait), [this] { return stop_; })) break;
      lk.unlock();
      FlushOnce();
      lk.lock();
      // libpf.AddJitter(interval, 0.2) (:1222): next tick uniformly within +-20 %
      std::uniform_real_distribution<double> jitter(0.8, 1.2);
      wait = cfg_.reportIntervalSeconds * jitter(rng);
    }
  });
  return 0;
}

void ParcaReporter::Stop() {
  {
    std::lock_guard<std::mutex> g(tick_mu_);
    if (!started_) return;
    stop_ = true;
  }
  tick_cv_.notify_all();
  if (ticker_.joinable()) ticker_.join();
  std::lock_guard<std::mutex> g(tick_mu_);
  started_ = false;
}

}  // namespace parca
