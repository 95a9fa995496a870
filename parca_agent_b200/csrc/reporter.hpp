// reporter.hpp — C++ host-side mirror of the reference's reporter for the V2 sample path.
//
// The reference implements go.opentelemetry.io/ebpf-profiler/reporter.Reporter in Go
// (reporter/parca_reporter.go:56). Go is not available in this environment, so the layer a cgo
// shim would provide is written here in C++ with the same method names, argument meaning and
// error behaviour; it only *feeds* the C ABI (include/parcaagg.h) — all aggregation happens on
// the GPU behind pa_agg_*. What lives here is exactly what cannot cross a C boundary as-is:
//   * unique.Handle[libpf.Frame] -> dense frame ids (interning, equality == Frame value equality)
//   * libpf.String -> string ids
//   * the per-PID `labels` LRU (parca_reporter.go:569-604) -> labelset ids (+ custom labels, :380-392)
//   * the Origin switch expansion of memory events into up to four rows (:343-360)
//   * Start/Stop: the jittered report ticker (:1199-1225)
// Out of scope (SURVEY §2): metadata providers, relabel rules, gRPC, debuginfo upload.
#pragma once
#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <functional>
#include <map>
#include <mutex>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../../include/parcaagg.h"

namespace parca {

// ---- the slice of libpf / samples / support the path reads (un-vendored module, go.mod:39,:186) ----
struct TraceHash { uint64_t hi = 0, lo = 0; };
struct FileID { uint64_t hi = 0, lo = 0; bool operator<(const FileID& o) const { return hi != o.hi ? hi < o.hi : lo < o.lo; } };

// libpf.FrameType: only its String() and the branch appendLocationV2 takes matter to this path.
struct FrameType {
  uint8_t kind = PA_FRAME_NATIVE;  // PA_FRAME_*
  std::string name = "native";     // FrameType.String()
  bool IsAbort() const { return kind == PA_FRAME_ABORT; }
  const std::string& String() const { return name; }
};
struct Frame {  // libpf.Frame — the dedup key of appendLocationV2 (parca_reporter.go:421)
  FrameType Type;
  std::string FunctionName, SourceFile;
  uint32_t SourceLine = 0, SourceColumn = 0;
  uint64_t AddressOrLineno = 0;
  bool MappingValid = false;     // frame.Mapping.Valid()
  bool MappingHasFile = false;   // m.File != (libpf.FrameMappingFile{})
  FileID MappingFileID;          // mf.FileID
  std::string MappingFileName, MappingGnuBuildID;  // mf.FileName / mf.GnuBuildID (v1 stacktrace record, :1716-1719)
  // unique.Handle[libpf.Frame] (what libpf.Frames iterates, arrow_v2.go:305-306): handle equality == Frame value equality,
  // so a non-zero Handle is the whole interning key (one 8-byte hash lookup per frame instead of serialising the value).
  uint64_t Handle = 0;
};
struct Trace {  // libpf.Trace
  TraceHash Hash;
  std::vector<Frame> Frames;
  std::map<std::string, std::string> CustomLabels;
};
enum TraceOrigin { TraceOriginSampling = 0, TraceOriginOffCPU = 1, TraceOriginMemory = 2, TraceOriginCuda = 3 };
struct MemorySample {  // oomprof.Sample
  uint64_t Allocs = 0, Frees = 0, AllocBytes = 0, FreeBytes = 0;
  std::vector<uint64_t> Addresses;  // the allocation site's stack, read by SampleEvents (:728-735)
};
struct OomprofSampleMeta {  // oomprof.SampleMeta as read at :718-745
  int64_t Timestamp = 0;
  std::string Comm, ProcessName, ExecutablePath, BuildID;
  uint32_t PID = 0;
  std::map<std::string, std::string> CustomLabels;
};
struct TraceEventMeta {  // samples.TraceEventMeta
  int64_t Timestamp = 0;
  std::string Comm;
  uint32_t PID = 0, TID = 0;
  int CPU = 0;
  TraceOrigin Origin = TraceOriginSampling;
  int64_t OffTime = 0;
  const MemorySample* OriginData = nullptr;
};
struct ExecutableMetadata { FileID ID; std::string FileName, GnuBuildID; };  // reporter.ExecutableMetadata (:650-693)

using Labels = std::vector<std::pair<std::string, std::string>>;  // labels.Labels: sorted by name, no empty values

// The aggregator as seen from the host layer; the production implementation forwards to pa_agg_*.
struct Sink {
  virtual ~Sink() = default;
  virtual uint32_t RegisterString(const std::string& s) = 0;
  virtual uint64_t RegisterFrame(const pa_frame_desc& d) = 0;
  virtual uint32_t RegisterLabelset(const std::vector<pa_label_pair>& pairs) = 0;
  virtual int Submit(const pa_sample_hdr& hdr, const uint64_t* frame_ids) = 0;  // may buffer rows until Publish
  // Config::registeredStacks: register one stack (its trace hash and frame ids); returns its stack id, ~0 on failure
  virtual uint64_t RegisterStack(const TraceHash& /*hash*/, const uint64_t* /*ids*/, uint32_t /*n*/) { return ~0ull; }
  // Config::retireIdleBatches (PA_CFG_RETIRE_STACKS aggregator): retire the stacks no batch has named for `idle` batches and
  // append their handles to *handles; called after a flush, on the flushing thread. Returns 0 or a PA_E* code.
  virtual int RetireStacks(uint32_t /*idle*/, std::vector<uint64_t>* /*handles*/) { return PA_EINVAL; }
  virtual int Publish() { return 0; }  // hand buffered rows to the aggregator; called under the reporter's ingest lock
  virtual int Flush(pa_agg_result* out) = 0;
  virtual void Release(pa_agg_result* res) = 0;
  // v1 schema only: the ids of the last flushed batch's unique stacks, and the stacktrace record for a set of ids
  virtual int LastStackIds(uint8_t* /*out*/, uint64_t /*n*/) { return PA_EINVAL; }
  virtual int Stacktraces(const uint8_t* /*ids*/, uint64_t /*n*/, pa_agg_result* /*out*/) { return PA_EINVAL; }
};
// owns nothing; forwards to the C ABI. hash_mode: the aggregator's (RegisterStack passes the trace hash in PA_HASH_PROVIDED mode
// only; in PA_HASH_XXH64X2 mode the library computes the stack id)
Sink* NewAggSink(pa_agg* agg, uint32_t hash_mode = PA_HASH_PROVIDED);

// trace.Hash -> (off, n): open addressing with linear probing in one flat array (a hit is one cache line, where a node-based map
// takes a bucket and a node). erase() shifts the rest of the probe chain back, so no tombstones are left behind.
struct TraceSlot { TraceHash key; uint64_t off; uint32_t n; uint32_t used; };
struct TraceCache {
  std::vector<TraceSlot> slots;
  size_t count = 0;
  static size_t home(const TraceHash& h, size_t mask) { return (size_t)(h.hi * 0x9E3779B97F4A7C15ull ^ h.lo) & mask; }
  const TraceSlot* find(const TraceHash& h) const {
    if (slots.empty()) return nullptr;
    const size_t mask = slots.size() - 1;
    for (size_t i = home(h, mask);; i = (i + 1) & mask) {
      const TraceSlot& s = slots[i];
      if (!s.used) return nullptr;
      if (s.key.hi == h.hi && s.key.lo == h.lo) return &s;
    }
  }
  void put(const TraceHash& h, uint64_t off, uint32_t n) {
    if (slots.empty()) slots.resize(1u << 16);
    if ((count + 1) * 4 > slots.size() * 3) {  // grow (rehash); the reporter clears the cache at kTraceCacheEntries
      std::vector<TraceSlot> old;
      old.swap(slots);
      slots.resize(old.size() * 2);
      count = 0;
      for (auto& s : old) if (s.used) put(s.key, s.off, s.n);
    }
    const size_t mask = slots.size() - 1;
    for (size_t i = home(h, mask);; i = (i + 1) & mask) {
      TraceSlot& s = slots[i];
      if (!s.used) { s = TraceSlot{h, off, n, 1u}; count++; return; }
      if (s.key.hi == h.hi && s.key.lo == h.lo) { s.off = off; s.n = n; return; }
    }
  }
  // backward-shift deletion: every later entry of the chain whose home is not in (hole, entry] moves into the hole
  bool erase(const TraceHash& h) {
    if (slots.empty()) return false;
    const size_t mask = slots.size() - 1;
    size_t i = home(h, mask);
    for (;; i = (i + 1) & mask) {
      if (!slots[i].used) return false;
      if (slots[i].key.hi == h.hi && slots[i].key.lo == h.lo) break;
    }
    for (size_t j = (i + 1) & mask; slots[j].used; j = (j + 1) & mask) {
      const size_t k = home(slots[j].key, mask);
      const bool stays = i <= j ? (i < k && k <= j) : (i < k || k <= j);
      if (!stays) { slots[i] = slots[j]; i = j; }
    }
    slots[i].used = 0;
    count--;
    return true;
  }
  void clear() { slots.clear(); count = 0; }
  size_t size() const { return count; }
};

struct Config {
  std::string nodeName;
  uint32_t samplesPerSecond = 19;          // --profiling-cpu-sampling-frequency
  double reportIntervalSeconds = 5.0;      // --profiling-duration
  bool reportAllocs = false;
  size_t customLabelMaxValLen = 48;        // support.CustomLabelMaxValLen
  // stands in for addMetadataForPID + relabel.ProcessBuilder (:571-585): fill labels, return keep
  std::function<bool(uint32_t pid, Labels* lb)> labelsForPID;
  // receives each non-empty interval's IPC stream (what WriteArrowRequest.IpcBuffer / the offline log carry)
  std::function<void(const uint8_t* ipc, uint64_t len, uint64_t rows)> onBatch;
  // v1 schema in offline mode (:1262-1349): after every sample record, the stacktrace record of the stacks this log
  // has not seen yet is appended as a second batch. The aggregator behind the sink must be a PA_SCHEMA_V1 one.
  bool offlineV1Stacktraces = false;
  // registered stacks (PA_CFG_REGISTERED_STACKS aggregator behind the sink): each distinct trace is registered once through
  // Sink::RegisterStack and its rows carry the stack id in frame_off with no frame ids. Traces are keyed by trace.Hash, the
  // zero hash (oomprof traces) by the frame-id list.
  bool registeredStacks = false;
  // with registeredStacks, on a PA_CFG_RETIRE_STACKS aggregator: after every flush, retire the stacks no batch has named for this
  // many batches (Sink::RetireStacks) and forget their handles, so their traces register again on their next sighting. 0 = off.
  uint32_t retireIdleBatches = 0;
};

class ParcaReporter {
 public:
  ParcaReporter(Sink* sink, Config cfg);
  ~ParcaReporter();

  // reporter.Reporter (observable contract at parca_reporter.go:183-802)
  int ReportTraceEvent(const Trace* trace, const TraceEventMeta* meta);            // :219 — returns 0 (nil) in every V2 branch
  bool SupportsReportTraceEvent() const { return true; }                           // :183
  void ReportFramesForTrace(const Trace*) {}                                       // :635 NOP
  void ReportCountForTrace(TraceHash, uint16_t, const TraceEventMeta*) {}          // :638 NOP
  bool ExecutableKnown(FileID id);                                                 // :643
  void ReportExecutable(const ExecutableMetadata& md);                             // :650
  void ReportHostMetadata(const std::map<std::string, std::string>&) {}            // :695 NOP
  int ReportHostMetadataBlocking(const std::map<std::string, std::string>&, int, double) { return 0; }  // :700 NOP, nil
  // oomprof.Reporter (:709-758): every sample becomes a memory-origin trace of oomprof frames (BuildID stashed in
  // FunctionName, ExecutablePath in SourceFile) and goes through ReportTraceEvent; trace.Hash stays the zero value
  int SampleEvents(const std::vector<MemorySample>& samples, const OomprofSampleMeta& meta);
  void ReportMetrics(uint32_t, const std::vector<uint32_t>&, const std::vector<int64_t>&) {}  // :761 (metric export is out of scope)
  int Start();                                                                     // :1176 — starts the report ticker
  void Stop();                                                                     // :802
  // one tick of the loop at :1199-1225: buildSampleRecordV2 + serialise; returns rows flushed or <0
  int64_t FlushOnce();
  void ResetLoggedStacks();  // log rotation purges offlineModeLoggedStacks (:1131-1133)

  // counters mirroring :899-941
  std::atomic<uint64_t> cpuSamples{0}, offcpuSamples{0}, memorySamples{0}, gpuSamples{0}, emptySamples{0}, skippedByRelabeling{0},
      sampleWrites{0}, sampleWriteRequestBytes{0}, droppedBatches{0}, stacktraceWriteRequestBytes{0}, stacksRetired{0};

 private:
  struct PidLabels { uint32_t labelset = 0; bool keep = true; Labels base; };
  Sink* sink_;
  Config cfg_;
  std::mutex mu_;  // sampleWriterV2Mu (:335): row order == lock acquisition order
  std::unordered_map<std::string, uint32_t> strings_;
  std::string last_comm_;            // consecutive samples mostly come from the same few threads: skip the string hash on a repeat
  uint32_t last_comm_sid_ = 0;
  bool last_comm_valid_ = false;
  std::unordered_map<std::string, uint64_t> frames_;          // serialised Frame value (+exec state) -> frame id
  std::unordered_map<uint64_t, uint64_t> frames_by_handle_;   // Frame::Handle -> frame id (the fast path)
  // trace.Hash -> the frame ids of that trace (the role of the reference's `stacks` LRU, :224-227, turned into an interning
  // cache): a stack seen before costs ONE 16-byte lookup and a copy of its ids instead of one lookup per frame. Bounded;
  // cleared when full and whenever an executable becomes known (frames resolved as UNKNOWN must be looked at again).
  struct TraceHashHasher { size_t operator()(const TraceHash& h) const { return (size_t)(h.hi * 0x9E3779B97F4A7C15ull ^ h.lo); } };
  struct TraceHashEq { bool operator()(const TraceHash& a, const TraceHash& b) const { return a.hi == b.hi && a.lo == b.lo; } };
  // trace.Hash -> (offset, count) in trace_ids_, cleared as a whole when it is three quarters full
  TraceCache trace_cache_;
  std::vector<uint64_t> trace_ids_;
  std::vector<uint64_t> scratch_ids_;
  // Config::registeredStacks: trace.Hash -> stack id (off = the id, n = the depth), and frame-id list -> stack id for the zero hash
  TraceCache stack_cache_;
  std::unordered_map<std::string, uint64_t> zero_hash_stacks_;
  // Config::retireIdleBatches: stack handle -> its key in stack_cache_ / zero_hash_stacks_ (cleared with them), so the handles a
  // retirement returns can be dropped from the caches
  std::unordered_map<uint64_t, TraceHash> hash_of_stack_;
  std::unordered_map<uint64_t, std::string> zero_key_of_stack_;
  static constexpr size_t kTraceCacheEntries = 1u << 20;
  std::map<FileID, ExecutableMetadata> executables_;          // r.executables (:650-693)
  std::map<FileID, std::vector<std::string>> unknown_by_file_;  // frames interned while their executable was unknown
  std::unordered_map<uint32_t, PidLabels> labels_;            // r.labels LRU content (:569)
  std::unordered_map<std::string, uint32_t> labelsets_;       // serialised Labels -> labelset id
  std::unordered_map<std::string, bool> logged_stacks_;       // offlineModeLoggedStacks (:168, :1313-1318)
  std::thread ticker_;
  std::mutex tick_mu_;
  std::condition_variable tick_cv_;
  bool stop_ = false, started_ = false;

  uint32_t sid(const std::string& s);
  uint64_t frameId(const Frame& f);
  uint32_t labelsetId(const Labels& l);
  bool labelsForPID(uint32_t pid, PidLabels** out);
  int writeSampleV2(const Trace* trace, const TraceEventMeta* meta, uint32_t labelset, uint8_t kind, int64_t value, const uint64_t* ids, size_t nids);
  uint64_t stackId(const Trace* trace);  // Config::registeredStacks: the trace's stack id, registered on first sight; ~0 = failed
  int retireStacks();                    // Config::retireIdleBatches: after a flush
};

// maybeFixTruncation (parca_reporter.go:190-216)
bool MaybeFixTruncation(std::string* s, size_t maxLen);

// Offline-mode log framing (SURVEY §8f rank 1; parca_reporter.go:1102-1116, :1807-1831):
// magic A6E7CCCA, u16 BE version, u16 BE batch count, then per batch u32 BE size || IPC stream.
class OfflineLog {
 public:
  explicit OfflineLog(uint16_t version = 0) { header(version); }
  void Append(const uint8_t* ipc, uint64_t len);
  const std::vector<uint8_t>& Bytes() const { return buf_; }
  uint16_t Batches() const { return n_; }
 private:
  std::vector<uint8_t> buf_;
  uint16_t n_ = 0;
  void header(uint16_t version);
};

}  // namespace parca
