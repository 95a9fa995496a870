// Host-layer tests of parca::ParcaReporter with Config::registeredStacks (parca_agent_b200/csrc/reporter.hpp): each distinct
// trace is registered once through Sink::RegisterStack and its rows name the stack in frame_off, with no frame ids.
//   ./test_reporter_stacks   — CPU only, against a recording Sink; prints "ok"
#include <cstdio>
#include <cstdlib>
#include <cstring>

#include "../../parca_agent_b200/csrc/reporter.hpp"

using namespace parca;

static int failures = 0;
#define REQUIRE(cond) do { if (!(cond)) { fprintf(stderr, "FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); failures++; } } while (0)

struct StackSink : Sink {
  uint32_t n_strings = 1;
  uint64_t n_frames = 0;
  uint32_t n_labelsets = 0;
  struct Reg { TraceHash hash; std::vector<uint64_t> ids; };
  std::vector<Reg> stacks;
  std::vector<pa_sample_hdr> rows;
  std::vector<bool> row_has_ids;
  uint32_t RegisterString(const std::string&) override { return n_strings++; }
  uint64_t RegisterFrame(const pa_frame_desc&) override { return n_frames++; }
  uint32_t RegisterLabelset(const std::vector<pa_label_pair>&) override { return n_labelsets++; }
  uint64_t RegisterStack(const TraceHash& h, const uint64_t* ids, uint32_t n) override {
    stacks.push_back(Reg{h, std::vector<uint64_t>(ids, ids + n)});
    return stacks.size() - 1;
  }
  int Submit(const pa_sample_hdr& h, const uint64_t* ids) override { rows.push_back(h); row_has_ids.push_back(ids != nullptr); return 0; }
  int Flush(pa_agg_result* out) override { memset(out, 0, sizeof *out); out->n_rows = rows.size(); rows.clear(); row_has_ids.clear(); return 0; }
  void Release(pa_agg_result*) override {}
};

// a sink that only knows the ring: the default RegisterStack refuses
struct RingOnlySink : Sink {
  uint32_t ns = 1;
  uint64_t nf = 0;
  std::vector<pa_sample_hdr> rows;
  std::vector<std::vector<uint64_t>> row_frames;
  uint32_t RegisterString(const std::string&) override { return ns++; }
  uint64_t RegisterFrame(const pa_frame_desc&) override { return nf++; }
  uint32_t RegisterLabelset(const std::vector<pa_label_pair>&) override { return 0; }
  int Submit(const pa_sample_hdr& h, const uint64_t* ids) override { rows.push_back(h); row_frames.emplace_back(ids, ids + h.nframes); return 0; }
  int Flush(pa_agg_result* out) override { memset(out, 0, sizeof *out); return 0; }
  void Release(pa_agg_result*) override {}
};

static Frame nativeFrame(uint64_t addr, bool mapped = false, FileID fid = {}) {
  Frame f; f.Type = FrameType{PA_FRAME_NATIVE, "native"}; f.AddressOrLineno = addr; f.MappingValid = mapped; f.MappingHasFile = mapped; f.MappingFileID = fid; return f;
}

static Config config(bool registered) {
  Config cfg;
  cfg.nodeName = "n";
  cfg.registeredStacks = registered;
  return cfg;
}

static void testOneRegistrationPerTrace() {
  StackSink sink;
  ParcaReporter r(&sink, config(true));
  Trace a; a.Hash = {1, 2}; a.Frames = {nativeFrame(0x10), nativeFrame(0x20), nativeFrame(0x30)};
  Trace b; b.Hash = {3, 4}; b.Frames = {nativeFrame(0x20)};
  Trace e; e.Hash = {5, 6};  // no frames
  TraceEventMeta m; m.PID = 7; m.TID = 8; m.Comm = "c";
  for (int i = 0; i < 3; i++) { r.ReportTraceEvent(&a, &m); r.ReportTraceEvent(&b, &m); r.ReportTraceEvent(&e, &m); }
  REQUIRE(sink.stacks.size() == 3);
  REQUIRE(sink.stacks[0].hash.hi == 1 && sink.stacks[0].hash.lo == 2 && sink.stacks[0].ids == (std::vector<uint64_t>{0, 1, 2}));
  REQUIRE(sink.stacks[1].hash.hi == 3 && sink.stacks[1].ids == (std::vector<uint64_t>{1}));
  REQUIRE(sink.stacks[2].ids.empty());
  REQUIRE(sink.rows.size() == 9);
  for (size_t i = 0; i < sink.rows.size(); i++) {
    REQUIRE(!sink.row_has_ids[i]);                   // rows carry no frame ids
    REQUIRE(sink.rows[i].frame_off == i % 3);        // frame_off = the stack id
    REQUIRE(sink.rows[i].hash_hi == (i % 3 == 0 ? 1u : i % 3 == 1 ? 3u : 5u));
  }
  REQUIRE(sink.rows[0].nframes == 3 && sink.rows[2].nframes == 0);
}

static void testZeroHashKeyedByFrames() {
  StackSink sink;
  ParcaReporter r(&sink, config(true));
  Trace x; x.Frames = {nativeFrame(0x10), nativeFrame(0x20)};  // the zero hash (oomprof traces)
  Trace y; y.Frames = {nativeFrame(0x20), nativeFrame(0x10)};
  Trace x2 = x;
  TraceEventMeta m; m.PID = 7;
  r.ReportTraceEvent(&x, &m); r.ReportTraceEvent(&y, &m); r.ReportTraceEvent(&x2, &m); r.ReportTraceEvent(&y, &m);
  REQUIRE(sink.stacks.size() == 2);
  REQUIRE(sink.stacks[0].ids == (std::vector<uint64_t>{0, 1}) && sink.stacks[1].ids == (std::vector<uint64_t>{1, 0}));
  REQUIRE(sink.rows.size() == 4 && sink.rows[0].frame_off == 0 && sink.rows[1].frame_off == 1 && sink.rows[2].frame_off == 0 && sink.rows[3].frame_off == 1);
  // oomprof samples go through the same path
  std::vector<MemorySample> ms(2);
  ms[0].Allocs = 2; ms[0].Addresses = {0x100, 0x200};
  ms[1].Allocs = 3; ms[1].Addresses = {0x100, 0x200};
  OomprofSampleMeta om; om.PID = 9; om.BuildID = "bid"; om.ExecutablePath = "/bin/x";
  REQUIRE(r.SampleEvents(ms, om) == 0);
  REQUIRE(sink.stacks.size() == 3 && sink.stacks[2].hash.hi == 0 && sink.stacks[2].hash.lo == 0 && sink.stacks[2].ids.size() == 2);
  REQUIRE(sink.rows.size() == 6 && sink.rows[4].frame_off == 2 && sink.rows[5].frame_off == 2);
}

static void testReregistrationAfterReportExecutable() {
  StackSink sink;
  ParcaReporter r(&sink, config(true));
  const FileID fid{0xaa, 0xbb};
  Trace t; t.Hash = {9, 9}; t.Frames = {nativeFrame(0x10, true, fid), nativeFrame(0x20)};
  TraceEventMeta m; m.PID = 7;
  r.ReportTraceEvent(&t, &m);
  r.ReportTraceEvent(&t, &m);
  REQUIRE(sink.stacks.size() == 1 && sink.n_frames == 2);
  r.ReportExecutable(ExecutableMetadata{fid, "/bin/app", "gnu"});  // the unknown-executable frame is interned again
  r.ReportTraceEvent(&t, &m);
  REQUIRE(sink.stacks.size() == 2 && sink.n_frames == 3);
  REQUIRE(sink.stacks[1].ids == (std::vector<uint64_t>{2, 1}));
  REQUIRE(sink.rows.size() == 3 && sink.rows[1].frame_off == 0 && sink.rows[2].frame_off == 1);
  r.ReportExecutable(ExecutableMetadata{fid, "/bin/app", "gnu"});  // already known: nothing is forgotten
  r.ReportTraceEvent(&t, &m);
  REQUIRE(sink.stacks.size() == 2 && sink.rows[3].frame_off == 1);
}

static void testFailedRegistrationDropsTheSample() {
  RingOnlySink sink;
  ParcaReporter r(&sink, config(true));
  Trace t; t.Hash = {1, 1}; t.Frames = {nativeFrame(0x10)};
  TraceEventMeta m; m.PID = 7;
  REQUIRE(r.ReportTraceEvent(&t, &m) == 0);
  REQUIRE(sink.rows.empty() && r.droppedBatches == 1);
}

static void testRingModeUnchanged() {
  RingOnlySink sink;
  ParcaReporter r(&sink, config(false));
  Trace t; t.Hash = {1, 2}; t.Frames = {nativeFrame(0x10), nativeFrame(0x20)};
  Trace z; z.Frames = {nativeFrame(0x20)};
  TraceEventMeta m; m.PID = 7;
  r.ReportTraceEvent(&t, &m); r.ReportTraceEvent(&z, &m); r.ReportTraceEvent(&t, &m);
  REQUIRE(sink.rows.size() == 3);
  REQUIRE(sink.row_frames[0] == (std::vector<uint64_t>{0, 1}) && sink.row_frames[1] == (std::vector<uint64_t>{1}) && sink.row_frames[2] == sink.row_frames[0]);
  REQUIRE(sink.rows[0].frame_off == 0 && sink.rows[2].frame_off == 0 && sink.rows[0].nframes == 2);
}

int main() {
  testOneRegistrationPerTrace();
  testZeroHashKeyedByFrames();
  testReregistrationAfterReportExecutable();
  testFailedRegistrationDropsTheSample();
  testRingModeUnchanged();
  if (failures) { fprintf(stderr, "%d failures\n", failures); return 1; }
  printf("ok\n");
  return 0;
}
