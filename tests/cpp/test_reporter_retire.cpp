// Host-layer tests of stack retirement in parca::ParcaReporter (Config::retireIdleBatches, parca_agent_b200/csrc/reporter.hpp):
// after every flush the reporter retires idle stacks through Sink::RetireStacks and drops their handles from its caches, and
// TraceCache::erase keeps every other entry reachable across probe chains.
//   ./test_reporter_retire   — CPU only, against a recording Sink; prints "ok"
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <random>

#include "../../parca_agent_b200/csrc/reporter.hpp"

using namespace parca;

static int failures = 0;
#define REQUIRE(cond) do { if (!(cond)) { fprintf(stderr, "FAIL %s:%d: %s\n", __FILE__, __LINE__, #cond); failures++; } } while (0)

// hands out handles generation << 32 | slot; RetireStacks returns whatever the test queued
struct RetireSink : Sink {
  uint32_t n_strings = 1;
  uint64_t n_frames = 0, n_stacks = 0;
  std::vector<TraceHash> registered;
  std::vector<uint64_t> to_retire;
  std::vector<pa_sample_hdr> rows;
  int retire_calls = 0;
  uint32_t RegisterString(const std::string&) override { return n_strings++; }
  uint64_t RegisterFrame(const pa_frame_desc&) override { return n_frames++; }
  uint32_t RegisterLabelset(const std::vector<pa_label_pair>&) override { return 0; }
  uint64_t RegisterStack(const TraceHash& h, const uint64_t*, uint32_t) override {
    registered.push_back(h);
    return (7ull << 32) | n_stacks++;
  }
  int RetireStacks(uint32_t idle, std::vector<uint64_t>* out) override {
    REQUIRE(idle == 2);
    retire_calls++;
    out->insert(out->end(), to_retire.begin(), to_retire.end());
    to_retire.clear();
    return 0;
  }
  int Submit(const pa_sample_hdr& h, const uint64_t* ids) override { REQUIRE(ids == nullptr); rows.push_back(h); return 0; }
  int Flush(pa_agg_result* out) override { memset(out, 0, sizeof *out); out->n_rows = rows.size(); return 0; }
  void Release(pa_agg_result*) override {}
};

static Frame nativeFrame(uint64_t addr, bool mapped = false, FileID fid = {}) {
  Frame f; f.Type = FrameType{PA_FRAME_NATIVE, "native"}; f.AddressOrLineno = addr; f.MappingValid = mapped; f.MappingHasFile = mapped; f.MappingFileID = fid; return f;
}
static Trace trace(uint64_t hi, uint64_t lo, std::vector<uint64_t> addrs, bool mapped = false, FileID fid = {}) {
  Trace t; t.Hash = TraceHash{hi, lo};
  for (uint64_t a : addrs) t.Frames.push_back(nativeFrame(a, mapped, fid));
  return t;
}
// the stack handle each trace's row carries (one row per trace, in order)
static std::vector<uint64_t> report(ParcaReporter& r, RetireSink& s, const std::vector<const Trace*>& ts) {
  s.rows.clear();
  TraceEventMeta m; m.PID = 1; m.TID = 1; m.Comm = "c";
  for (const Trace* t : ts) r.ReportTraceEvent(t, &m);
  std::vector<uint64_t> out;
  for (auto& h : s.rows) out.push_back(h.frame_off);
  return out;
}

static void testRetiredTracesRegisterAgain() {
  RetireSink s;
  Config cfg; cfg.nodeName = "n"; cfg.registeredStacks = true; cfg.retireIdleBatches = 2;
  ParcaReporter r(&s, cfg);
  Trace a = trace(1, 2, {10, 11}), b = trace(3, 4, {12}), z1 = trace(0, 0, {20, 21}), z2 = trace(0, 0, {22});
  std::vector<uint64_t> h = report(r, s, {&a, &b, &z1, &z2});
  REQUIRE(s.registered.size() == 4 && h.size() == 4);
  REQUIRE(r.FlushOnce() == 4 && s.retire_calls == 1);
  s.to_retire = {h[0], h[2]};  // a and the zero-hash z1 go idle
  REQUIRE(r.FlushOnce() == 4 && s.retire_calls == 2 && r.stacksRetired == 2);
  std::vector<uint64_t> h2 = report(r, s, {&a, &b, &z1, &z2});
  REQUIRE(s.registered.size() == 6);  // a and z1 registered again, b and z2 kept their handles
  REQUIRE(h2[0] != h[0] && h2[1] == h[1] && h2[2] != h[2] && h2[3] == h[3]);
  REQUIRE(s.registered[4].hi == 1 && s.registered[5].hi == 0);
  std::vector<uint64_t> h3 = report(r, s, {&a, &b, &z1, &z2});
  REQUIRE(h3 == h2 && s.registered.size() == 6);
  s.to_retire = {h[0], 0xDEADull};  // a handle that is no longer (or never was) in the caches changes nothing
  r.FlushOnce();
  REQUIRE(report(r, s, {&a, &b, &z1, &z2}) == h2 && s.registered.size() == 6);
}

static void testReplacedEntryStays() {
  // ReportExecutable clears the caches: the next sighting registers a second copy; retiring the first copy must not drop the second
  RetireSink s;
  Config cfg; cfg.nodeName = "n"; cfg.registeredStacks = true; cfg.retireIdleBatches = 2;
  ParcaReporter r(&s, cfg);
  FileID fid{9, 9};
  Trace a = trace(5, 6, {30, 31}, true, fid), z = trace(0, 0, {40}, true, fid);
  std::vector<uint64_t> h = report(r, s, {&a, &z});
  r.ReportExecutable(ExecutableMetadata{fid, "exe", "bid"});
  std::vector<uint64_t> h2 = report(r, s, {&a, &z});
  REQUIRE(s.registered.size() == 4 && h2[0] != h[0] && h2[1] != h[1]);
  s.to_retire = {h[0], h[1]};
  r.FlushOnce();
  REQUIRE(report(r, s, {&a, &z}) == h2 && s.registered.size() == 4);
}

static void testEraseAcrossProbeChains() {
  // keys with hi = 0 have home lo & mask: lo = k << 16 | p collide at home p in the initial 65536-slot table
  const size_t size = 1u << 16;
  auto key = [](uint64_t p, uint64_t k) { return TraceHash{0, (k << 16) | p}; };
  TraceCache c;
  std::vector<TraceHash> all;
  for (uint64_t k = 1; k <= 6; k++) { all.push_back(key(5, k)); all.push_back(key(6, k)); }        // two interleaved chains
  for (uint64_t k = 1; k <= 5; k++) { all.push_back(key(size - 2, k)); all.push_back(key(0, k)); }  // a chain that wraps past the end
  for (size_t i = 0; i < all.size(); i++) c.put(all[i], i, 1);
  REQUIRE(c.slots.size() == size);
  std::vector<bool> gone(all.size(), false);
  auto check = [&] {
    size_t live = 0;
    for (size_t i = 0; i < all.size(); i++) {
      const TraceSlot* s = c.find(all[i]);
      if (gone[i]) REQUIRE(s == nullptr); else { REQUIRE(s && s->off == i); live++; }
    }
    REQUIRE(c.size() == live);
  };
  for (size_t i : {0u, 3u, 12u, 13u, 20u, 7u}) { REQUIRE(c.erase(all[i])); gone[i] = true; check(); }
  REQUIRE(!c.erase(all[0]) && !c.erase(key(5, 99)));
  // random insert / erase against a std::map, in a small table with many collisions (home = lo & 65535 over 64 homes)
  std::mt19937_64 rng(3);
  TraceCache d;
  std::map<uint64_t, uint64_t> ref;
  for (int step = 0; step < 200000; step++) {
    const uint64_t lo = ((rng() % 512) << 16) | (rng() % 64);
    if (rng() % 3) { d.put(TraceHash{0, lo}, step, 1); ref[lo] = step; }
    else { REQUIRE(d.erase(TraceHash{0, lo}) == (ref.erase(lo) == 1)); }
  }
  REQUIRE(d.size() == ref.size());
  for (auto& kv : ref) { const TraceSlot* s = d.find(TraceHash{0, kv.first}); REQUIRE(s && s->off == kv.second); }
  size_t used = 0;
  for (auto& s : d.slots) used += s.used;
  REQUIRE(used == ref.size());
}

int main() {
  testRetiredTracesRegisterAgain();
  testReplacedEntryStays();
  testEraseAcrossProbeChains();
  if (failures) return 1;
  printf("ok\n");
  return 0;
}
