// Host-shim throughput with ring rows vs registered stacks: bench_reporter.cpp's measurement (samples/s through
// parca::ParcaReporter::ReportTraceEvent, parca_agent_b200/csrc/reporter.hpp) with the row form as an argument.
//   ./bench_reporter_stacks N F U P null|gpu handle|value ring|stacks
//     N samples of F frames drawn from U stacks over P distinct frames; sink = a counting stub (host cost alone) or the real
//     aggregator on cuda:0 (ingest + one flush at the end); frame key = unique.Handle-style 8-byte handle or the whole value;
//     rows = frame ids in the ring or registered stacks (PA_CFG_REGISTERED_STACKS: each trace registered once, rows
//     name their stack).
// Prints one JSON line. Single producer thread (the reference serialises producers on sampleWriterV2Mu, parca_reporter.go:335).
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>

#include "../../parca_agent_b200/csrc/reporter.hpp"

using namespace parca;

struct NullSink : Sink {
  uint32_t ns = 1, nl = 0;
  uint64_t nf = 0, rows = 0, frames = 0, nst = 0;
  uint32_t RegisterString(const std::string&) override { return ns++; }
  uint64_t RegisterFrame(const pa_frame_desc&) override { return nf++; }
  uint64_t RegisterStack(const TraceHash&, const uint64_t*, uint32_t) override { return nst++; }
  uint32_t RegisterLabelset(const std::vector<pa_label_pair>&) override { return nl++; }
  int Submit(const pa_sample_hdr& h, const uint64_t* ids) override { rows++; if (ids) frames += h.nframes; return 0; }
  int Flush(pa_agg_result* out) override { memset(out, 0, sizeof *out); out->n_rows = rows; rows = 0; return 0; }
  void Release(pa_agg_result*) override {}
};

static double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

int main(int argc, char** argv) {
  if (argc < 8) { fprintf(stderr, "usage: %s N F U P null|gpu handle|value ring|stacks\n", argv[0]); return 2; }
  const uint64_t N = strtoull(argv[1], nullptr, 10);
  const uint32_t F = (uint32_t)atoi(argv[2]), U = (uint32_t)atoi(argv[3]), P = (uint32_t)atoi(argv[4]);
  const bool gpu = !strcmp(argv[5], "gpu"), handle = !strcmp(argv[6], "handle"), stacks_mode = !strcmp(argv[7], "stacks");
  std::mt19937_64 rng(0x5EED);
  std::vector<Frame> frames(P);
  for (uint32_t i = 0; i < P; i++) {
    Frame& f = frames[i];
    const bool native = i % 5 != 0;
    f.Type = native ? FrameType{PA_FRAME_NATIVE, "native"} : FrameType{PA_FRAME_INTERP, "python"};
    f.AddressOrLineno = 0x400000 + 16ull * i;
    if (!native) { f.FunctionName = "mod.fn_" + std::to_string(i / 4); f.SourceFile = "/usr/lib/python/site/m" + std::to_string(i / 32) + ".py"; f.SourceLine = i % 5000; }
    f.Handle = handle ? 0x7f0000000000ull + 64ull * i : 0;  // a stable, unique, pointer-like value per distinct Frame
  }
  std::vector<Trace> stacks(U);
  for (uint32_t u = 0; u < U; u++) {
    stacks[u].Hash = TraceHash{rng(), rng()};
    for (uint32_t j = 0; j < F; j++) stacks[u].Frames.push_back(frames[rng() % P]);
  }
  pa_agg* agg = nullptr;
  Sink* sink = nullptr;
  NullSink null_sink;
  if (gpu) {
    pa_agg_config cfg;
    memset(&cfg, 0, sizeof cfg);
    cfg.abi_version = PA_ABI_VERSION; cfg.device = 0; cfg.hash_mode = PA_HASH_XXH64X2; cfg.samples_per_second = 19;
    cfg.max_samples = N; cfg.max_frames = stacks_mode ? (uint64_t)U * F : N * F; cfg.chunk_samples = 1u << 20;
    if (stacks_mode) cfg.flags |= PA_CFG_REGISTERED_STACKS;
    if (pa_agg_create(&cfg, &agg) != PA_OK) { fprintf(stderr, "pa_agg_create failed\n"); return 1; }
    sink = NewAggSink(agg, cfg.hash_mode);
  } else {
    sink = &null_sink;
  }
  Config cfg;
  cfg.nodeName = "node-0";
  cfg.registeredStacks = stacks_mode;
  cfg.labelsForPID = [](uint32_t pid, Labels* lb) { lb->emplace_back("comm", "proc-" + std::to_string(pid)); return true; };
  uint64_t out_bytes = 0, out_rows = 0;
  cfg.onBatch = [&](const uint8_t*, uint64_t len, uint64_t rows) { out_bytes += len; out_rows += rows; };
  ParcaReporter rep(sink, cfg);
  // warm the interning tables with one pass over every stack (a steady-state agent has seen its frames before)
  TraceEventMeta meta;
  meta.Comm = "worker";
  for (uint32_t u = 0; u < U; u++) { meta.PID = 1000 + u % 4096; meta.TID = meta.PID * 16 + u % 16; rep.ReportTraceEvent(&stacks[u], &meta); }
  rep.FlushOnce();
  out_bytes = out_rows = 0;
  const double t0 = now_s();
  for (uint64_t i = 0; i < N; i++) {
    const Trace& t = stacks[rng() % U];
    meta.PID = 1000 + (uint32_t)(i % 4096);
    meta.TID = meta.PID * 16 + (uint32_t)(i % 16);
    meta.CPU = (int)(i % 192);
    meta.Timestamp = 1700000000000000000ll + (int64_t)i * 52631;
    rep.ReportTraceEvent(&t, &meta);
  }
  const double t1 = now_s();
  const int64_t rows = rep.FlushOnce();
  const double t2 = now_s();
  printf("{\"samples\": %llu, \"frames_per_sample\": %u, \"unique_stacks\": %u, \"distinct_frames\": %u, \"sink\": \"%s\", \"frame_key\": \"%s\", \"rows\": \"%s\", "
         "\"ingest_s\": %.6f, \"flush_s\": %.6f, \"ingest_samples_per_s\": %.1f, \"ingest_plus_flush_samples_per_s\": %.1f, \"rows_flushed\": %lld, \"ipc_bytes\": %llu}\n",
         (unsigned long long)N, F, U, P, gpu ? "gpu" : "null", handle ? "handle" : "value", stacks_mode ? "stacks" : "ring", t1 - t0, t2 - t1, N / (t1 - t0), N / (t2 - t0), (long long)rows,
         (unsigned long long)out_bytes);
  if (agg) { delete sink; pa_agg_destroy(agg); }
  return rows == (int64_t)N ? 0 : 1;
}
