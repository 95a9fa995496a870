// agg.cu — libparcaagg: host orchestration + C ABI (include/parcaagg.h).
//
// One pa_agg = one ParcaReporter's V2 sample writer (reporter/parca_reporter.go). Ingest lands in
// a C-owned pinned ring (double-buffered: flush swaps buffers under the ingest lock exactly like
// buildSampleRecordV2 swaps writers, :1743-1748), flush stages the detached buffer to HBM in
// chunks (copy stream) while the compute stream hashes/dedups the chunks already resident, then
// ranks/gathers dictionaries, run-end encodes the label and constant columns, and finally copies
// each finished Arrow buffer device->host straight into its place in the IPC stream.
#include <cuda_runtime.h>
#include <execinfo.h>
#include <signal.h>
#include <unistd.h>

#include <algorithm>
#include <functional>
#include <chrono>
#include <cstdlib>
#include <condition_variable>
#include <map>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/parcaagg.h"
#include "host_tables.hpp"
#include "ipc_lz4.hpp"
#include "ipc_out.hpp"
#include "kernels.cuh"

namespace pa {

static double now_ms() {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

struct DBuf {
  void* p = nullptr;
  size_t cap = 0;
  cudaError_t ensure(size_t n) {
    if (n <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    size_t want = std::max(n, cap + cap / 2);
    cudaError_t e = cudaMalloc(&p, want);
    cap = e == cudaSuccess ? want : 0;
    return e;
  }
  template <class T> T* as() const { return (T*)p; }
  void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

// growable device mirror of an append-only host vector
template <class T>
struct Mirror {
  DBuf buf;
  size_t uploaded = 0;
  cudaError_t sync(const std::vector<T>& h, cudaStream_t s) {
    if (!buf.p || h.size() * sizeof(T) > buf.cap) {
      DBuf nb;
      cudaError_t e = nb.ensure(std::max<size_t>(h.size() * sizeof(T) * 2, 256));
      if (e != cudaSuccess) return e;
      buf.release();
      buf = nb;
      uploaded = 0;
    }
    if (uploaded < h.size()) {
      cudaError_t e = cudaMemcpyAsync(buf.as<T>() + uploaded, h.data() + uploaded, (h.size() - uploaded) * sizeof(T), cudaMemcpyHostToDevice, s);
      if (e != cudaSuccess) return e;
      uploaded = h.size();
    }
    return cudaSuccess;
  }
  const T* ptr() const { return buf.as<T>(); }
};

struct ColPlan {
  std::string name;
  uint32_t type = COL_LS;
  uint32_t param = 0;              // LS: column of the batch's key matrix; KIND: table row
  uint32_t ord = 0;                // LS: the label name's ordinal (its value ids index LabelSets::vals[ord])
  uint32_t universe = 0;
  // device pointers for this flush
  int* run_ends = nullptr;
  uint32_t* run_keys = nullptr;    // becomes the dictionary indices in place
  uint32_t* validity = nullptr;
  uint32_t* order = nullptr;
};

struct Timer {
  cudaEvent_t a = nullptr, b = nullptr;
  uint32_t launches = 0;
  double ms = 0;
};
static const char* kTimerNames[] = {"header", "hash", "rank", "locations", "labels", "dicts", "total", "lz4"};
enum { T_HEADER, T_HASH, T_RANK, T_LOC, T_LABELS, T_DICTS, T_TOTAL, T_LZ4 /* collect / stacktraces, not process */, T_COUNT };

}  // namespace pa

using namespace pa;

// this aggregator as shard `rank` of a merged batch (mode B): its rows are the global rows row_base .. row_base+N-1
struct MergeDims { uint32_t world = 1, rank = 0; uint64_t row_base = 0, n_total = 0, nf_total = 0; const uint32_t* slice_len_ptr = nullptr; };

// everything the stages of one pass share (valid from pass_plan until the batch is collected)
struct Pass {
  // registration state as mirrored to the device for this batch (snapshot taken under reg_mu in upload_tables)
  uint32_t n_cstr = 0, n_frames = 0, n_funcs = 0, n_sids = 0, n_labelsets = 0, n_names = 0;
  uint32_t n_stacks = 0;         // stack slots on the device (PA_CFG_REGISTERED_STACKS)
  uint64_t n_stack_frames = 0;    // and the frame ids of their arena (freed stacks' included until a compaction)
  uint64_t stack_digest = 0;      // PA_CFG_GROUP_STACKS: digest of those stacks (merge groups check it is the same on every member)
  uint64_t stack_frames_live = 0; // frames of the uploaded stacks not yet freed (in a merge group, the same on every member)
  uint64_t N = 0, NT = 0, row_base = 0;
  uint32_t world = 1, rank = 0, ncols = 0, nlab = 0;
  bool v1 = false, provided = false, merged = false;  // provided: the stack ids arrive with the rows (or their registered stacks)
  uint64_t cap = 0, tcap = 0;
  uint32_t mask = 0;
  size_t Pn = 1, S = 1, FN = 1, NI = 1;
  size_t cls_bytes[3] = {0, 0, 0};
  uint32_t *rowbits = nullptr, *row_wprefix = nullptr, *uniq_slot = nullptr, *uniq_size = nullptr, *first_ls = nullptr, *claimed = nullptr;
  uint32_t *loc_bits = nullptr, *loc_wp = nullptr, *sd_bits[4] = {}, *sd_wp[4] = {}, *fn_bits = nullptr, *fn_wp = nullptr;
  unsigned long long* edge_keys = nullptr;
  // label column plan check (k_ls_plan): per labelset its row of the key matrix [used labelsets][planned LS columns], the
  // used-labelset count, the used-name bitmap over the name ordinals (read back with the counters)
  uint32_t *ls_rank = nullptr, *ls_keys = nullptr, *ls_used = nullptr, *used_names = nullptr;
  uint32_t* red_block = nullptr; // [first_ls | first_cpu | first_comm | v1: first_kind]: the direct first-row tables mode B all-reduces
  size_t red_count = 0;
  std::vector<uint32_t*> col_first, col_rank, col_bits, col_wp;
  int j_loc = 0, j_type = 0, j_file = 0, j_lab0 = 0;
  std::vector<FoJob> jobs;
  std::vector<ReeCol> rc;
  ReeArgs ra{};
  ReeGroups rg{};        // every column group
};

struct pa_agg {
  pa_agg_config cfg{};
  std::string err;
  int device = 0, sms = 148, G = 592;
  cudaStream_t s_copy = nullptr, s_comp = nullptr, s_aux = nullptr, s_d2h = nullptr;
  cudaEvent_t ev_fork = nullptr, ev_join = nullptr;
  // Early copy-out during a flush (XXH64 mode, v2, more than one chunk): all headers are uploaded first, k_header and the label
  // chain run while the frame ids are still uploading, and stacktrace_id / value / timestamp leave for the host on s_d2h as soon
  // as they are final, at positions counted from the END of the output buffer (see append_tail_v2). collect() anchors the stream
  // so that it ends there and skips what is already in place; anything that does not match is copied the ordinary way.
  struct Early {
    bool hdr_first = false;   // this batch was staged headers-first
    bool issued = false;      // early copies are in flight / done
    uint8_t* out_end = nullptr;
    uint64_t dist_ts = 0, dist_value = 0, dist_uuid = 0;
    uint64_t dist_stoff = 0, dist_stsize = 0, dist_stream = 0;  // second wave (collect): list offsets / sizes and the location-index stream sit right before stacktrace_id
  } early;
  bool early_enabled = true, early_force = false;
  cudaEvent_t ev_hdr_all = nullptr, ev_hdr_done = nullptr, ev_early = nullptr, ev_early_done = nullptr;
  std::vector<cudaEvent_t> hash_ev;
  uint8_t* h_early = nullptr;  // pinned: Counters, then the run keys of the eight kind-derived columns
  static constexpr uint32_t kEarlyMaxRuns = 512;
  bool forked_early = false;  // headers-first staging: the label chain was forked right after the header pass, beside the hash kernel
  bool serial = false;       // PA_SERIAL=1: the label chain stays on the compute stream (per-group timings do not overlap)
  Pass P;
  bool merged_part = false;  // the processed batch is one shard of a merged record (collected through pa_merge_collect)

  // ---- registration state
  std::mutex reg_mu;
  StringPool sp;
  FrameTableHost ft;
  LabelSets ls;
  std::vector<std::pair<uint32_t, uint32_t>> external;  // canonical ids
  std::vector<ColPlan> cols;  // label columns of this batch's plan, then the 8 constant-ish columns
  uint32_t n_label_cols = 0, n_lscols = 0;  // label columns; the labelset-derived ones among them (the first n_lscols)
  // Label column plan (DESIGN section 4): the labelset-derived columns of a batch are a predicted set of name ordinals, the
  // names the previous batch's rows used plus every name registered since; the pass checks it and is redone on a miss.
  std::vector<uint32_t> used_prev;  // name ordinals the rows of the last processed batch used, ascending
  uint32_t names_planned = 0;       // names registered when that batch was planned
  bool plan_pending = false;        // a batch was planned and has not completed: the next plan starts cold
  uint64_t label_replans = 0;       // passes redone because the prediction missed a used name, since creation
  uint64_t plan_digest = 0;         // digest of the planned name ordinals (merge groups check that every member has the same plan)
  uint32_t* h_used = nullptr;       // pinned: the used-name bitmap of the last pass
  size_t h_used_words = 0;
  std::vector<uint32_t> kindtab;           // [8][8]
  std::vector<std::vector<std::string>> kind_strings;  // class -> string for the 6 string columns
  std::vector<int64_t> period_vals;
  std::vector<uint64_t> duration_vals;

  Mirror<uint64_t> m_addr, m_line;
  Mirror<uint32_t> m_type, m_map, m_bid, m_func, m_fnfile, m_sid2cid;
  Mirror<uint32_t> m_ls_off, m_ls_pairs;  // the registered labelsets (LabelSets::off, LabelSets::pairs)
  DBuf d_kindtab, d_cols, d_jobs;
  // PA_CFG_REGISTERED_STACKS: the stack registry. The device holds it (records, last_use, the frame arena with ids at the ring's
  // width, idb / 4 words each). The host keeps per-slot metadata, the free slots (a min-heap), the retired stacks waiting for
  // their grace batch, and the registrations not yet uploaded. Without PA_CFG_RETIRE_STACKS no slot is ever freed, so every
  // stack takes the next slot with generation 0 and its handle is its consecutive id.
  bool registered = false;
  bool group_stacks = false;  // PA_CFG_GROUP_STACKS: the stack ids are group-wide (merge groups)
  uint64_t reg_digest = 0;    // PA_CFG_GROUP_STACKS: running digest of every registered stack's (handle, id, depth, frame ids)
  // PA_CFG_GROUP_RETIRE: running digest of every group retirement's (idle_batches, handles), kept apart from reg_digest so that a
  // registration running concurrently with pa_merge_retire_stacks may land before or after it on each member; rs_upload combines
  // the two
  uint64_t retire_digest = 0;
  enum : uint8_t { RS_LIVE, RS_RETIRING, RS_FREE };
  bool retire = false;  // PA_CFG_RETIRE_STACKS: stacks can be retired and their slots reused
  bool group_retire = false;  // PA_CFG_GROUP_RETIRE (retire is set too): the merge group retires, through pa_merge_retire_stacks
  std::vector<uint32_t> rs_depth, rs_gen;  // rs_gen: the generation of the slot's current (or next) stack
  std::vector<uint8_t> rs_state;
  std::vector<uint32_t> rs_free;
  std::vector<std::pair<uint32_t, uint64_t>> rs_retiring;  // (slot, stage count at which it is freed)
  std::vector<RegStack> rs_pend;  // off relative to rs_pend_frames
  std::vector<uint32_t> rs_pend_slot, rs_pend_seq, rs_pend_frames;
  uint64_t rs_stages = 0;         // batches staged so far (the sequence number of the last one)
  uint64_t rs_live = 0, rs_frames_live = 0, rs_frames_dead = 0, rs_retired = 0, rs_compactions = 0;
  uint64_t rs_dev_slots = 0, rs_dev_len = 0;  // records and arena ids on the device (dead frames included)
  DBuf d_rs_recs, d_rs_last, d_rs_arena[2], d_rs_tmp, d_rs_upd;
  int rs_cur = 0;
  Timer rs_tm;  // the last compaction
  // v1: frames resolved by the buildStacktraceRecord rules + the device-resident store of known stacks
  Mirror<uint32_t> m1_map, m1_bid, m1_fn, m1_file;
  Mirror<uint64_t> m1_line, m1_col;
  Mirror<uint8_t> m1_complete;
  DBuf d_store, d_store_arena, d_store_ctl, d_v1_ids, d_st1;
  DBuf d_store_stamp, d_v1_last, d_select;  // last access per store slot; last row per stack of the batch; radix-select scratch
  uint64_t store_entries = 0, store_slots = 0, store_frames = 0, last_unique = 0;
  uint64_t store_epoch = 0;                  // LRU clock: one tick per ingested batch and per stacktrace request
  uint32_t* h_select = nullptr;              // pinned: 256-bin histogram of a select pass, then a StoreCtl read-back
  uint64_t store_compactions = 0, store_evictions = 0;
  uint64_t store_frames_sent = 0;            // v1 merge groups: frame ids this member sent in the last store exchange
  uint64_t store_refs_sent = 0;              // v1 PA_CFG_GROUP_STACKS merge groups: the stack handles it sent instead
  uint32_t cid_unknown = 0, cid_missing = 0;  // "unknown" (libpf.UnknownFrame.String()) and "missing stacktrace" (:1561, :1568)

  // ---- ring (pinned host), double buffered
  struct Ring { pa_sample_hdr* hdr = nullptr; uint64_t* frames = nullptr; const uint64_t* frames_dev = nullptr; uint64_t rows = 0, nfr = 0; } ring[2];
  int active = 0, inflight = 0;
  uint32_t idb = 8;          // bytes per frame id in the ring and in d_frames (pa_agg_config.frame_id_bytes)
  bool single_ring = false, ring_busy = false;  // PA_CFG_SINGLE_RING: the one buffer is held by a flush until it is collected
  std::mutex ring_mu;
  std::condition_variable ring_cv;
  std::mutex flush_mu;

  // ---- staged batch
  int staged = -1;
  uint64_t N = 0, NF = 0;
  std::vector<cudaEvent_t> chunk_ev;
  std::vector<std::pair<uint64_t, uint64_t>> chunk_rows;    // [row0,row1)
  std::vector<uint64_t> chunk_frames_end;
  cudaEvent_t ev_h2d0 = nullptr, ev_h2d1 = nullptr, ev_d2h0 = nullptr, ev_d2h1 = nullptr;
  bool processed = false, hash_timed = false;
  const unsigned long long* src_frames = nullptr;  // where the staged batch's frame ids can be read by kernels (set by stage / stage_device)
  // 8 = tma24x2 (default: wide's lane layout over per-sample cp.async.bulk copies into shared memory, 24 warps x 2 stages per
  // SM; on an H100 its hash pass takes 2.11 ms where wide takes 2.26 on config 2), 2 = wide (2 lanes/sample, 16-byte loads;
  // also the uint32-ring kernel), 0 = direct (4 lanes/sample), 1 = cp.async-staged, 3 / 4 = cp.async.bulk + mbarrier staged,
  // thread-per-sample (4 warps x 3 stages / 6 warps x 2 stages per SM); PA_HASH_VARIANT=tma24x2|wide|direct|staged|bulk|...
  static constexpr int kDefaultHashVariant = 8;
  int hash_variant = kDefaultHashVariant;

  // ---- device batch buffers
  DBuf d_hdr, d_frames, d_ts, d_value, d_uuid, d_stoff, d_stsize, d_slot, d_kind, d_nfr, d_foff, d_ls, d_cpu, d_tid, d_comm;
  DBuf d_ustream, d_uniq_row, d_uniq_count, d_table, d_ctr, d_arena, d_partial, d_partial2, d_ree_partial;
  uint64_t table_cap = 0, retry_cap = 0, tid_cap = 0, retry_tcap = 0, prev_tids = 0;
  uint64_t prev_unique = 0;
  Counters h_ctr{};
  Counters* h_ctr_pinned = nullptr;
  // arena-carved pointers (valid for the current flush)
  uint32_t *loc_first = nullptr, *loc_rank = nullptr, *loc_order = nullptr;
  uint32_t *sd_first[4] = {}, *sd_rank[4] = {}, *sd_order[4] = {}, *sd_keys[4] = {}, *sd_valid[4] = {};  // type,map,bid,file
  uint32_t *fn_first = nullptr, *fn_rank = nullptr, *fn_order = nullptr, *fn_keys = nullptr;
  LocOut lo{};
  uint32_t *v1_ord = nullptr, *v1_first_kind = nullptr, *v1_kindrank = nullptr, *v1_kind_order = nullptr, *v1_n_kind_dict = nullptr;
  long long* v1_ts_vals = nullptr;
  uint8_t* v1_ids = nullptr;
  int* v1_id_off = nullptr;
  unsigned long long* tid_slots = nullptr;
  uint32_t* tid_rank = nullptr;
  uint32_t tid_mask = 0;

  // ---- output
  uint8_t* out = nullptr;
  uint64_t out_cap = 0;
  uint8_t* h_desc = nullptr;
  size_t h_desc_cap = 0;
  std::vector<std::vector<uint8_t>> hostbufs;  // host-built Arrow buffers of the current result
  std::vector<uint8_t> comp_out;               // PA_IPC_LZ4_FRAME: the re-encoded stream the result points at
  DBuf d_lz4, d_lz4_body;                      // PA_IPC_LZ4_FRAME_GPU: block tables, host-source staging and block slots; compressed bodies
  uint64_t lz4_head_bytes = 0;                 // merge groups in that mode: bytes of block heads this member sent in the last plan
  cudaEvent_t ev_lz4p0 = nullptr, ev_lz4p1 = nullptr;  // around k_lz4_pack (T_LZ4 covers compress + layout)
  Timer tm[T_COUNT];
  uint32_t launches = 0;
  double h2d_ms = 0;

  int fail(int code, const char* what, cudaError_t e = cudaSuccess) {
    err = what;
    if (e != cudaSuccess) { err += ": "; err += cudaGetErrorString(e); }
    return code;
  }
};

// PA_BACKTRACE=1: print the native call stack of a fatal signal (addresses are offsets into libparcaagg.so: addr2line -e)
static void fatal_backtrace(int sig) {
  void* frames[64];
  int n = backtrace(frames, 64);
  const char msg[] = "libparcaagg: fatal signal, native backtrace:\n";
  if (write(2, msg, sizeof msg - 1) < 0) {}
  backtrace_symbols_fd(frames, n, 2);
  signal(sig, SIG_DFL);
  raise(sig);
}
static uint64_t pow2_at_least(uint64_t v) { uint64_t p = 1; while (p < v) p <<= 1; return p; }

#define CK(expr)                                                        \
  do {                                                                  \
    cudaError_t e_ = (expr);                                            \
    if (e_ != cudaSuccess) return a->fail(PA_EIO, #expr, e_);           \
  } while (0)

// ---------------------------------------------------------------------------------------------
// column plan: which REE columns exist and how each row's key is derived
static void build_kind_tables(pa_agg* a) {
  // reportTraceEventV2's per-origin constants (reporter/parca_reporter.go:338-363)
  static const char* producer[7] = {"parca_agent", "parca_agent", "parca_agent", "memory", "memory", "memory", "memory"};
  static const char* stype[7] = {"samples", "wallclock", "cuda", "inuse_objects", "inuse_space", "alloc_objects", "alloc_space"};
  static const char* sunit[7] = {"count", "nanoseconds", "nanoseconds", "count", "bytes", "count", "bytes"};
  static const char* ptype[7] = {"cpu", "samples", "cuda", "space", "space", "space", "space"};
  static const char* punit[7] = {"nanoseconds", "count", "nanoseconds", "bytes", "bytes", "bytes", "bytes"};
  static const char* tempo[7] = {"delta", "delta", "delta", nullptr, nullptr, nullptr, nullptr};
  const char* const* tabs[6] = {producer, stype, sunit, ptype, punit, tempo};
  a->kindtab.assign(8 * 8, kNull);
  a->kind_strings.assign(6, {});
  for (int t = 0; t < 6; t++)
    for (int k = 0; k < 7; k++) {
      if (!tabs[t][k]) continue;
      auto& v = a->kind_strings[t];
      auto it = std::find(v.begin(), v.end(), std::string(tabs[t][k]));
      if (it == v.end()) { v.push_back(tabs[t][k]); it = v.end() - 1; }
      a->kindtab[t * 8 + k] = (uint32_t)(it - v.begin());
    }
  const int64_t persec = 1000000000ll / (int64_t)a->cfg.samples_per_second;
  const bool v1 = a->cfg.schema == PA_SCHEMA_V1;  // the v1 writer keeps period = 1e9/Hz for off-CPU and CUDA (parca_reporter.go:289, :322)
  int64_t per[7] = {persec, v1 ? persec : 0, v1 ? persec : 1, 524288, 524288, 524288, 524288};
  uint64_t dur[7] = {1000000000ull, 1000000000ull, 1000000000ull, 0, 0, 0, 0};
  a->period_vals.clear();
  a->duration_vals.clear();
  for (int k = 0; k < 7; k++) {  // equal values share a class: run merging compares values (arrow.go:170-207)
    auto ip = std::find(a->period_vals.begin(), a->period_vals.end(), per[k]);
    if (ip == a->period_vals.end()) { a->period_vals.push_back(per[k]); ip = a->period_vals.end() - 1; }
    a->kindtab[6 * 8 + k] = (uint32_t)(ip - a->period_vals.begin());
    auto id = std::find(a->duration_vals.begin(), a->duration_vals.end(), dur[k]);
    if (id == a->duration_vals.end()) { a->duration_vals.push_back(dur[k]); id = a->duration_vals.end() - 1; }
    a->kindtab[7 * 8 + k] = (uint32_t)(id - a->duration_vals.begin());
  }
}

// cpu / thread_id / thread_name columns of the config; a labelset's pair of the same name never reaches a column when the
// column is on: the per-sample labels.Builder.Set overrides the cached value (:616-625)
static uint32_t sample_label_cols(const pa_agg* a) {
  const uint32_t f = a->cfg.label_flags;
  return !(f & PA_LABEL_DISABLE_CPU) + !(f & PA_LABEL_DISABLE_THREAD_ID) + !(f & PA_LABEL_DISABLE_THREAD_COMM);
}
static bool overridden_name(const pa_agg* a, uint32_t name_cid) {
  const uint32_t f = a->cfg.label_flags, n = a->sp.len(name_cid);
  const char* p = (const char*)a->sp.ptr(name_cid);
  auto is = [&](const char* z) { return n == strlen(z) && !memcmp(p, z, n); };
  return (is("cpu") && !(f & PA_LABEL_DISABLE_CPU)) || (is("thread_id") && !(f & PA_LABEL_DISABLE_THREAD_ID)) ||
         (is("thread_name") && !(f & PA_LABEL_DISABLE_THREAD_COMM));
}
// the label columns take kMaxCols minus the 8 kind-derived columns and v1's two
static bool plan_fits(const pa_agg* a, size_t n_names) { return n_names + sample_label_cols(a) + 10 <= (size_t)kMaxCols; }

// The column plan of a batch: one labelset-derived column per planned name ordinal (ascending), the sample label columns,
// the kind-derived columns. reg_mu held.
static int build_columns(pa_agg* a, const std::vector<uint32_t>& names) {
  if (!plan_fits(a, names.size())) return a->fail(PA_ERANGE, "too many distinct label names in one batch (limit 246)");
  a->cols.clear();
  const uint32_t flags = a->cfg.label_flags;
  for (uint32_t ord : names) {
    ColPlan c;
    const uint32_t cid = a->ls.name_cid[ord];
    c.name.assign((const char*)a->sp.ptr(cid), a->sp.len(cid));
    c.type = COL_LS;
    c.param = (uint32_t)a->cols.size();
    c.ord = ord;
    c.universe = (uint32_t)a->ls.vals[ord].size();
    a->cols.push_back(std::move(c));
  }
  a->n_lscols = (uint32_t)a->cols.size();
  uint64_t d = 0xcbf29ce484222325ull ^ names.size();  // FNV-1a over the ordinals
  for (uint32_t ord : names) d = (d ^ ord) * 0x100000001b3ull;
  a->plan_digest = d;
  auto add = [a](const char* name, uint32_t type, uint32_t universe) { ColPlan c; c.name = name; c.type = type; c.universe = universe; a->cols.push_back(std::move(c)); };
  if (!(flags & PA_LABEL_DISABLE_CPU)) add("cpu", COL_CPU, 65536);
  if (!(flags & PA_LABEL_DISABLE_THREAD_ID)) add("thread_id", COL_TID, 0);
  if (!(flags & PA_LABEL_DISABLE_THREAD_COMM)) add("thread_name", COL_COMM, 0 /* = canonical string count, set per flush */);
  a->n_label_cols = (uint32_t)a->cols.size();
  static const char* fixed[8] = {"producer", "sample_type", "sample_unit", "period_type", "period_unit", "temporality", "period", "duration"};
  for (uint32_t t = 0; t < 8; t++) { ColPlan c; c.name = fixed[t]; c.type = COL_KIND; c.param = t; a->cols.push_back(std::move(c)); }
  if (a->cfg.schema == PA_SCHEMA_V1) {  // v1: stacktrace_id and timestamp are run-end encoded too (arrow.go:395-400, :471-474)
    ColPlan o; o.name = "stacktrace_id"; o.type = COL_ORD; a->cols.push_back(std::move(o));
    ColPlan t; t.name = "timestamp"; t.type = COL_TS; a->cols.push_back(std::move(t));
  }
  return PA_OK;
}

// The predicted plan (reg_mu held, P.n_names snapshotted): the names the previous batch's rows used plus every name registered
// since it was planned; when that does not fit, the previously used names alone; when those do not either, none. A cold
// start (no previous batch, or the previous one failed) has no used names and every name is new. The pass checks the
// prediction on the device and is redone with exactly the used names when it missed one (replan_labels).
static int plan_labels(pa_agg* a) {
  if (a->plan_pending) { a->used_prev.clear(); a->names_planned = 0; }
  std::vector<uint32_t> pred = a->used_prev;
  for (uint32_t o = a->names_planned; o < a->P.n_names; o++) pred.push_back(o);  // (every used ordinal is below names_planned)
  if (!plan_fits(a, pred.size())) pred = plan_fits(a, a->used_prev.size()) ? a->used_prev : std::vector<uint32_t>{};
  a->plan_pending = true;
  return build_columns(a, pred);
}
// The members of a merge group predicted different plans (one of them flushed alone since the last merged batch): every member
// plans cold, which depends on the registrations only, so the columns are the same on every member again (reg_mu not held)
static int plan_cold(pa_agg* a) {
  std::lock_guard<std::mutex> g(a->reg_mu);
  a->plan_pending = true;  // plan_labels then starts from no used names and the first name
  return plan_labels(a);
}
// the names the last pass's rows used, from the bitmap pass_finish read back
static std::vector<uint32_t> used_names(const pa_agg* a) {
  std::vector<uint32_t> v;
  for (uint32_t w = 0; w < (a->P.n_names + 31) / 32; w++)
    for (uint32_t m = a->h_used[w]; m; m &= m - 1) v.push_back(w * 32 + (uint32_t)__builtin_ctz(m));
  return v;
}
// the prediction missed a name: plan exactly the used ones for the redo
static int replan_labels(pa_agg* a) {
  std::lock_guard<std::mutex> g(a->reg_mu);
  a->label_replans++;
  return build_columns(a, used_names(a));
}

// ---------------------------------------------------------------------------------------------
extern "C" {

uint32_t pa_agg_abi_version(void) { return PA_ABI_VERSION; }
const char* pa_agg_last_error(const pa_agg* a) { return a ? a->err.c_str() : "null handle"; }

int pa_agg_create(const pa_agg_config* cfg, pa_agg** out) {
  if (!cfg || !out || cfg->abi_version != PA_ABI_VERSION || cfg->samples_per_second == 0 || cfg->max_samples == 0 || cfg->hash_mode > 1 || cfg->schema > 1 || cfg->ipc_compression > PA_IPC_LZ4_FRAME_GPU ||
      (cfg->frame_id_bytes != 0 && cfg->frame_id_bytes != 4 && cfg->frame_id_bytes != 8)) return PA_EINVAL;
  if ((cfg->flags & PA_CFG_GROUP_STACKS) && !(cfg->flags & PA_CFG_REGISTERED_STACKS)) return PA_EINVAL;
  if ((cfg->flags & PA_CFG_RETIRE_STACKS) && (!(cfg->flags & PA_CFG_REGISTERED_STACKS) || (cfg->flags & PA_CFG_GROUP_STACKS))) return PA_EINVAL;
  if ((cfg->flags & PA_CFG_GROUP_RETIRE) &&
      ((cfg->flags & PA_CFG_RETIRE_STACKS) || !(cfg->flags & PA_CFG_REGISTERED_STACKS) || !(cfg->flags & PA_CFG_GROUP_STACKS))) return PA_EINVAL;
  if (cfg->max_samples > 0x7FFFFFFFull) return PA_ERANGE;  // run ends / ListView offsets are int32
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || cfg->device < 0 || cfg->device >= ndev) return PA_ENODEV;
  if (getenv("PA_BACKTRACE")) { signal(SIGSEGV, fatal_backtrace); signal(SIGABRT, fatal_backtrace); signal(SIGBUS, fatal_backtrace); }
  pa_agg* a = new pa_agg();
  a->cfg = *cfg;
  a->cfg.external_labels = nullptr;
  a->device = cfg->device;
  a->idb = cfg->frame_id_bytes == 4 ? 4u : 8u;
  a->single_ring = (cfg->flags & PA_CFG_SINGLE_RING) != 0;
  a->registered = (cfg->flags & PA_CFG_REGISTERED_STACKS) != 0;
  a->group_stacks = (cfg->flags & PA_CFG_GROUP_STACKS) != 0;
  a->group_retire = (cfg->flags & PA_CFG_GROUP_RETIRE) != 0;
  a->retire = (cfg->flags & PA_CFG_RETIRE_STACKS) != 0 || a->group_retire;
  auto bail = [&](int code) { pa_agg_destroy(a); return code; };
  if (cudaSetDevice(a->device) != cudaSuccess) return bail(PA_ENODEV);
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, a->device) != cudaSuccess) return bail(PA_ENODEV);
  a->sms = prop.multiProcessorCount;
  a->G = a->sms * 4;
  if (a->cfg.chunk_samples == 0) a->cfg.chunk_samples = 1u << 20;
  if (a->cfg.max_frames == 0) a->cfg.max_frames = a->cfg.max_samples * 64;
  for (uint32_t i = 0; i < cfg->n_external_labels; i++) {  // resolved to canonical ids lazily at flush (strings may come later)
    a->external.emplace_back(cfg->external_labels[i].name_sid, cfg->external_labels[i].value_sid);
  }
  if (const char* hv = getenv("PA_HASH_VARIANT")) {
    static const struct { const char* name; int id; } kVariants[] = {{"direct", 0}, {"staged", 1}, {"wide", 2}, {"bulk", 3}, {"bulk6x2", 4}, {"widepf", 5},
                                                                   {"tma", 6}, {"tma12x4", 7}, {"tma24x2", 8}, {"tma12x2r", 9}, {"tma13x2r", 10}, {"tma8x3r", 11}, {"tmag13x2", 12}, {"tmag9x3", 13}, {"tmag6x4", 14}, {"widepf3", 15}, {"widenp", 16}};
    a->hash_variant = pa_agg::kDefaultHashVariant;
    for (auto& v : kVariants) if (strcmp(hv, v.name) == 0) a->hash_variant = v.id;
  }
  if (cudaFuncSetAttribute(k_hash_insert_staged, cudaFuncAttributeMaxDynamicSharedMemorySize, kHashStagedSmem) != cudaSuccess) return bail(PA_EIO);
  if (cudaFuncSetAttribute(k_hash_insert_bulk<4, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(BulkSmem<4, 3>)) != cudaSuccess) return bail(PA_EIO);
  if (cudaFuncSetAttribute(k_hash_insert_tma<16, 3, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TmaSmem<16, 3, 8>)) != cudaSuccess) return bail(PA_EIO);
  if (cudaFuncSetAttribute(k_hash_insert_tma<12, 4, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TmaSmem<12, 4, 8>)) != cudaSuccess) return bail(PA_EIO);
  if (cudaFuncSetAttribute(k_hash_insert_tma<24, 2, 8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TmaSmem<24, 2, 8>)) != cudaSuccess) return bail(PA_EIO);
  if (cudaFuncSetAttribute(k_hash_insert_tma<12, 2, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TmaSmem<12, 2, 16>)) != cudaSuccess) return bail(PA_EIO);
  if (cudaFuncSetAttribute(k_hash_insert_tma<13, 2, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TmaSmem<13, 2, 16>)) != cudaSuccess) return bail(PA_EIO);
  if (cudaFuncSetAttribute(k_hash_insert_tma<8, 3, 16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TmaSmem<8, 3, 16>)) != cudaSuccess) return bail(PA_EIO);
  if (cudaFuncSetAttribute(k_hash_insert_tmag<13, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TmagSmem<13, 2>)) != cudaSuccess) return bail(PA_EIO);
  if (cudaFuncSetAttribute(k_hash_insert_tmag<9, 3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TmagSmem<9, 3>)) != cudaSuccess) return bail(PA_EIO);
  if (cudaFuncSetAttribute(k_hash_insert_tmag<6, 4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TmagSmem<6, 4>)) != cudaSuccess) return bail(PA_EIO);
  if (cudaFuncSetAttribute(k_hash_insert_bulk<6, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(BulkSmem<6, 2>)) != cudaSuccess) return bail(PA_EIO);
  if (cudaStreamCreateWithFlags(&a->s_copy, cudaStreamNonBlocking) != cudaSuccess) return bail(PA_EIO);
  int prio_lo = 0, prio_hi = 0;
  cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi);  // numerically lower = higher priority
  // the compute stream carries the chain of short dependent launches (stack rank, dictionaries): its blocks are scheduled
  // ahead of the label chain's large run-end grids, which fill whatever is left
  if (cudaStreamCreateWithPriority(&a->s_comp, cudaStreamNonBlocking, prio_hi) != cudaSuccess) return bail(PA_EIO);
  if (cudaStreamCreateWithPriority(&a->s_aux, cudaStreamNonBlocking, prio_lo) != cudaSuccess) return bail(PA_EIO);
  if (cudaStreamCreateWithFlags(&a->s_d2h, cudaStreamNonBlocking) != cudaSuccess) return bail(PA_EIO);
  cudaEventCreateWithFlags(&a->ev_hdr_all, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&a->ev_hdr_done, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&a->ev_early, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&a->ev_early_done, cudaEventDisableTiming);
  if (cudaHostAlloc((void**)&a->h_early, sizeof(Counters) + 8 * pa_agg::kEarlyMaxRuns * 4, cudaHostAllocDefault) != cudaSuccess) return bail(PA_ENOMEM);
  if (getenv("PA_NO_EARLY_D2H")) a->early_enabled = false;
  if (getenv("PA_EARLY_D2H_ALWAYS")) a->early_force = true;  // tests: take the early path even when the (tiny) upload is already over
  cudaEventCreateWithFlags(&a->ev_fork, cudaEventDisableTiming);
  cudaEventCreateWithFlags(&a->ev_join, cudaEventDisableTiming);
  if (const char* sv = getenv("PA_SERIAL")) a->serial = sv[0] == '1';
  cudaEventCreate(&a->ev_h2d0);
  cudaEventCreate(&a->ev_h2d1);
  cudaEventCreate(&a->ev_d2h0);
  cudaEventCreate(&a->ev_d2h1);
  for (int t = 0; t < T_COUNT; t++) { cudaEventCreate(&a->tm[t].a); cudaEventCreate(&a->tm[t].b); }
  if (a->registered) { cudaEventCreate(&a->rs_tm.a); cudaEventCreate(&a->rs_tm.b); }
  if (a->cfg.ipc_compression == PA_IPC_LZ4_FRAME_GPU) { cudaEventCreate(&a->ev_lz4p0); cudaEventCreate(&a->ev_lz4p1); }
  const uint64_t N = a->cfg.max_samples, NF = a->cfg.max_frames;
  if (a->idb == 4 && a->hash_variant != 5) a->hash_variant = 2;  // (the tma variants fall through to wide32 in launch_hash)  // the narrow ring is read by the `wide` kernel (widening loads); the other variants take uint64 ids
  for (int r = 0; r < (a->single_ring ? 1 : 2); r++) {
    if (cudaHostAlloc((void**)&a->ring[r].hdr, N * sizeof(pa_sample_hdr), cudaHostAllocDefault) != cudaSuccess) return bail(PA_ENOMEM);
    if (a->registered) continue;  // rows name registered stacks: the ring carries no frame ids
    if (cudaHostAlloc((void**)&a->ring[r].frames, std::max<uint64_t>(NF, 1) * a->idb + 64, cudaHostAllocMapped) != cudaSuccess) return bail(PA_ENOMEM);
    void* dp = nullptr;  // device alias of the pinned frame ring (provided-hash mode gathers unique stacks straight from it)
    if (cudaHostGetDevicePointer(&dp, a->ring[r].frames, 0) != cudaSuccess) return bail(PA_EIO);
    a->ring[r].frames_dev = (const uint64_t*)dp;
  }
  if (cudaHostAlloc((void**)&a->h_ctr_pinned, sizeof(Counters), cudaHostAllocDefault) != cudaSuccess) return bail(PA_ENOMEM);
  bool ok = true;
  auto need = [&](DBuf& b, uint64_t bytes) { ok = ok && b.ensure(std::max<uint64_t>(bytes, 256)) == cudaSuccess; };
  need(a->d_hdr, N * 64);
  if (a->cfg.hash_mode == PA_HASH_XXH64X2 && !a->registered) need(a->d_frames, NF * a->idb + 64);  // provided-hash mode never uploads the frame stream (+ slack: bulk copies round up to 16 B)
  need(a->d_ts, N * 8); need(a->d_value, N * 8); need(a->d_uuid, N * 16); need(a->d_stoff, N * 4); need(a->d_stsize, N * 4);
  need(a->d_slot, N * 4); need(a->d_kind, N); need(a->d_nfr, N * 2); need(a->d_foff, N * 8);
  need(a->d_ls, N * 4); need(a->d_cpu, N * 4); need(a->d_tid, N * 4); need(a->d_comm, N * 4);
  need(a->d_ustream, std::min<uint64_t>(NF, 0x7FFFFFFFull) * 4 + 256);
  need(a->d_uniq_row, N * 4); need(a->d_uniq_count, N * 4);
  need(a->d_ctr, sizeof(Counters));
  need(a->d_partial, (uint64_t)a->G * kMaxCols * 16 + 256);
  need(a->d_partial2, (uint64_t)a->G * kMaxCols * 16 + 256);
  need(a->d_ree_partial, (uint64_t)a->sms * 8 * kWarps * kMaxCols * sizeof(uint32_t) + 256);  // lives across the ranking launches between the two REE passes
  if (a->cfg.schema == PA_SCHEMA_V1) {  // the `stacks` LRU (parca_reporter.go:876): known stacks stay resident in HBM
    a->cid_unknown = a->sp.intern("unknown");
    a->cid_missing = a->sp.intern("missing stacktrace");
    a->store_entries = cfg->stack_cache_entries ? cfg->stack_cache_entries : std::min<uint64_t>(std::max<uint64_t>(65536, N), 1ull << 24);
    if (a->store_entries > (1ull << 28)) return bail(PA_ERANGE);
    // room for the cache's content PLUS one batch's new stacks (fewer than the capacity, or the batch replaces the content): the
    // batch is inserted first and the least recently used entries are evicted afterwards
    a->store_slots = pow2_at_least(4 * a->store_entries);
    a->store_frames = cfg->stack_cache_frames ? cfg->stack_cache_frames : a->store_entries * 128;
    need(a->d_store, (a->store_slots + 2) * sizeof(StoreSlot));
    need(a->d_store_arena, a->store_frames * 4);
    need(a->d_store_ctl, sizeof(StoreCtl));
    need(a->d_store_stamp, (a->store_slots + 2) * 8);
    need(a->d_select, 256 * 4);
    need(a->d_v1_ids, N * 16);
    if (ok) ok = cudaMemset(a->d_store.p, 0, (a->store_slots + 2) * sizeof(StoreSlot)) == cudaSuccess && cudaMemset(a->d_store_ctl.p, 0, sizeof(StoreCtl)) == cudaSuccess &&
                 cudaMemset(a->d_store_stamp.p, 0, (a->store_slots + 2) * 8) == cudaSuccess &&
                 cudaHostAlloc((void**)&a->h_select, 256 * 4 + sizeof(StoreCtl), cudaHostAllocDefault) == cudaSuccess;
  }
  if (!ok) return bail(PA_ENOMEM);
  *out = a;
  return PA_OK;
}

void pa_agg_destroy(pa_agg* a) {
  if (!a) return;
  cudaSetDevice(a->device);
  if (a->s_comp) cudaStreamSynchronize(a->s_comp);
  if (a->s_aux) cudaStreamSynchronize(a->s_aux);
  if (a->s_copy) cudaStreamSynchronize(a->s_copy);
  if (a->s_d2h) cudaStreamSynchronize(a->s_d2h);
  if (a->h_early) cudaFreeHost(a->h_early);
  if (a->h_select) cudaFreeHost(a->h_select);
  for (auto e : a->hash_ev) cudaEventDestroy(e);
  for (cudaEvent_t e : {a->ev_hdr_all, a->ev_hdr_done, a->ev_early, a->ev_early_done}) if (e) cudaEventDestroy(e);
  if (a->s_d2h) cudaStreamDestroy(a->s_d2h);
  for (int r = 0; r < 2; r++) { if (a->ring[r].hdr) cudaFreeHost(a->ring[r].hdr); if (a->ring[r].frames) cudaFreeHost(a->ring[r].frames); }
  if (a->h_ctr_pinned) cudaFreeHost(a->h_ctr_pinned);
  if (a->out) cudaFreeHost(a->out);
  if (a->h_desc) cudaFreeHost(a->h_desc);
  if (a->h_used) cudaFreeHost(a->h_used);
  DBuf* all[] = {&a->d_hdr, &a->d_frames, &a->d_ts, &a->d_value, &a->d_uuid, &a->d_stoff, &a->d_stsize, &a->d_slot, &a->d_kind, &a->d_nfr,
                 &a->d_foff, &a->d_ls, &a->d_cpu, &a->d_tid, &a->d_comm, &a->d_ustream, &a->d_uniq_row, &a->d_uniq_count, &a->d_table, &a->d_ctr,
                 &a->d_arena, &a->d_partial, &a->d_partial2, &a->d_ree_partial, &a->d_kindtab, &a->d_cols, &a->d_jobs,
                 &a->m_addr.buf, &a->m_line.buf, &a->m_type.buf, &a->m_map.buf, &a->m_bid.buf, &a->m_func.buf, &a->m_fnfile.buf, &a->m_sid2cid.buf, &a->m_ls_off.buf, &a->m_ls_pairs.buf,
                 &a->m1_map.buf, &a->m1_bid.buf, &a->m1_fn.buf, &a->m1_file.buf, &a->m1_line.buf, &a->m1_col.buf, &a->m1_complete.buf,
                 &a->d_store, &a->d_store_arena, &a->d_store_ctl, &a->d_v1_ids, &a->d_st1, &a->d_store_stamp, &a->d_v1_last, &a->d_select, &a->d_lz4, &a->d_lz4_body,
                 &a->d_rs_recs, &a->d_rs_last, &a->d_rs_arena[0], &a->d_rs_arena[1], &a->d_rs_tmp, &a->d_rs_upd};
  for (DBuf* b : all) b->release();
  for (auto e : a->chunk_ev) cudaEventDestroy(e);
  if (a->ev_h2d0) cudaEventDestroy(a->ev_h2d0);
  if (a->ev_h2d1) cudaEventDestroy(a->ev_h2d1);
  if (a->ev_d2h0) cudaEventDestroy(a->ev_d2h0);
  if (a->ev_d2h1) cudaEventDestroy(a->ev_d2h1);
  if (a->ev_lz4p0) cudaEventDestroy(a->ev_lz4p0);
  if (a->ev_lz4p1) cudaEventDestroy(a->ev_lz4p1);
  for (int t = 0; t < T_COUNT; t++) { if (a->tm[t].a) cudaEventDestroy(a->tm[t].a); if (a->tm[t].b) cudaEventDestroy(a->tm[t].b); }
  if (a->rs_tm.a) cudaEventDestroy(a->rs_tm.a);
  if (a->rs_tm.b) cudaEventDestroy(a->rs_tm.b);
  if (a->ev_fork) cudaEventDestroy(a->ev_fork);
  if (a->ev_join) cudaEventDestroy(a->ev_join);
  if (a->s_copy) cudaStreamDestroy(a->s_copy);
  if (a->s_comp) cudaStreamDestroy(a->s_comp);
  if (a->s_aux) cudaStreamDestroy(a->s_aux);
  delete a;
}

// ---- registration ---------------------------------------------------------------------------
int pa_agg_register_strings(pa_agg* a, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, uint32_t* first_id) {
  if (!a || (n && !offsets) || (n && !bytes && offsets[n] != 0)) return PA_EINVAL;
  std::lock_guard<std::mutex> g(a->reg_mu);
  if (first_id) *first_id = (uint32_t)a->sp.sid2cid.size();
  for (uint32_t i = 0; i < n; i++) {
    if (offsets[i + 1] < offsets[i]) return a->fail(PA_EINVAL, "string offsets must be non-decreasing");
    a->sp.sid2cid.push_back(a->sp.intern((const char*)bytes + offsets[i], offsets[i + 1] - offsets[i]));
  }
  return PA_OK;
}
int pa_agg_register_frames(pa_agg* a, const pa_frame_desc* descs, uint32_t n, uint64_t* first_frame_id) {
  if (!a || (n && !descs)) return PA_EINVAL;
  std::lock_guard<std::mutex> g(a->reg_mu);
  if (first_frame_id) *first_frame_id = a->ft.count();
  for (uint32_t i = 0; i < n; i++)
    if (!a->ft.resolve(descs[i], a->sp)) return a->fail(PA_EINVAL, "frame refers to an unregistered string id");
  return PA_OK;
}
int pa_agg_register_labelsets(pa_agg* a, const pa_label_pair* pairs, const uint32_t* offsets, uint32_t n, uint32_t* first_id) {
  if (!a || (n && !offsets)) return PA_EINVAL;
  std::lock_guard<std::mutex> g(a->reg_mu);
  if (first_id) *first_id = a->ls.count();
  for (uint32_t i = 0; i < n; i++) {
    std::vector<std::pair<uint32_t, uint32_t>> set;
    for (uint32_t k = offsets[i]; k < offsets[i + 1]; k++) {
      if (pairs[k].name_sid >= a->sp.sid2cid.size() || pairs[k].value_sid >= a->sp.sid2cid.size()) return a->fail(PA_EINVAL, "labelset refers to an unregistered string id");
      uint32_t v = a->sp.sid2cid[pairs[k].value_sid], name = a->sp.sid2cid[pairs[k].name_sid];
      if (v == 0) continue;  // labels.Labels never carries empty values
      if (overridden_name(a, name)) continue;
      set.emplace_back(name, v);
    }
    a->ls.add(set);
  }
  return PA_OK;
}
// Validation shared by both registration calls (a refused call registers nothing). check_stack_args runs before reg_mu is
// taken, check_stack_shape and check_stack_frames under it, with the space checks in between.
static int check_stack_args(pa_agg* a, const uint64_t* hashes, const uint64_t* offsets, uint32_t n, const char* fn) {
  if (!a->registered) return a->fail(PA_EINVAL, (std::string(fn) + " needs an aggregator created with PA_CFG_REGISTERED_STACKS").c_str());
  if (n && !offsets) return PA_EINVAL;
  const bool provided = a->cfg.hash_mode == PA_HASH_PROVIDED;
  if (n && provided && !hashes) return a->fail(PA_EINVAL, "PA_HASH_PROVIDED: register_stacks needs the stack ids (hashes)");
  if (!provided && hashes) return a->fail(PA_EINVAL, "PA_HASH_XXH64X2: the library computes the stack ids (hashes must be NULL)");
  return PA_OK;
}
static int check_stack_shape(pa_agg* a, const uint64_t* frames, const uint64_t* offsets, uint32_t n, uint64_t* total_out) {
  uint64_t total = 0;
  for (uint32_t i = 0; i < n; i++) {
    if (offsets[i + 1] < offsets[i]) return a->fail(PA_EINVAL, "stack offsets must be non-decreasing");
    const uint64_t d = offsets[i + 1] - offsets[i];
    if (d > 0xFFFFu) return a->fail(PA_ERANGE, "stack deeper than 65535 frames");
    total += d;
  }
  if (total && !frames) return PA_EINVAL;
  *total_out = total;
  return PA_OK;
}
static int check_stack_frames(pa_agg* a, const uint64_t* frames, const uint64_t* offsets, uint32_t n) {
  const uint64_t nf_reg = a->ft.count();
  const uint32_t* f32 = (const uint32_t*)frames;
  for (uint32_t i = 0; i < n; i++)
    for (uint64_t j = offsets[i]; j < offsets[i + 1]; j++)
      if ((a->idb == 4 ? (uint64_t)f32[j] : frames[j]) >= nf_reg) return a->fail(PA_EINVAL, "stack refers to an unregistered frame id");
  return PA_OK;
}
// the stack id of stack i: given (PA_HASH_PROVIDED) or, as for a ring row with these frames (DESIGN section 3), XXH64 over the
// ids as little-endian uint64
static void stack_key(const pa_agg* a, const uint64_t* hashes, const uint64_t* frames, const uint64_t* offsets, uint32_t i, RegStack* s, std::vector<uint64_t>& wide) {
  if (a->cfg.hash_mode == PA_HASH_PROVIDED) {
    s->hash_hi = hashes[2 * i];
    s->hash_lo = hashes[2 * i + 1];
    return;
  }
  const uint64_t d = offsets[i + 1] - offsets[i];
  const uint32_t* f32 = (const uint32_t*)frames;
  wide.resize(d);
  for (uint64_t j = 0; j < d; j++) wide[j] = a->idb == 4 ? (uint64_t)f32[offsets[i] + j] : frames[offsets[i] + j];
  s->hash_hi = pa_xxh64(wide.data(), d * 8, 0);
  s->hash_lo = pa_xxh64(wide.data(), d * 8, PA_XXH_SEED_LO);
}

// Both registration calls, after check_stack_args: each stack takes the lowest free slot, or a new one. `handles` (if not null)
// receives generation << 32 | slot for each stack, `first_slot` (if not null) the slot count before the call.
static int register_stacks(pa_agg* a, const uint64_t* hashes, const uint64_t* frames, const uint64_t* offsets, uint32_t n, uint64_t* handles, uint64_t* first_slot) {
  std::lock_guard<std::mutex> g(a->reg_mu);
  uint64_t total = 0;
  int rc;
  if ((rc = check_stack_shape(a, frames, offsets, n, &total))) return rc;
  if (a->rs_frames_live + total > a->cfg.max_frames) return a->fail(PA_ENOSPC, "live registered frames would exceed max_frames");
  if (n > a->rs_free.size() && a->rs_state.size() + (n - a->rs_free.size()) > 0xFFFFFFFFull) return a->fail(PA_ENOSPC, "more than 2^32 - 1 stack slots");
  if ((rc = check_stack_frames(a, frames, offsets, n))) return rc;
  if (first_slot) *first_slot = a->rs_state.size();
  const uint64_t words = a->idb / 4;
  std::vector<uint64_t> wide;
  for (uint32_t i = 0; i < n; i++) {
    const uint64_t d = offsets[i + 1] - offsets[i];
    uint32_t slot;
    if (!a->rs_free.empty()) {  // the lowest free slot
      std::pop_heap(a->rs_free.begin(), a->rs_free.end(), std::greater<uint32_t>());
      slot = a->rs_free.back();
      a->rs_free.pop_back();
    } else {
      slot = (uint32_t)a->rs_state.size();
      a->rs_state.push_back(pa_agg::RS_FREE); a->rs_depth.push_back(0); a->rs_gen.push_back(0);
    }
    RegStack s{};
    s.off = a->rs_pend_frames.size() / words;
    s.depth = (uint32_t)d;
    s.pad = a->rs_gen[slot];
    stack_key(a, hashes, frames, offsets, i, &s, wide);
    a->rs_pend_frames.resize(a->rs_pend_frames.size() + d * words);
    if (d) memcpy(a->rs_pend_frames.data() + s.off * words, (const uint8_t*)frames + offsets[i] * a->idb, d * a->idb);
    a->rs_pend.push_back(s); a->rs_pend_slot.push_back(slot); a->rs_pend_seq.push_back((uint32_t)a->rs_stages);
    a->rs_state[slot] = pa_agg::RS_LIVE; a->rs_depth[slot] = (uint32_t)d;
    a->rs_live++; a->rs_frames_live += d;
    const uint64_t handle = ((uint64_t)a->rs_gen[slot] << 32) | slot;
    if (handles) handles[i] = handle;
    if (a->group_stacks) {  // the registry's digest: XXH64 of (handle, hash_hi, hash_lo, depth, frame ids as uint64), seeded with the digest so far
      wide.resize(d + 4);
      wide[0] = handle; wide[1] = s.hash_hi; wide[2] = s.hash_lo; wide[3] = d;
      for (uint64_t j = 0; j < d; j++) wide[4 + j] = a->idb == 4 ? (uint64_t)((const uint32_t*)frames)[offsets[i] + j] : frames[offsets[i] + j];
      a->reg_digest = pa_xxh64(wide.data(), (d + 4) * 8, a->reg_digest);
    }
  }
  return PA_OK;
}

int pa_agg_register_stacks(pa_agg* a, const uint64_t* hashes, const uint64_t* frames, const uint64_t* offsets, uint32_t n, uint64_t* first_stack_id) {
  if (!a) return PA_EINVAL;
  int rc = check_stack_args(a, hashes, offsets, n, "pa_agg_register_stacks");
  if (rc) return rc;
  if (a->retire) return a->fail(PA_EINVAL, "PA_CFG_RETIRE_STACKS: register through pa_agg_register_stack_handles");
  return register_stacks(a, hashes, frames, offsets, n, nullptr, first_stack_id);  // (no slot is ever freed: the ids are consecutive)
}
int pa_agg_register_stack_handles(pa_agg* a, const uint64_t* hashes, const uint64_t* frames, const uint64_t* offsets, uint32_t n, uint64_t* handles) {
  if (!a || (n && !handles)) return PA_EINVAL;
  int rc = check_stack_args(a, hashes, offsets, n, "pa_agg_register_stack_handles");
  if (rc) return rc;
  return register_stacks(a, hashes, frames, offsets, n, handles, nullptr);
}

// ---- ingest ----------------------------------------------------------------------------------
int pa_agg_acquire(pa_agg* a, uint64_t n_rows, uint64_t n_frames, pa_sample_hdr** hdrs, uint64_t** frames, uint64_t* frame_base) {
  if (!a || !hdrs || !frames) return PA_EINVAL;
  if (a->registered && n_frames) return PA_EINVAL;  // rows name registered stacks (ingest may be concurrent: no error text)
  std::lock_guard<std::mutex> g(a->ring_mu);
  if (a->ring_busy) return PA_ENOSPC;  // single ring: a flush holds the buffer
  pa_agg::Ring& r = a->ring[a->active];
  if (n_rows > a->cfg.max_samples || n_frames > a->cfg.max_frames || r.rows + n_rows > a->cfg.max_samples || r.nfr + n_frames > a->cfg.max_frames) return PA_ENOSPC;
  *hdrs = r.hdr + r.rows;
  *frames = a->registered ? nullptr : (uint64_t*)((uint8_t*)r.frames + r.nfr * a->idb);  // uint32 ids when the ring is narrow
  if (frame_base) *frame_base = r.nfr;
  r.rows += n_rows;
  r.nfr += n_frames;
  a->inflight++;
  return PA_OK;
}
int pa_agg_commit(pa_agg* a, uint64_t) {
  if (!a) return PA_EINVAL;
  std::lock_guard<std::mutex> g(a->ring_mu);
  if (a->inflight > 0) a->inflight--;
  a->ring_cv.notify_all();
  return PA_OK;
}
int pa_agg_submit(pa_agg* a, const pa_sample_hdr* hdrs, const uint64_t* frames, uint64_t n_rows) {
  if (!a || (n_rows && !hdrs)) return PA_EINVAL;
  if (a->registered) {  // frame_off is the caller's stack id: copied as it is
    pa_sample_hdr* dh; uint64_t* df; uint64_t base;
    int rc = pa_agg_acquire(a, n_rows, 0, &dh, &df, &base);
    if (rc) return rc;
    if (n_rows) memcpy(dh, hdrs, n_rows * sizeof(pa_sample_hdr));
    return pa_agg_commit(a, n_rows);
  }
  uint64_t nf = 0;
  for (uint64_t i = 0; i < n_rows; i++) nf += hdrs[i].nframes;
  if (nf && !frames) return PA_EINVAL;
  pa_sample_hdr* dh; uint64_t* df; uint64_t base;
  int rc = pa_agg_acquire(a, n_rows, nf, &dh, &df, &base);
  if (rc) return rc;
  if (n_rows) memcpy(dh, hdrs, n_rows * sizeof(pa_sample_hdr));
  if (nf) memcpy(df, frames, (size_t)nf * a->idb);  // the caller's ids are concatenated in row order, exactly as the ring holds them
  uint64_t off = 0;
  for (uint64_t i = 0; i < n_rows; i++) {
    dh[i].frame_off = base + off;
    off += hdrs[i].nframes;
  }
  return pa_agg_commit(a, n_rows);
}

}  // extern "C"

static int rs_stage(pa_agg* a);
static void release_staged(pa_agg* a);

// ---------------------------------------------------------------------------------------------
// stage: swap ring buffers, start the chunked H2D copies
static int stage_async(pa_agg* a) {
  CK(cudaSetDevice(a->device));
  // the detached ring buffer stays in use until collect() (provided-hash mode reads frames from it in place)
  if (a->staged >= 0) return a->fail(PA_EINVAL, "the previously staged batch has not been collected");
  int buf;
  {
    std::unique_lock<std::mutex> g(a->ring_mu);
    a->ring_cv.wait(g, [a] { return a->inflight == 0; });
    buf = a->active;
    if (a->single_ring) {
      a->ring_busy = true;  // producers get PA_ENOSPC until this batch is collected
    } else {
      a->active ^= 1;
      a->ring[a->active].rows = 0;
      a->ring[a->active].nfr = 0;
    }
  }
  if (a->registered) {
    int rc = rs_stage(a);
    if (rc) { release_staged(a); return rc; }  // (a CUDA failure: the detached batch is dropped)
  }
  pa_agg::Ring& r = a->ring[buf];
  a->staged = buf;
  // (registered stacks: the device arena, set by upload_tables once the batch's registrations are mirrored)
  a->src_frames = a->registered ? nullptr : a->cfg.hash_mode == PA_HASH_PROVIDED ? (const unsigned long long*)r.frames_dev : a->d_frames.as<unsigned long long>();
  a->N = r.rows;
  a->NF = r.nfr;
  a->processed = false;
  a->chunk_rows.clear();
  a->chunk_frames_end.clear();
  const uint64_t C = a->cfg.chunk_samples;
  uint64_t nchunks = (a->N + C - 1) / C;
  while (a->chunk_ev.size() < nchunks) { cudaEvent_t e; CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); a->chunk_ev.push_back(e); }
  CK(cudaEventRecord(a->ev_h2d0, a->s_copy));
  if (a->early.issued) CK(cudaStreamSynchronize(a->s_d2h));  // a batch that was discarded or failed after its early copies were started
  a->early = pa_agg::Early{};
  // headers first when the frame ids take several chunks: everything that depends only on the headers (k_header, the label chain,
  // the early copy-out) then overlaps the upload of the ids
  // (the compressed stream's layout is only known once its bodies are encoded: PA_IPC_LZ4_FRAME_GPU has no early copy-out)
  const bool upload_ids = a->cfg.hash_mode == PA_HASH_XXH64X2 && !a->registered;
  a->early.hdr_first = a->early_enabled && a->cfg.ipc_compression != PA_IPC_LZ4_FRAME_GPU && nchunks > 1 && upload_ids && a->cfg.schema != PA_SCHEMA_V1 && !a->serial;
  if (a->early.hdr_first) {
    CK(cudaMemcpyAsync(a->d_hdr.p, r.hdr, a->N * 64, cudaMemcpyHostToDevice, a->s_copy));
    CK(cudaEventRecord(a->ev_hdr_all, a->s_copy));
    while (a->hash_ev.size() < nchunks) { cudaEvent_t e; CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming)); a->hash_ev.push_back(e); }
  }
  uint64_t fdone = 0;
  for (uint64_t k = 0; k < nchunks; k++) {
    uint64_t r0 = k * C, r1 = std::min(a->N, r0 + C);
    // frames are laid out in row order (acquire hands out ascending frame_base): a chunk's frames end where the next chunk's begin
    uint64_t fend = (r1 < a->N && !a->registered) ? std::min<uint64_t>(r.hdr[r1].frame_off, a->NF) : a->NF;
    if (fend < fdone) fend = fdone;
    if (!a->early.hdr_first) CK(cudaMemcpyAsync(a->d_hdr.as<uint8_t>() + r0 * 64, r.hdr + r0, (r1 - r0) * 64, cudaMemcpyHostToDevice, a->s_copy));
    // The stack id arrives with the sample in PA_HASH_PROVIDED mode (the reference's dataflow, parca_reporter.go:224):
    // frames are only needed for each stack's FIRST occurrence, so nothing is uploaded here and k_gather_unique
    // reads those few stacks from the mapped pinned ring over PCIe (U*F*8 bytes instead of N*F*8).
    // Registered stacks: the ring holds headers only; the frames are in the device arena already.
    if (fend > fdone && upload_ids)
      CK(cudaMemcpyAsync(a->d_frames.as<uint8_t>() + fdone * a->idb, (const uint8_t*)r.frames + fdone * a->idb, (fend - fdone) * a->idb, cudaMemcpyHostToDevice, a->s_copy));
    fdone = fend;
    CK(cudaEventRecord(a->chunk_ev[k], a->s_copy));
    a->chunk_rows.emplace_back(r0, r1);
    a->chunk_frames_end.push_back(fend);
  }
  CK(cudaEventRecord(a->ev_h2d1, a->s_copy));
  return PA_OK;
}

// the staged batch is done with (collected, discarded or failed): the ring buffer it held is free again
static void release_staged(pa_agg* a) {
  a->staged = -1;
  if (a->ring_busy) {
    std::lock_guard<std::mutex> g(a->ring_mu);
    a->ring[0].rows = 0;
    a->ring[0].nfr = 0;
    a->ring_busy = false;
  }
}

template <class F>
static void launch_scan(pa_agg* a, F f, int njobs, Timer& t, int gx, cudaStream_t s, DBuf& scratch) {
  if (gx <= 0) gx = a->G;
  dim3 grid(gx, njobs);
  typename F::T* partial = scratch.as<typename F::T>();  // per-block totals: two concurrent scans need two scratch buffers
  k_scan_reduce<F><<<grid, kThreads, 0, s>>>(f, partial);
  k_scan_emit<F><<<grid, kThreads, 0, s>>>(f, partial);
  t.launches += 2;
}
// grid for a pass over at most `bound` elements: >= 2048 elements per CTA, never more than the full grid
static int small_grid(const pa_agg* a, uint64_t bound) { return (int)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)a->G, (bound + 2047) / 2048)); }

// PA_CFG_REGISTERED_STACKS, under reg_mu, on the compute stream: applies `frees` (records with kStackFree, for free_slots),
// compacts the arena when the dead frames outweigh the live ones (at a stage only: no batch is resident then) or when the
// pending frames would not fit (a regrow, before the pass that reads the records), then uploads the pending registrations.
static int rs_upload(pa_agg* a, const std::vector<RegStack>& frees, const std::vector<uint32_t>& free_slots, bool at_stage) {
  cudaStream_t s = a->s_comp;
  const uint64_t words = a->idb / 4, n_slots = a->rs_state.size();
  if (n_slots * sizeof(RegStack) > a->d_rs_recs.cap) {  // more slots than the device arrays hold: regrow them
    DBuf nr, nl;
    const size_t want = std::max<size_t>(2 * n_slots, 1024);
    CK(nr.ensure(want * sizeof(RegStack)));
    CK(nl.ensure(want * 4));
    if (a->rs_dev_slots) {
      CK(cudaMemcpyAsync(nr.p, a->d_rs_recs.p, a->rs_dev_slots * sizeof(RegStack), cudaMemcpyDeviceToDevice, s));
      CK(cudaMemcpyAsync(nl.p, a->d_rs_last.p, a->rs_dev_slots * 4, cudaMemcpyDeviceToDevice, s));
    }
    CK(cudaStreamSynchronize(s));
    a->d_rs_recs.release(); a->d_rs_last.release();
    a->d_rs_recs = nr; a->d_rs_last = nl;
  }
  RegStack* recs = a->d_rs_recs.as<RegStack>();
  uint32_t* last = a->d_rs_last.as<uint32_t>();
  // the record updates go up in one copy: [records][slots][seqs], frees first
  const uint64_t nf = frees.size(), nr = a->rs_pend.size(), nu = nf + nr;
  RegStack* du = nullptr;
  uint32_t *dslot = nullptr, *dseq = nullptr;
  if (nu) {
    std::vector<uint8_t> up(nu * (sizeof(RegStack) + 8));
    RegStack* hu = (RegStack*)up.data();
    uint32_t* hslot = (uint32_t*)(hu + nu);
    uint32_t* hseq = hslot + nu;
    std::copy(frees.begin(), frees.end(), hu); std::copy(a->rs_pend.begin(), a->rs_pend.end(), hu + nf);
    std::copy(free_slots.begin(), free_slots.end(), hslot); std::copy(a->rs_pend_slot.begin(), a->rs_pend_slot.end(), hslot + nf);
    std::fill(hseq, hseq + nf, 0u); std::copy(a->rs_pend_seq.begin(), a->rs_pend_seq.end(), hseq + nf);
    CK(a->d_rs_upd.ensure(up.size()));
    CK(cudaMemcpyAsync(a->d_rs_upd.p, up.data(), up.size(), cudaMemcpyHostToDevice, s));  // (pageable: the source is consumed on return)
    du = a->d_rs_upd.as<RegStack>(); dslot = (uint32_t*)(du + nu); dseq = dslot + nu;
  }
  if (nf) k_stack_scatter<<<small_grid(a, nf), kThreads, 0, s>>>(du, dslot, dseq, (uint32_t)nf, 0ull, recs, last);
  const uint64_t pend = a->rs_pend_frames.size() / words;
  const uint64_t cap = a->d_rs_arena[a->rs_cur].cap / a->idb, live_dev = a->rs_dev_len - a->rs_frames_dead;
  const bool grow = a->rs_dev_len + pend > cap;
  if (grow || (at_stage && a->rs_frames_dead > live_dev)) {
    DBuf& dst = a->d_rs_arena[a->rs_cur ^ 1];
    CK(dst.ensure(std::max<uint64_t>(grow ? 2 * (live_dev + pend) : cap, 1024) * a->idb));
    if (a->rs_dev_slots) {
      const uint32_t ns = (uint32_t)a->rs_dev_slots;
      const uint64_t max_chunks = ns + live_dev / kCompactChunk + 1;
      CK(a->d_rs_tmp.ensure(ns * 8 + max_chunks * 8 + 64));
      unsigned long long* new_off = a->d_rs_tmp.as<unsigned long long>();
      uint2* chunks = (uint2*)(new_off + ns);
      Pair* total = (Pair*)(chunks + max_chunks);
      a->rs_tm.launches = 0;
      CK(cudaEventRecord(a->rs_tm.a, s));
      launch_scan(a, StackLiveF{recs, ns, new_off, chunks, total}, 1, a->rs_tm, small_grid(a, ns), s, a->d_partial);
      k_stack_compact_copy<<<a->G, kThreads, 0, s>>>(total, chunks, recs, new_off, (uint32_t)words, a->d_rs_arena[a->rs_cur].as<uint32_t>(), dst.as<uint32_t>());
      k_stack_rebase<<<small_grid(a, ns), kThreads, 0, s>>>(recs, ns, new_off);
      a->rs_tm.launches += 2;
      CK(cudaEventRecord(a->rs_tm.b, s));
      CK(cudaEventSynchronize(a->rs_tm.b));
      float ms = 0;
      cudaEventElapsedTime(&ms, a->rs_tm.a, a->rs_tm.b);
      a->rs_tm.ms = ms;
      a->rs_compactions++;
    }
    a->rs_cur ^= 1;
    a->rs_dev_len = live_dev;
    a->rs_frames_dead = 0;
  }
  if (nr) {
    if (pend) CK(cudaMemcpyAsync(a->d_rs_arena[a->rs_cur].as<uint32_t>() + a->rs_dev_len * words, a->rs_pend_frames.data(), pend * a->idb, cudaMemcpyHostToDevice, s));
    k_stack_scatter<<<small_grid(a, nr), kThreads, 0, s>>>(du + nf, dslot + nf, dseq + nf, (uint32_t)nr, a->rs_dev_len, recs, last);
    a->rs_dev_len += pend;
    a->rs_pend.clear(); a->rs_pend_slot.clear(); a->rs_pend_seq.clear(); a->rs_pend_frames.clear();
  }
  CK(cudaGetLastError());
  // A grow leaves the old arena allocated as the next compaction's target. A registry that never frees a slot never compacts,
  // so it releases that arena after a grow, and the upload and compaction scratch the grown burst sized.
  if (grow && !a->retire) {
    CK(cudaStreamSynchronize(s));
    a->d_rs_arena[a->rs_cur ^ 1].release(); a->d_rs_tmp.release(); a->d_rs_upd.release();
  }
  a->rs_dev_slots = n_slots;
  a->src_frames = (const unsigned long long*)a->d_rs_arena[a->rs_cur].p;
  a->P.n_stacks = (uint32_t)n_slots;
  a->P.n_stack_frames = a->rs_dev_len;
  const uint64_t digests[2] = {a->reg_digest, a->retire_digest};
  a->P.stack_digest = pa_xxh64(digests, sizeof digests, 0);
  a->P.stack_frames_live = a->rs_frames_live;  // (nothing is pending now: these are the uploaded stacks not yet freed)
  return PA_OK;
}

// A new batch is staged: the stacks whose grace batch this is not (retired before the previous stage) are freed.
static int rs_stage(pa_agg* a) {
  std::lock_guard<std::mutex> g(a->reg_mu);
  a->rs_stages++;
  std::vector<RegStack> frees;
  std::vector<uint32_t> slots;
  size_t keep = 0;
  for (const auto& e : a->rs_retiring) {
    if (e.second > a->rs_stages) { a->rs_retiring[keep++] = e; continue; }
    const uint32_t slot = e.first, d = a->rs_depth[slot];
    a->rs_state[slot] = pa_agg::RS_FREE;
    a->rs_live--; a->rs_frames_live -= d; a->rs_frames_dead += d;
    RegStack r{};
    r.pad = kStackFree | ++a->rs_gen[slot];
    frees.push_back(r); slots.push_back(slot);
    if (a->rs_gen[slot] < kStackFree) {  // (a slot whose 31-bit generation is spent stays free for good)
      a->rs_free.push_back(slot);
      std::push_heap(a->rs_free.begin(), a->rs_free.end(), std::greater<uint32_t>());
    }
  }
  a->rs_retiring.resize(keep);
  return rs_upload(a, frees, slots, true);
}

// plan_batch: a pass follows, which takes the label column plan predicted here (pa_agg_stacktraces only needs the mirrors)
static int upload_tables(pa_agg* a, bool plan_batch) {
  std::lock_guard<std::mutex> g(a->reg_mu);
  cudaStream_t s = a->s_comp;
  CK(a->m_addr.sync(a->ft.addr, s)); CK(a->m_line.sync(a->ft.line, s)); CK(a->m_type.sync(a->ft.type_cid, s));
  CK(a->m_map.sync(a->ft.map_cid, s)); CK(a->m_bid.sync(a->ft.bid_cid, s)); CK(a->m_func.sync(a->ft.func, s));
  CK(a->m_fnfile.sync(a->ft.fn_file_cid, s)); CK(a->m_sid2cid.sync(a->sp.sid2cid, s));
  if (a->cfg.schema == PA_SCHEMA_V1) {
    CK(a->m1_map.sync(a->ft.v1_map_cid, s)); CK(a->m1_bid.sync(a->ft.v1_bid_cid, s)); CK(a->m1_fn.sync(a->ft.v1_fn_cid, s));
    CK(a->m1_file.sync(a->ft.v1_file_cid, s)); CK(a->m1_line.sync(a->ft.v1_line, s)); CK(a->m1_col.sync(a->ft.v1_col, s));
    CK(a->m1_complete.sync(a->ft.v1_complete, s));
  }
  if (a->registered) {
    int rc = rs_upload(a, {}, {}, false);
    if (rc) return rc;
  }
  CK(a->m_ls_off.sync(a->ls.off, s)); CK(a->m_ls_pairs.sync(a->ls.pairs, s));
  // what the device mirrors now hold: the pass uses these counts only (registration may continue concurrently)
  a->P.n_cstr = a->sp.count(); a->P.n_frames = a->ft.count(); a->P.n_funcs = a->ft.n_funcs();
  a->P.n_sids = (uint32_t)a->sp.sid2cid.size(); a->P.n_labelsets = a->ls.count(); a->P.n_names = a->ls.n_names();
  if (!a->d_kindtab.p) {
    build_kind_tables(a);
    CK(a->d_kindtab.ensure(a->kindtab.size() * 4));
    CK(cudaMemcpyAsync(a->d_kindtab.p, a->kindtab.data(), a->kindtab.size() * 4, cudaMemcpyHostToDevice, s));
  }
  return plan_batch ? plan_labels(a) : PA_OK;
}

// first-occurrence ranking of a batch of FoJobs (blockIdx.y = job). elem_bound: upper bound on elements per job;
// table_bound: on table entries; both pick right-sized grids
static void run_fo_jobs(pa_agg* a, const FoJob* djobs, int first, int count, bool need_min, Timer& t, uint64_t elem_bound, uint64_t table_bound,
                        bool do_map, cudaStream_t s, DBuf& scratch) {
  const int ge = small_grid(a, elem_bound), gt = small_grid(a, table_bound), gw = small_grid(a, elem_bound / 32 + 1);
  k_fo_zero<<<dim3(gw, count), kThreads, 0, s>>>(djobs + first);
  if (need_min) { k_fo_min<<<dim3(ge, count), kThreads, 0, s>>>(djobs + first); t.launches++; }
  k_fo_bits<<<dim3(gt, count), kThreads, 0, s>>>(djobs + first);
  launch_scan(a, FoWordsF{djobs + first, -1}, count, t, gw, s, scratch);
  k_fo_assign<<<dim3(gt, count), kThreads, 0, s>>>(djobs + first);
  if (do_map) { k_fo_map<<<dim3(ge, count), kThreads, 0, s>>>(djobs + first); t.launches++; }
  t.launches += 3;
}

// descriptor tables go up from pinned staging: a pageable cudaMemcpyAsync would synchronise the stream in the
// middle of the pipeline and leave the tail launch-bound
static int upload_descriptors(pa_agg* a, const void* jobs, size_t jb, const void* cols, size_t cb) {
  if (jb + cb > a->h_desc_cap) {
    if (a->h_desc) cudaFreeHost(a->h_desc);
    a->h_desc = nullptr;
    a->h_desc_cap = 0;
    CK(cudaHostAlloc((void**)&a->h_desc, (jb + cb) * 2, cudaHostAllocDefault));
    a->h_desc_cap = (jb + cb) * 2;
  }
  memcpy(a->h_desc, jobs, jb);
  if (cb) memcpy(a->h_desc + jb, cols, cb);
  CK(a->d_jobs.ensure(std::max<size_t>(jb, 256)));
  CK(a->d_cols.ensure(std::max<size_t>(cb, 256)));
  CK(cudaMemcpyAsync(a->d_jobs.p, a->h_desc, jb, cudaMemcpyHostToDevice, a->s_comp));
  if (cb) CK(cudaMemcpyAsync(a->d_cols.p, a->h_desc + jb, cb, cudaMemcpyHostToDevice, a->s_comp));
  return PA_OK;
}

// v1: the batch's accesses to the `stacks` LRU (parca_reporter.go:224-227): every unique stack of the batch is looked up and, if
// unknown, added; known ones (evicted ones included) get the batch's access time
static StoreInsertArgs store_insert_args(pa_agg* a, uint32_t min_last_p1) {
  StoreInsertArgs sa{};
  Counters* ctr = a->d_ctr.as<Counters>();
  sa.ctr = ctr; sa.uniq_row = a->d_uniq_row.as<uint32_t>(); sa.slot_of_row = a->d_slot.as<uint32_t>(); sa.tab = a->d_table.as<StackSlot>();
  sa.nframes = a->d_nfr.as<uint16_t>(); sa.frame_off = a->d_foff.as<unsigned long long>();
  sa.frames = a->src_frames;
  sa.narrow = a->idb == 4 ? 1u : 0u;
  sa.n_frames_registered = a->P.n_frames;
  sa.st = a->d_store.as<StoreSlot>(); sa.mask = (uint32_t)(a->store_slots - 1); sa.arena = a->d_store_arena.as<uint32_t>();
  sa.cap_frames = a->store_frames; sa.cap_entries = (uint32_t)(a->store_slots - a->store_slots / 4); sa.ctl = a->d_store_ctl.as<StoreCtl>(); sa.ctr_w = ctr;
  sa.stamp = a->d_store_stamp.as<unsigned long long>(); sa.last_row = a->d_v1_last.as<uint32_t>();
  sa.epoch_hi = a->store_epoch << 32; sa.min_last_p1 = min_last_p1;
  return sa;
}
static void launch_store_insert(pa_agg* a, uint32_t min_last_p1) { k_store_insert<false><<<a->G, kThreads, 0, a->s_comp>>>(store_insert_args(a, min_last_p1)); }
// the k-th largest of the non-zero keys (k >= 1, at least k of them exist): eight histogram passes from the top byte down
static int select_kth_largest(pa_agg* a, const unsigned long long* keys, uint64_t n, uint64_t k, unsigned long long* out) {
  cudaStream_t s = a->s_comp;
  unsigned long long prefix = 0;
  for (int shift = 56; shift >= 0; shift -= 8) {
    CK(cudaMemsetAsync(a->d_select.p, 0, 256 * 4, s));
    k_select_hist<<<small_grid(a, n), kThreads, 0, s>>>(keys, n, prefix, shift, a->d_select.as<uint32_t>());
    CK(cudaMemcpyAsync(a->h_select, a->d_select.p, 256 * 4, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    int b = 255;
    for (; b > 0; b--) {
      if (a->h_select[b] >= k) break;
      k -= a->h_select[b];
    }
    prefix |= (unsigned long long)b << shift;
  }
  *out = prefix;
  return PA_OK;
}
static int store_ctl_read(pa_agg* a, StoreCtl* out) {
  CK(cudaMemcpyAsync(a->h_select + 256, a->d_store_ctl.p, sizeof(StoreCtl), cudaMemcpyDeviceToHost, a->s_comp));
  CK(cudaStreamSynchronize(a->s_comp));
  memcpy(out, a->h_select + 256, sizeof(StoreCtl));
  return PA_OK;
}
static int store_clear(pa_agg* a) {
  CK(cudaMemsetAsync(a->d_store.p, 0, (a->store_slots + 2) * sizeof(StoreSlot), a->s_comp));
  CK(cudaMemsetAsync(a->d_store_stamp.p, 0, (a->store_slots + 2) * 8, a->s_comp));
  CK(cudaMemsetAsync(a->d_store_ctl.p, 0, sizeof(StoreCtl), a->s_comp));
  return PA_OK;
}
// compaction: evicted entries give their slots and frames back (the live ones move to a fresh table and arena)
static int store_compact(pa_agg* a) {
  cudaStream_t s = a->s_comp;
  DBuf st2, stamp2, arena2;
  CK(st2.ensure((a->store_slots + 2) * sizeof(StoreSlot)));
  CK(stamp2.ensure((a->store_slots + 2) * 8));
  CK(arena2.ensure(a->store_frames * 4));
  CK(cudaMemsetAsync(st2.p, 0, (a->store_slots + 2) * sizeof(StoreSlot), s));
  CK(cudaMemsetAsync(stamp2.p, 0, (a->store_slots + 2) * 8, s));
  CK(cudaMemsetAsync(a->d_store_ctl.p, 0, sizeof(StoreCtl), s));
  StoreRebuildArgs ra{};
  ra.old_st = a->d_store.as<StoreSlot>(); ra.old_stamp = a->d_store_stamp.as<unsigned long long>(); ra.old_arena = a->d_store_arena.as<uint32_t>();
  ra.old_mask = (uint32_t)(a->store_slots - 1);
  ra.st = st2.as<StoreSlot>(); ra.stamp = stamp2.as<unsigned long long>(); ra.arena = arena2.as<uint32_t>(); ra.mask = ra.old_mask; ra.ctl = a->d_store_ctl.as<StoreCtl>();
  k_store_rebuild<<<small_grid(a, a->store_slots * 32), kThreads, 0, s>>>(ra);
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  std::swap(a->d_store, st2); std::swap(a->d_store_stamp, stamp2); std::swap(a->d_store_arena, arena2);
  st2.release(); stamp2.release(); arena2.release();
  a->store_compactions++;
  return PA_OK;
}
// One batch's worth of LRU traffic, after the pass has ranked the batch's unique stacks (a->h_ctr is current).
static int v1_store_update(pa_agg* a) {
  cudaStream_t s = a->s_comp;
  const uint64_t U = a->h_ctr.n_unique, C = a->store_entries, N = a->N;
  Counters* ctr = a->d_ctr.as<Counters>();
  a->store_epoch++;
  if (a->store_epoch >= (1ull << 32)) return a->fail(PA_ERANGE, "stack store: access clock overflow");
  CK(a->d_v1_last.ensure((a->table_cap + 2) * 4));
  CK(cudaMemsetAsync(a->d_v1_last.p, 0, (a->table_cap + 2) * 4, s));
  k_last_rows<<<a->G, kThreads, 0, s>>>((uint32_t)N, a->d_slot.as<uint32_t>(), a->d_v1_last.as<uint32_t>());
  uint32_t min_last_p1 = 0;
  StoreCtl ctl{};
  int rc;
  if (U >= C) {
    // the batch alone touches at least as many stacks as the cache holds: afterwards it holds exactly the C of them seen last
    DBuf tmp;
    CK(tmp.ensure(U * 8));
    k_batch_stamps<<<small_grid(a, U), kThreads, 0, s>>>(ctr, a->d_uniq_row.as<uint32_t>(), a->d_slot.as<uint32_t>(), a->d_v1_last.as<uint32_t>(), tmp.as<unsigned long long>());
    unsigned long long t = 0;
    if ((rc = select_kth_largest(a, tmp.as<unsigned long long>(), U, C, &t))) return rc;
    tmp.release();
    min_last_p1 = (uint32_t)t;
    if ((rc = store_clear(a))) return rc;
    a->store_evictions++;
  } else {
    if ((rc = store_ctl_read(a, &ctl))) return rc;
    const uint64_t phys = a->store_slots - a->store_slots / 4;
    if (ctl.entries > ctl.live && (ctl.entries + U > phys || ctl.used_frames + a->h_ctr.n_indices64 > a->store_frames) && (rc = store_compact(a))) return rc;
  }
  bool cleared = U >= C;
  for (int attempt = 0; attempt < 3; attempt++) {
    CK(cudaMemsetAsync(&ctr->store_overflow, 0, 4, s));
    launch_store_insert(a, min_last_p1);
    CK(cudaMemcpyAsync(a->h_ctr_pinned, ctr, sizeof(Counters), cudaMemcpyDeviceToHost, s));
    if ((rc = store_ctl_read(a, &ctl))) return rc;
    CK(cudaGetLastError());
    a->h_ctr.err |= a->h_ctr_pinned->err;
    if (!a->h_ctr_pinned->store_overflow || attempt == 2) break;  // (third time: whatever still does not fit stays marked as dropped)
    // out of slots or of frame space: first give back what evicted entries hold; if that is not enough, start over with this
    // batch only (the frame arena is this library's limit, not the reference's: DESIGN section 5a)
    if (ctl.entries > ctl.live && !cleared && attempt == 0) {
      if ((rc = store_compact(a))) return rc;
    } else {
      if ((rc = store_clear(a))) return rc;
      cleared = true;
      a->store_evictions++;
    }
  }
  if (ctl.live > C) {  // evict everything but the C entries accessed last
    unsigned long long t = 0;
    if ((rc = select_kth_largest(a, a->d_store_stamp.as<unsigned long long>(), a->store_slots + 2, C, &t))) return rc;
    k_store_kill<<<small_grid(a, a->store_slots + 2), kThreads, 0, s>>>(a->d_store_stamp.as<unsigned long long>(), a->store_slots + 2, t, a->d_store_ctl.as<StoreCtl>());
    CK(cudaStreamSynchronize(s));
    CK(cudaGetLastError());
    a->store_evictions++;
  }
  return PA_OK;
}

// ---------------------------------------------------------------------------------------------
// The per-interval pass, in stages. A single aggregator runs them back to back (process_once); a group of shard
// aggregators that builds ONE merged record (mode B, merge_impl.hpp) runs the same stages with its exchanges in between.
// Upper bound on distinct keys used to size an open-address table: small batches take their row count; large ones take
// 4x what the previous interval saw, and a cold start assumes one distinct key per 16 rows (a 10M-row batch then starts
// with a 64 MB table instead of 1 GB). A wrong guess costs a redo of the pass with a 4x larger table (ERR_TABLE_FULL).
static uint64_t table_bound(uint64_t n, uint64_t prev, uint64_t big, uint64_t floor_) {
  if (n <= big) return n;
  return std::min<uint64_t>(n, std::max<uint64_t>(prev ? prev * 4 : n / 16, floor_));
}

// sizes, arena layout, job / column descriptor tables for the staged batch. md != nullptr: this aggregator is shard
// md->rank of a merged batch (row-indexed bitmaps and dictionary tables are sized for the whole batch)
static int pass_plan(pa_agg* a, const MergeDims* md) {
  Pass& P = a->P;
  const uint64_t N = a->N;
  P.N = N;
  P.merged = md != nullptr;
  P.row_base = md ? md->row_base : 0;
  P.NT = md ? md->n_total : N;
  P.world = md ? md->world : 1;
  P.rank = md ? md->rank : 0;
  P.ncols = (uint32_t)a->cols.size();
  P.nlab = a->n_label_cols;
  P.v1 = a->cfg.schema == PA_SCHEMA_V1;
  P.provided = a->cfg.hash_mode == PA_HASH_PROVIDED || a->registered;
  const uint32_t ncols = P.ncols, nlab = P.nlab;
  const bool v1 = P.v1;

  // ---- stack table capacity: 2x an upper bound on this batch's unique stacks (adaptive, retried on overflow)
  uint64_t bound = table_bound(N, a->prev_unique, 1u << 20, 1u << 18);
  uint64_t cap = std::max<uint64_t>(pow2_at_least(2 * std::max<uint64_t>(bound, 1)), 1024);
  if (cap < a->retry_cap) cap = a->retry_cap;
  if (cap > (1ull << 31)) cap = 1ull << 31;  // slot index mask+1 must stay below 2^32
  a->table_cap = cap;
  P.cap = cap;
  P.mask = (uint32_t)(cap - 1);
  CK(a->d_table.ensure((cap + 2) * sizeof(StackSlot)));
  // thread_id dictionary table (hashed): same policy; a merged batch holds every shard's thread ids
  uint64_t tbound = table_bound(P.NT, a->prev_tids, 1u << 18, 1u << 16);
  uint64_t tcap = std::max<uint64_t>(pow2_at_least(2 * std::max<uint64_t>(tbound, 16)), 1024);
  if (tcap < a->retry_tcap) tcap = a->retry_tcap;
  if (tcap > (1ull << 31)) tcap = 1ull << 31;
  a->tid_cap = tcap;
  a->tid_mask = (uint32_t)(tcap - 1);
  P.tcap = tcap;

  // ---- arena: per-flush scratch and small output buffers; three classes (0xFF / zero / uninitialised)
  struct Req { void** pp; size_t bytes; int cls; };
  std::vector<Req> reqs;
  auto want = [&reqs](auto** pp, size_t bytes, int cls = 2) { reqs.push_back(Req{(void**)pp, (bytes + 255) & ~(size_t)255, cls}); };
  const size_t Pn = std::max<uint32_t>(P.n_frames, 1), S = std::max<uint32_t>(P.n_cstr, 1), FN = std::max<uint32_t>(P.n_funcs, 1);
  // (registered stacks: the unique stacks' frames are a subset of the arena's, as in the ring they are of the batch's)
  const uint64_t nf_all = md ? md->nf_total : a->registered ? P.n_stack_frames : a->NF;
  const size_t NI = (size_t)std::min<uint64_t>(std::max<uint64_t>(nf_all, 1), 0x7FFFFFFFull);
  const size_t Nn = (size_t)std::max<uint64_t>(N, 1), NTn = (size_t)std::max<uint64_t>(P.NT, 1);
  P.Pn = Pn; P.S = S; P.FN = FN; P.NI = NI;
  // direct first-row tables that a merged batch all-reduces (min) in one go: [labelset | cpu | comm], contiguous
  uint32_t *first_cpu = nullptr, *first_comm = nullptr;
  bool has_cpu = false, has_comm = false;
  for (uint32_t c = 0; c < nlab; c++) { has_cpu |= a->cols[c].type == COL_CPU; has_comm |= a->cols[c].type == COL_COMM; }
  want(&P.first_ls, std::max<size_t>(P.n_labelsets, 1) * 4, 0);
  if (has_cpu) want(&first_cpu, 65536 * 4, 0);
  if (has_comm) want(&first_comm, S * 4, 0);
  if (v1) want(&a->v1_first_kind, 8 * 4, 0);  // (a merged batch takes the minimum over the shards: the kind columns' dictionary order)
  size_t red_bytes = 0;
  for (auto& r : reqs) red_bytes += r.bytes;
  // the label column plan check: the key matrix has one row per labelset the (merged) batch names, at most one per row
  P.ls_rank = P.ls_keys = P.ls_used = P.used_names = nullptr;
  if (P.n_names) {
    const size_t used_words = (P.n_names + 31) / 32;
    want(&P.ls_rank, (size_t)P.n_labelsets * 4);
    want(&P.ls_keys, std::max<size_t>((size_t)std::min<uint64_t>(P.n_labelsets, NTn) * a->n_lscols, 1) * 4);
    want(&P.ls_used, 4, 1); want(&P.used_names, used_words * 4, 1);
    if (used_words > a->h_used_words) {
      if (a->h_used) cudaFreeHost(a->h_used);
      a->h_used = nullptr;
      a->h_used_words = 0;
      CK(cudaHostAlloc((void**)&a->h_used, used_words * 2 * 4, cudaHostAllocDefault));
      a->h_used_words = used_words * 2;
    }
  }
  if (v1) {
    want(&a->v1_ord, Nn * 4); want(&a->v1_ts_vals, Nn * 8); want(&a->v1_id_off, (Nn + 1) * 4);
    a->v1_ids = a->d_v1_ids.as<uint8_t>();  // outlives the arena: pa_agg_last_stack_ids / pa_agg_stacktraces run after the flush
    want(&a->v1_kindrank, 64 * 4); want(&a->v1_kind_order, 64 * 4); want(&a->v1_n_kind_dict, 8 * 4);
  }
  want(&P.rowbits, (NTn / 32 + 2) * 4, 1); want(&P.row_wprefix, (NTn / 32 + 2) * 4);
  if (!md) { want(&P.uniq_slot, Nn * 4); want(&P.uniq_size, Nn * 4); }  // merged: sized by the merged dictionary (merge_impl.hpp)
  want(&P.claimed, Nn * 4);
  want(&a->loc_first, Pn * 4, 0); want(&a->loc_rank, Pn * 4); want(&a->loc_order, Pn * 4);
  want(&P.loc_bits, (NI / 32 + 2) * 4); want(&P.loc_wp, (NI / 32 + 2) * 4);
  for (int d = 0; d < 4; d++) {
    size_t n = d == 3 ? FN : Pn;
    want(&a->sd_first[d], S * 4, 0); want(&a->sd_rank[d], S * 4); want(&a->sd_order[d], S * 4);
    want(&a->sd_keys[d], n * 4); want(&a->sd_valid[d], (n / 32 + 2) * 4);
    want(&P.sd_bits[d], (n / 32 + 2) * 4); want(&P.sd_wp[d], (n / 32 + 2) * 4);
  }
  want(&a->fn_first, FN * 4, 0); want(&a->fn_rank, FN * 4); want(&a->fn_order, FN * 4); want(&a->fn_keys, Pn * 4);
  want(&P.fn_bits, (Pn / 32 + 2) * 4); want(&P.fn_wp, (Pn / 32 + 2) * 4);
  want(&a->lo.address, Pn * 8); want(&a->lo.line_off, Pn * 4); want(&a->lo.line_size, Pn * 4); want(&a->lo.line_valid, (Pn / 32 + 2) * 4);
  want(&a->lo.line_no, Pn * 8);
  if (md) want(&P.edge_keys, (size_t)ncols * 32, 1);
  P.col_first.assign(ncols, nullptr); P.col_rank.assign(ncols, nullptr); P.col_bits.assign(ncols, nullptr); P.col_wp.assign(ncols, nullptr);
  a->tid_slots = nullptr; a->tid_rank = nullptr;
  for (uint32_t c = 0; c < ncols; c++) {
    ColPlan& cp = a->cols[c];
    cp.validity = nullptr; cp.order = nullptr;
    want(&cp.run_ends, Nn * 4);
    want(&cp.run_keys, Nn * 4);
    if (v1 && cp.type == COL_KIND && cp.param == 5) want(&cp.validity, (Nn / 32 + 3) * 4, 1);  // temporality has null runs
    if (c >= nlab) continue;
    want(&cp.validity, (Nn / 32 + 3) * 4, 1);
    want(&P.col_bits[c], (NTn / 32 + 2) * 4); want(&P.col_wp[c], (NTn / 32 + 2) * 4);
    if (cp.type == COL_COMM) cp.universe = P.n_cstr;
    if (cp.type == COL_TID) {
      want(&a->tid_slots, (size_t)tcap * 8, 0);
      want(&a->tid_rank, (size_t)tcap * 4);
      want(&cp.order, (size_t)std::min<uint64_t>(NTn, tcap) * 4);
    } else {
      size_t u = std::max<uint32_t>(cp.universe, 1);
      if (cp.type == COL_CPU) P.col_first[c] = first_cpu;
      else if (cp.type == COL_COMM) P.col_first[c] = first_comm;
      else want(&P.col_first[c], u * 4, 0);
      want(&P.col_rank[c], u * 4); want(&cp.order, u * 4);
    }
  }
  P.cls_bytes[0] = P.cls_bytes[1] = P.cls_bytes[2] = 0;
  for (auto& r : reqs) P.cls_bytes[r.cls] += r.bytes;
  CK(a->d_arena.ensure(std::max<size_t>(P.cls_bytes[0] + P.cls_bytes[1] + P.cls_bytes[2], 256)));
  {
    size_t off[3] = {0, P.cls_bytes[0], P.cls_bytes[0] + P.cls_bytes[1]};  // [0xFF region][zero region][rest]
    for (auto& r : reqs) { *r.pp = a->d_arena.as<uint8_t>() + off[r.cls]; off[r.cls] += r.bytes; }
  }
  for (uint32_t c = 0; c < nlab; c++) {  // the shared tables were carved before the loop
    if (a->cols[c].type == COL_CPU) P.col_first[c] = first_cpu;
    if (a->cols[c].type == COL_COMM) P.col_first[c] = first_comm;
  }
  P.red_block = P.first_ls;
  P.red_count = red_bytes / 4;
  a->lo.type_key = a->sd_keys[0]; a->lo.map_key = a->sd_keys[1]; a->lo.bid_key = a->sd_keys[2]; a->lo.func_key = a->fn_keys;

  Counters* ctr = a->d_ctr.as<Counters>();
  // ---- dictionaries: jobs table
  std::vector<FoJob>& jobs = P.jobs;
  jobs.clear();
  auto job = [&](const uint32_t* keys, const uint32_t* n_ptr, uint32_t* first, uint32_t universe, uint32_t* rank, uint32_t* order, uint32_t* out,
                 uint32_t* validity, uint32_t* bitmap, uint32_t* wprefix, uint32_t* n_unique, uint32_t* n_null, bool nullable, bool skip_min) {
    FoJob j{};
    j.keys = keys; j.n_ptr = n_ptr; j.first = first; j.universe = universe; j.rank = rank; j.order = order; j.out = out; j.validity = validity;
    j.bitmap = bitmap; j.wprefix = wprefix; j.n_unique = n_unique; j.n_null = n_null; j.nullable = nullable; j.skip_min = skip_min; j.ctr = ctr;
    jobs.push_back(j);
    return (int)jobs.size() - 1;
  };
  // the low 32 bits of n_indices64 are the index count (overflow is flagged separately)
  const uint32_t* n_idx_ptr = (const uint32_t*)&ctr->n_indices64;
  const uint32_t n_cstr = P.n_cstr;
  P.j_loc = job(a->d_ustream.as<uint32_t>(), n_idx_ptr, a->loc_first, P.n_frames, a->loc_rank, a->loc_order, a->d_ustream.as<uint32_t>(), nullptr,
                P.loc_bits, P.loc_wp, &ctr->n_locations, nullptr, false, true);
  P.j_type = job(a->sd_keys[0], &ctr->n_locations, a->sd_first[0], n_cstr, a->sd_rank[0], a->sd_order[0], a->sd_keys[0], nullptr, P.sd_bits[0], P.sd_wp[0], &ctr->n_dict_type, nullptr, false, false);
  job(a->sd_keys[1], &ctr->n_locations, a->sd_first[1], n_cstr, a->sd_rank[1], a->sd_order[1], a->sd_keys[1], nullptr, P.sd_bits[1], P.sd_wp[1], &ctr->n_dict_map, nullptr, false, false);
  job(a->sd_keys[2], &ctr->n_locations, a->sd_first[2], n_cstr, a->sd_rank[2], a->sd_order[2], a->sd_keys[2], a->sd_valid[2], P.sd_bits[2], P.sd_wp[2], &ctr->n_dict_bid, &ctr->null_bid, true, false);
  job(a->fn_keys, &ctr->n_lines, a->fn_first, P.n_funcs, a->fn_rank, a->fn_order, a->fn_keys, nullptr, P.fn_bits, P.fn_wp, &ctr->n_functions, nullptr, false, false);
  P.j_file = job(a->sd_keys[3], &ctr->n_functions, a->sd_first[3], n_cstr, a->sd_rank[3], a->sd_order[3], a->sd_keys[3], a->sd_valid[3], P.sd_bits[3], P.sd_wp[3], &ctr->n_dict_file, &ctr->null_file, true, false);
  P.j_lab0 = (int)jobs.size();
  for (uint32_t c = 0; c < nlab; c++) {
    ColPlan& cp = a->cols[c];
    bool nullable = cp.type == COL_LS || cp.type == COL_COMM;
    // first ROWS are recorded by k_header / k_ls_plan (skip_min); the emit pass applies the ranks itself (no map pass)
    int ji = job(nullptr, nullptr, P.col_first[c], cp.universe, P.col_rank[c], cp.order, nullptr, nullptr, P.col_bits[c], P.col_wp[c],
                 &ctr->n_dict[c], nullptr, nullable, true);
    jobs[ji].n_imm = (uint32_t)P.NT;
    if (cp.type == COL_TID) { jobs[ji].hashed = 1; jobs[ji].hslots = a->tid_slots; jobs[ji].hmask = a->tid_mask; jobs[ji].rank = a->tid_rank; }
  }
  std::vector<ReeCol>& rc = P.rc;
  rc.assign(ncols, ReeCol{});
  ReeArgs& ra = P.ra;
  ra = ReeArgs{};
  ra.c_cpu = ra.c_tid = ra.c_comm = ra.c_ord = ra.c_ts = -1;
  for (uint32_t c = 0; c < ncols; c++) {
    const ColPlan& cp = a->cols[c];
    rc[c] = ReeCol{cp.type, cp.param, cp.run_ends, cp.run_keys, c < nlab ? P.col_first[c] : nullptr, nullptr, 0,
                   (cp.type == COL_LS || cp.type == COL_COMM) ? 1u : 0u, c < nlab ? P.col_rank[c] : nullptr, c < nlab ? cp.validity : nullptr};
    if (cp.type == COL_TID) { rc[c].hslots = a->tid_slots; rc[c].hmask = a->tid_mask; rc[c].rank = a->tid_rank; }
    if (cp.type == COL_CPU) ra.c_cpu = (int)c;
    if (cp.type == COL_TID) ra.c_tid = (int)c;
    if (cp.type == COL_COMM) ra.c_comm = (int)c;
    if (cp.type == COL_ORD) ra.c_ord = (int)c;
    if (cp.type == COL_TS) ra.c_ts = (int)c;
    if (v1 && cp.type == COL_KIND && cp.param == 5) { rc[c].nullable = 1; rc[c].validity = cp.validity; }
  }
  if (v1) { ra.ord = a->v1_ord; ra.ts = a->d_ts.as<long long>(); ra.ts_vals = a->v1_ts_vals; ra.kindrank = a->v1_kindrank; ra.kind_dict_mask = 0x3Fu; }
  ra.n_rows = (uint32_t)N; ra.ncols = ncols; ra.n_ls = a->n_lscols; ra.c_kind = nlab; ra.cols = nullptr /* set after the upload */;
  ra.ls = a->d_ls.as<uint32_t>(); ra.cpu = a->d_cpu.as<uint32_t>(); ra.tid = a->d_tid.as<uint32_t>(); ra.comm = a->d_comm.as<uint32_t>(); ra.kind = a->d_kind.as<uint8_t>();
  ra.ls_rank = P.ls_rank; ra.ls_keys = P.ls_keys; ra.n_lscols = std::max<uint32_t>(1, a->n_lscols); ra.kindtab = a->d_kindtab.as<uint32_t>();
  ra.partial = a->d_ree_partial.as<uint32_t>(); ra.ctr = ctr;
  ra.row_base = (uint32_t)P.row_base; ra.edge_keys = md ? P.edge_keys : nullptr; ra.mc = nullptr;
  ReeGroups& rg = P.rg;  // one launch row per column (the 8 kind-derived columns form one group)
  rg = ReeGroups{};
  for (uint32_t c = 0; c < ncols; c++) {
    const ColPlan& cp = a->cols[c];
    if (cp.type == COL_KIND && cp.param != 0) continue;
    rg.g[rg.n++] = ReeGroup{cp.type, c, cp.param};
  }
  int rcu = upload_descriptors(a, jobs.data(), jobs.size() * sizeof(FoJob), rc.data(), rc.size() * sizeof(ReeCol));
  if (rcu) return rcu;
  ra.cols = a->d_cols.as<ReeCol>();
  for (int t = 0; t < T_COUNT; t++) { a->tm[t].launches = 0; a->tm[t].ms = 0; }
  return PA_OK;
}

// memsets, header split (+insert in provided mode), hash+insert
static int pass_front(pa_agg* a) {
  Pass& P = a->P;
  const uint64_t N = P.N;
  cudaStream_t s = a->s_comp;
  Counters* ctr = a->d_ctr.as<Counters>();
  StackSlot* tab = a->d_table.as<StackSlot>();
  CK(cudaEventRecord(a->tm[T_TOTAL].a, s));
  CK(cudaMemsetAsync(ctr, 0, sizeof(Counters), s));
  CK(cudaMemsetAsync(tab, 0, (P.cap + 2) * sizeof(StackSlot), s));
  if (P.cls_bytes[0]) CK(cudaMemsetAsync(a->d_arena.p, 0xFF, P.cls_bytes[0], s));
  if (P.cls_bytes[1]) CK(cudaMemsetAsync(a->d_arena.as<uint8_t>() + P.cls_bytes[0], 0, P.cls_bytes[1], s));
  const bool provided = P.provided;
  // When the whole batch is already resident (pa_agg_stage) the two passes run back to back and
  // are timed separately; during an overlapped flush they interleave per chunk as copies land.
  const bool resident = a->chunk_ev.empty() || a->chunk_rows.empty() || cudaEventQuery(a->chunk_ev[a->chunk_rows.size() - 1]) == cudaSuccess;
  a->hash_timed = resident && !provided;
  auto launch_header = [&](uint64_t r0, uint64_t r1, uint64_t frames_end) {
    HeaderArgs h{};
    h.hdr = a->d_hdr.as<uint4>(); h.row0 = (uint32_t)r0; h.row1 = (uint32_t)r1; h.row_base = (uint32_t)P.row_base;
    h.timestamp = a->d_ts.as<long long>(); h.value = a->d_value.as<long long>(); h.uuid = a->d_uuid.as<uint8_t>();
    h.kind = a->d_kind.as<uint8_t>(); h.nframes = a->d_nfr.as<uint16_t>(); h.frame_off = a->d_foff.as<unsigned long long>();
    h.ls = a->d_ls.as<uint32_t>(); h.cpu = a->d_cpu.as<uint32_t>(); h.tid = a->d_tid.as<uint32_t>(); h.comm = a->d_comm.as<uint32_t>();
    h.sid2cid = a->m_sid2cid.ptr(); h.n_sids = P.n_sids; h.n_labelsets = P.n_labelsets;
    h.n_frame_ids = frames_end; h.provided = provided ? 1 : 0; h.tab = tab; h.mask = P.mask; h.slot_of_row = a->d_slot.as<uint32_t>(); h.ctr = ctr; h.claimed = P.claimed;
    h.first_ls = P.n_names ? P.first_ls : nullptr;
    for (uint32_t c = 0; c < P.nlab; c++) {
      if (a->cols[c].type == COL_CPU) h.first_cpu = P.col_first[c];
      if (a->cols[c].type == COL_TID) { h.tid_slots = a->tid_slots; h.tid_mask = a->tid_mask; }
      if (a->cols[c].type == COL_COMM) h.first_comm = P.col_first[c];
    }
    h.first_kind = P.v1 ? a->v1_first_kind : nullptr;
    h.stacks = (const uint4*)a->d_rs_recs.p; h.n_stacks = P.n_stacks;
    h.last_use = a->d_rs_last.as<uint32_t>(); h.seq = (uint32_t)a->rs_stages;
    uint64_t rows = r1 - r0;
    int hb = (int)std::min<uint64_t>((rows + kThreads - 1) / kThreads, (uint64_t)a->sms * kHdrBlocksPerSm);
    if (a->retire) k_header<true, true><<<std::max(hb, 1), kThreads, 0, s>>>(h);
    else if (a->registered) k_header<true><<<std::max(hb, 1), kThreads, 0, s>>>(h);
    else k_header<false><<<std::max(hb, 1), kThreads, 0, s>>>(h);
    a->tm[T_HEADER].launches++;
  };
  auto launch_hash = [&](uint64_t r0, uint64_t r1) {
    HashArgs ha{};
    ha.frames = a->d_frames.as<unsigned long long>(); ha.frames32 = a->idb == 4 ? a->d_frames.as<uint32_t>() : nullptr; ha.frame_off = a->d_foff.as<unsigned long long>(); ha.nframes = a->d_nfr.as<uint16_t>();
    ha.row0 = (uint32_t)r0; ha.row1 = (uint32_t)r1; ha.uuid = a->d_uuid.as<uint8_t>();
    ha.slot_of_row = a->d_slot.as<uint32_t>(); ha.tab = tab; ha.mask = P.mask; ha.ctr = ctr; ha.claimed = P.claimed;
    uint64_t rows = r1 - r0;
    int blocks = (int)std::min<uint64_t>((rows + kThreads - 1) / kThreads, (uint64_t)a->sms * (a->hash_variant == 1 ? 3 : 4));
    auto tma_grid = [&](int warps) { return (int)std::max<uint64_t>(1, std::min<uint64_t>((rows + 32ull * warps - 1) / (32ull * warps), (uint64_t)a->sms)); };
    if (a->hash_variant == 6 && a->idb == 8) k_hash_insert_tma<16, 3, 8><<<tma_grid(16), 16 * 32, sizeof(TmaSmem<16, 3, 8>), s>>>(ha);
    else if (a->hash_variant == 7 && a->idb == 8) k_hash_insert_tma<12, 4, 8><<<tma_grid(12), 12 * 32, sizeof(TmaSmem<12, 4, 8>), s>>>(ha);
    else if (a->hash_variant == 8 && a->idb == 8) k_hash_insert_tma<24, 2, 8><<<tma_grid(24), 24 * 32, sizeof(TmaSmem<24, 2, 8>), s>>>(ha);
    else if (a->hash_variant == 9 && a->idb == 8) k_hash_insert_tma<12, 2, 16><<<tma_grid(12), 12 * 32, sizeof(TmaSmem<12, 2, 16>), s>>>(ha);
    else if (a->hash_variant == 10 && a->idb == 8) k_hash_insert_tma<13, 2, 16><<<tma_grid(13), 13 * 32, sizeof(TmaSmem<13, 2, 16>), s>>>(ha);
    else if (a->hash_variant == 11 && a->idb == 8) k_hash_insert_tma<8, 3, 16><<<tma_grid(8), 8 * 32, sizeof(TmaSmem<8, 3, 16>), s>>>(ha);
    else if (a->hash_variant == 12 && a->idb == 8) k_hash_insert_tmag<13, 2><<<tma_grid(13), 13 * 32, sizeof(TmagSmem<13, 2>), s>>>(ha);
    else if (a->hash_variant == 13 && a->idb == 8) k_hash_insert_tmag<9, 3><<<tma_grid(9), 9 * 32, sizeof(TmagSmem<9, 3>), s>>>(ha);
    else if (a->hash_variant == 14 && a->idb == 8) k_hash_insert_tmag<6, 4><<<tma_grid(6), 6 * 32, sizeof(TmagSmem<6, 4>), s>>>(ha);
    else if (a->hash_variant == 15 && a->idb == 8) k_hash_insert_widepf3<<<(int)std::max<uint64_t>(1, std::min<uint64_t>((rows + kThreads - 1) / kThreads, (uint64_t)a->sms * 3)), kThreads, 0, s>>>(ha);
    else if (a->hash_variant == 5 && a->idb == 4) k_hash_insert_widepf32<<<std::max(blocks, 1), kThreads, 0, s>>>(ha);
    else if (a->hash_variant == 5) k_hash_insert_widepf<<<std::max(blocks, 1), kThreads, 0, s>>>(ha);
    else if (a->idb == 4) k_hash_insert_wide32<<<std::max(blocks, 1), kThreads, 0, s>>>(ha);
    else if (a->hash_variant == 3) k_hash_insert_bulk<4, 3><<<(int)std::max<uint64_t>(1, std::min<uint64_t>((rows + 127) / 128, (uint64_t)a->sms)), 128, sizeof(BulkSmem<4, 3>), s>>>(ha);
    else if (a->hash_variant == 4) k_hash_insert_bulk<6, 2><<<(int)std::max<uint64_t>(1, std::min<uint64_t>((rows + 191) / 192, (uint64_t)a->sms)), 192, sizeof(BulkSmem<6, 2>), s>>>(ha);
    else if (a->hash_variant == 1) k_hash_insert_staged<<<std::max(blocks, 1), kThreads, kHashStagedSmem, s>>>(ha);
    else if (a->hash_variant == 16 && a->idb == 8) k_hash_insert_wide_np<<<std::max(blocks, 1), kThreads, 0, s>>>(ha);
    else if (a->hash_variant == 2 || a->hash_variant == 16) k_hash_insert_wide<<<std::max(blocks, 1), kThreads, 0, s>>>(ha);
    else k_hash_insert<<<std::max(blocks, 1), kThreads, 0, s>>>(ha);
    a->tm[T_HASH].launches++;
  };
  CK(cudaEventRecord(a->tm[T_HEADER].a, s));
  if (resident) {
    if (N) launch_header(0, N, a->NF);  // whole resident batch: one launch per pass
    CK(cudaEventRecord(a->tm[T_HEADER].b, s));
    CK(cudaEventRecord(a->tm[T_HASH].a, s));
    if (!provided && N) launch_hash(0, N);
    CK(cudaEventRecord(a->tm[T_HASH].b, s));
  } else if (a->early.hdr_first && !provided) {
    CK(cudaStreamWaitEvent(s, a->ev_hdr_all, 0));
    if (N) launch_header(0, N, a->NF);
    CK(cudaEventRecord(a->tm[T_HEADER].b, s));
    CK(cudaEventRecord(a->ev_hdr_done, s));
    if (!a->serial && !P.v1 && !P.merged) { CK(cudaEventRecord(a->ev_fork, s)); a->forked_early = true; }  // the label chain starts here, under the upload of the ids
    for (size_t k = 0; k < a->chunk_rows.size(); k++) {
      CK(cudaStreamWaitEvent(s, a->chunk_ev[k], 0));
      launch_hash(a->chunk_rows[k].first, a->chunk_rows[k].second);
      CK(cudaEventRecord(a->hash_ev[k], s));
    }
  } else {
    for (size_t k = 0; k < a->chunk_rows.size(); k++) {
      CK(cudaStreamWaitEvent(s, a->chunk_ev[k], 0));
      launch_header(a->chunk_rows[k].first, a->chunk_rows[k].second, a->chunk_frames_end[k]);
      if (!provided) launch_hash(a->chunk_rows[k].first, a->chunk_rows[k].second);
    }
    CK(cudaEventRecord(a->tm[T_HEADER].b, s));
  }
  return PA_OK;
}

// unique stacks of ONE aggregator: ordinals from the first-row bitmap, offsets from a scan over the unique list,
// per-row ListView (offset, size), gather of the unique stacks' frames
static int pass_rank_single(pa_agg* a) {
  Pass& P = a->P;
  const uint64_t N = P.N;
  cudaStream_t s = a->s_comp;
  Counters* ctr = a->d_ctr.as<Counters>();
  StackSlot* tab = a->d_table.as<StackSlot>();
  const int G = a->G;
  CK(cudaEventRecord(a->tm[T_RANK].a, s));
  const int Gw = small_grid(a, N / 32 + 1), Gu = small_grid(a, std::min<uint64_t>(N, P.cap / 2));
  k_stack_bits<<<Gu, kThreads, 0, s>>>(tab, P.claimed, &ctr->n_claimed, P.rowbits);
  launch_scan(a, WordsF{P.rowbits, P.row_wprefix, (uint32_t)((N + 31) / 32), &ctr->n_unique}, 1, a->tm[T_RANK], Gw, s, a->d_partial);
  k_stack_assign<<<Gu, kThreads, 0, s>>>(tab, P.claimed, &ctr->n_claimed, P.rowbits, P.row_wprefix, a->d_nfr.as<uint16_t>(), a->d_uniq_row.as<uint32_t>(), P.uniq_slot, P.uniq_size);
  launch_scan(a, UniqOffsetF{ctr, ctr, P.uniq_size, P.uniq_slot, tab}, 1, a->tm[T_RANK], Gu, s, a->d_partial);
  a->tm[T_RANK].launches += 2;
  k_rows_materialize<<<G, kThreads, 0, s>>>((uint32_t)N, a->d_slot.as<uint32_t>(), tab, a->d_stoff.as<int>(), a->d_stsize.as<int>(), P.v1 ? a->v1_ord : nullptr);
  if (P.v1) {  // v1 has no inline stacktraces: only the dictionary of unique stack ids
    k_gather_ids<<<small_grid(a, std::min<uint64_t>(N, P.cap / 2) + 1), kThreads, 0, s>>>(ctr, a->d_uniq_row.as<uint32_t>(), a->d_uuid.as<uint8_t>(), a->v1_ids, a->v1_id_off);
    a->tm[T_RANK].launches++;
  } else {
    k_gather_unique<<<G, kThreads, 0, s>>>(ctr, a->d_uniq_row.as<uint32_t>(), a->d_slot.as<uint32_t>(), tab, a->src_frames, a->d_foff.as<unsigned long long>(), P.n_frames,
                                           a->d_ustream.as<uint32_t>(), a->loc_first, ctr, a->idb == 4 ? 1u : 0u);
  }
  a->tm[T_RANK].launches += 2;
  CK(cudaEventRecord(a->tm[T_RANK].b, s));
  return PA_OK;
}

// location / function / string dictionaries from the (merged) unique-stack frame stream
static int pass_locations(pa_agg* a) {
  Pass& P = a->P;
  cudaStream_t s = a->s_comp;
  Counters* ctr = a->d_ctr.as<Counters>();
  const FoJob* djobs = a->d_jobs.as<FoJob>();
  const int G = a->G;
  const size_t Pn = P.Pn, S = P.S, FN = P.FN;
  CK(cudaEventRecord(a->tm[T_LOC].a, s));
  FrameTable ftd{(const unsigned long long*)a->m_addr.ptr(), a->m_type.ptr(), a->m_map.ptr(), a->m_bid.ptr(), (const unsigned long long*)a->m_line.ptr(), a->m_func.ptr()};
  if (!P.v1) {  // v1 carries no locations in the sample record
    run_fo_jobs(a, djobs, P.j_loc, 1, false, a->tm[T_LOC], std::min<uint64_t>(P.NI, P.merged ? P.NI : P.cap * 32), Pn, true, s, a->d_partial);  // location index per unique-stack frame (in place over the gathered stream)
    launch_scan(a, LocLinesF{ctr, ctr, a->loc_order, ftd, a->lo}, 1, a->tm[T_LOC], small_grid(a, Pn), s, a->d_partial);
    k_line_validity<<<std::max(1, std::min(G, (int)(Pn / 256 + 1))), kThreads, 0, s>>>(ctr, a->lo.line_size, a->lo.line_valid);
    run_fo_jobs(a, djobs, P.j_type, 4, true, a->tm[T_LOC], Pn, std::max(S, FN), true, s, a->d_partial);  // frame_type, mapping_file, mapping_build_id, function
    k_func_keys<<<std::max(1, std::min(G, (int)(FN / 256 + 1))), kThreads, 0, s>>>(ctr, a->fn_order, a->m_fnfile.ptr(), a->sd_keys[3]);
    run_fo_jobs(a, djobs, P.j_file, 1, true, a->tm[T_LOC], FN, S, true, s, a->d_partial);  // function.filename
    a->tm[T_LOC].launches += 2;
  }
  CK(cudaEventRecord(a->tm[T_LOC].b, s));
  return PA_OK;
}

// run-end encoding of label + constant columns, three steps so that a merged batch can exchange in between:
// count (+ partial scan), dictionary ranks, emit. `s` may be a second stream (the chain only depends on k_header).
static int pass_labels_count(pa_agg* a, cudaStream_t s) {
  Pass& P = a->P;
  if (getenv("PA_DEBUG_SYNC")) CK(cudaStreamSynchronize(s));
  CK(cudaEventRecord(a->tm[T_LABELS].a, s));
  if (P.n_names) {  // check the column plan and apply it: key matrix and first rows of the labelset-derived values
    LsPlanArgs lp{};
    lp.first_ls = P.first_ls; lp.n_labelsets = P.n_labelsets;
    lp.off = a->m_ls_off.ptr(); lp.pairs = (const uint2*)a->m_ls_pairs.ptr();
    lp.n_cols = a->n_lscols; lp.rank = P.ls_rank; lp.keys = P.ls_keys; lp.n_used = P.ls_used; lp.used_names = P.used_names;
    lp.ctr = a->d_ctr.as<Counters>();
    for (uint32_t c = 0; c < a->n_lscols; c++) { lp.plan_ord[c] = a->cols[c].ord; lp.col_first[c] = P.col_first[c]; }
    k_ls_plan<<<small_grid(a, P.n_labelsets), kThreads, 0, s>>>(lp);
    a->tm[T_LABELS].launches++;
  }
  if (P.v1) { k_kind_ranks<<<1, 32, 0, s>>>(a->v1_first_kind, a->d_kindtab.as<uint32_t>(), a->v1_kindrank, a->v1_kind_order, a->v1_n_kind_dict); a->tm[T_LABELS].launches++; }
  const int Gr = a->sms * kReeBlocksPerSm;
  const dim3 ree_grid(Gr, P.rg.n);
  if (P.merged) k_ree_col<false, true><<<ree_grid, kThreads, 0, s>>>(P.ra, P.rg);  // run counts (+ this shard's border keys)
  else k_ree_col<false, false><<<ree_grid, kThreads, 0, s>>>(P.ra, P.rg);
  k_ree_scan_partials<<<P.ncols, kThreads, 0, s>>>(P.ra, Gr * kWarps, 0u);
  a->tm[T_LABELS].launches += 2;
  return PA_OK;
}
static int pass_label_dicts(pa_agg* a, cudaStream_t s, DBuf& partial) {
  Pass& P = a->P;
  CK(cudaEventRecord(a->tm[T_DICTS].a, s));
  if (P.nlab) run_fo_jobs(a, a->d_jobs.as<FoJob>(), P.j_lab0, (int)P.nlab, false, a->tm[T_DICTS], P.NT, std::max<uint64_t>(std::max<uint64_t>(P.S, 65536), P.tcap), false, s, partial);  // label dictionary ranks
  CK(cudaEventRecord(a->tm[T_DICTS].b, s));
  return PA_OK;
}
static int pass_labels_emit(pa_agg* a, cudaStream_t s) {
  Pass& P = a->P;
  const dim3 ree_grid(a->sms * kReeBlocksPerSm, P.rg.n);
  if (P.merged) k_ree_col<true, true><<<ree_grid, kThreads, 0, s>>>(P.ra, P.rg);   // run ends + final dictionary indices + validity bits
  else k_ree_col<true, false><<<ree_grid, kThreads, 0, s>>>(P.ra, P.rg);
  a->tm[T_LABELS].launches += 1;
  CK(cudaEventRecord(a->tm[T_LABELS].b, s));
  return PA_OK;
}

// counters to the host, synchronise, collect the group timings
static int pass_finish(pa_agg* a) {
  cudaStream_t s = a->s_comp;
  Counters* ctr = a->d_ctr.as<Counters>();
  CK(cudaMemcpyAsync(a->h_ctr_pinned, ctr, sizeof(Counters), cudaMemcpyDeviceToHost, s));
  if (a->P.used_names) CK(cudaMemcpyAsync(a->h_used, a->P.used_names, (a->P.n_names + 31) / 32 * 4, cudaMemcpyDeviceToHost, s));
  CK(cudaEventRecord(a->tm[T_TOTAL].b, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  a->h_ctr = *a->h_ctr_pinned;
  a->launches = 0;
  for (int t = 0; t < T_TOTAL; t++) {
    float ms = 0;
    if (a->tm[t].launches && (t != T_HASH || a->hash_timed)) { cudaEventElapsedTime(&ms, a->tm[t].a, a->tm[t].b); }
    a->tm[t].ms = ms;
    a->launches += a->tm[t].launches;
  }
  a->tm[T_LABELS].ms = std::max(0.0, a->tm[T_LABELS].ms - a->tm[T_DICTS].ms);  // the dictionary ranking runs between the two REE passes
  float tot = 0;
  cudaEventElapsedTime(&tot, a->tm[T_TOTAL].a, a->tm[T_TOTAL].b);
  a->tm[T_TOTAL].ms = tot;
  a->tm[T_TOTAL].launches = a->launches;
  return PA_OK;
}

static int early_copy_issue(pa_agg* a);

static int process_once(pa_agg* a) {
  int rc = pass_plan(a, nullptr);
  if (rc) return rc;
  a->forked_early = false;
  if ((rc = pass_front(a))) return rc;
  // The label chain depends only on k_header's outputs; the stack-rank / location chain only on the table. Both are
  // chains of small latency-bound launches, so they run side by side on two streams (PA_SERIAL=1: one stream, so
  // that the per-group event timings do not overlap).
  // (v1: the run-end encoded stacktrace_id column reads the stack ordinals the rank chain produces, so the chains stay in order)
  const bool fork = !a->serial && !a->P.v1;
  cudaStream_t s = a->s_comp, s2 = fork ? a->s_aux : a->s_comp;
  if (fork) { if (!a->forked_early) CK(cudaEventRecord(a->ev_fork, s)); CK(cudaStreamWaitEvent(s2, a->ev_fork, 0)); }
  if ((rc = pass_rank_single(a))) return rc;
  if ((rc = pass_locations(a))) return rc;
  if ((rc = pass_labels_count(a, s2))) return rc;
  if ((rc = pass_label_dicts(a, s2, fork ? a->d_partial2 : a->d_partial))) return rc;
  if ((rc = pass_labels_emit(a, s2))) return rc;
  // (the early copy-out is not worth starting when the upload has already finished: nothing left to hide behind)
  const bool early = fork && a->forked_early && a->early.hdr_first && !a->early.issued && !a->P.merged && a->out && !a->chunk_rows.empty() &&
                     (a->early_force || cudaEventQuery(a->chunk_ev[a->chunk_rows.size() - 1]) != cudaSuccess);
  if (early) {
    CK(cudaMemcpyAsync(a->h_early, a->d_ctr.p, sizeof(Counters), cudaMemcpyDeviceToHost, s2));
    CK(cudaEventRecord(a->ev_early, s2));
  }
  if (fork) { CK(cudaEventRecord(a->ev_join, s2)); CK(cudaStreamWaitEvent(s, a->ev_join, 0)); }
  if (early && (rc = early_copy_issue(a))) return rc;
  return pass_finish(a);
}

static int check_batch_errors(pa_agg* a, uint32_t e) {
  if (e & ERR_TABLE_FULL) return a->fail(PA_ENOMEM, "stack table overflow");
  if (e & ERR_LABEL_PLAN) return a->fail(PA_EIO, "label column plan: a used label name is still not planned after the redo");
  if (e & ERR_INDEX_OVERFLOW) return a->fail(PA_ERANGE, "location-index stream exceeds int32 (reporter/arrow_v2.go:233)");
  if (e & ERR_BAD_FRAME_ID) return a->fail(PA_EINVAL, "sample refers to an unregistered frame id");
  if (e & ERR_BAD_STRING_ID) return a->fail(PA_EINVAL, "sample refers to an unregistered string id");
  if (e & ERR_BAD_LABELSET) return a->fail(PA_EINVAL, "sample refers to an unregistered labelset id");
  if (e & ERR_BAD_KIND) return a->fail(PA_EINVAL, "sample kind out of range");
  if (e & ERR_BAD_CPU) return a->fail(PA_EINVAL, "cpu id >= 65536");
  if (e & ERR_BAD_FRAME_RANGE) return a->fail(PA_EINVAL, "sample frame range outside the staged frames (frame_off must ascend with the rows)");
  if (e & ERR_SLICE_CAP) return a->fail(PA_ENOSPC, "merged batch: this shard's part of the location-index stream exceeds max_frames");
  if (e & ERR_MERGE_LOOKUP) return a->fail(PA_EIO, "merged batch: a local stack is missing from the merged dictionary");
  if (e & ERR_BAD_STACK_ID) return a->fail(PA_EINVAL, "sample refers to an unregistered stack id (PA_CFG_REGISTERED_STACKS: frame_off is a stack id)");
  return PA_OK;
}

static void remember_sizes(pa_agg* a) {  // adaptive table sizing for the next interval
  a->prev_unique = a->h_ctr.n_unique;
  a->prev_tids = 0;
  for (uint32_t c = 0; c < a->n_label_cols; c++) if (a->cols[c].type == COL_TID) a->prev_tids = a->h_ctr.n_dict[c];
  a->retry_cap = 0;
  a->retry_tcap = 0;
  a->used_prev = used_names(a);  // the next batch's label column prediction starts from these
  a->names_planned = a->P.n_names;
  a->plan_pending = false;
}

static int process(pa_agg* a) {
  if (a->staged < 0) return a->fail(PA_EINVAL, "nothing staged");
  CK(cudaSetDevice(a->device));
  a->merged_part = false;
  if (a->N == 0) { a->processed = true; a->last_unique = 0; memset(&a->h_ctr, 0, sizeof a->h_ctr); return PA_OK; }
  int rc = upload_tables(a, true);
  if (rc) return rc;
  for (int attempt = 0; attempt < 6; attempt++) {
    rc = process_once(a);
    if (rc) return rc;
    const uint32_t e = a->h_ctr.err;
    if (!(e & (ERR_TABLE_FULL | ERR_LABEL_PLAN))) break;
    if (a->early.issued) CK(cudaStreamSynchronize(a->s_d2h));  // (k_header runs again and rewrites, with the same values, what is being copied out)
    if (e & ERR_TABLE_FULL) {
      a->retry_cap = a->table_cap * 4;  // unique-stack / thread-id estimate was too small: grow and redo the batch
      a->retry_tcap = a->tid_cap * 4;
    }
    if ((e & ERR_LABEL_PLAN) && (rc = replan_labels(a))) return rc;  // a used label name was not planned: plan the used ones, redo
  }
  if ((rc = check_batch_errors(a, a->h_ctr.err))) return rc;
  if (a->cfg.schema == PA_SCHEMA_V1) {
    if ((rc = v1_store_update(a))) return rc;
    if ((rc = check_batch_errors(a, a->h_ctr.err))) return rc;
    {  // the store's share belongs to the pass: "total" runs to the end of it
      CK(cudaEventRecord(a->tm[T_TOTAL].b, a->s_comp));
      CK(cudaEventSynchronize(a->tm[T_TOTAL].b));
      float tot = 0;
      cudaEventElapsedTime(&tot, a->tm[T_TOTAL].a, a->tm[T_TOTAL].b);
      a->tm[T_TOTAL].ms = tot;
      a->launches += 2;  // k_last_rows, k_store_insert (select / kill / rebuild launches come on top when they run)
      a->tm[T_TOTAL].launches = a->launches;
    }
    a->last_unique = a->h_ctr.n_unique;
  }
  remember_sizes(a);
  a->processed = true;
  return PA_OK;
}

// ---------------------------------------------------------------------------------------------
// collect: counters -> layout -> D2H of every device-resident Arrow buffer into its final place
namespace {

struct HostCol {  // a label column materialised on the host (only when an external label touches it)
  std::vector<int32_t> run_ends;
  std::vector<uint32_t> idx;
  std::vector<uint8_t> valid;
  std::vector<std::string> dict;
  int64_t len = 0;  // ree.Len()
};

std::vector<uint8_t>& keep(pa_agg* a, std::vector<uint8_t>&& v) { a->hostbufs.push_back(std::move(v)); return a->hostbufs.back(); }
template <class T>
BufRef host_ref(pa_agg* a, const std::vector<T>& v) {
  std::vector<uint8_t> b(v.size() * sizeof(T));
  if (!v.empty()) memcpy(b.data(), v.data(), b.size());
  auto& k = keep(a, std::move(b));
  return BufRef::host(k.data(), k.size());
}

Node int_node(const char* name, int bits, bool sgn, bool nullable, int64_t len, BufRef data) {
  Node n; n.ty = Ty::Int; n.name = name; n.bits = bits; n.is_signed = sgn; n.nullable = nullable; n.length = len; n.bufs = {data};
  return n;
}
// utf8 array from a list of strings
Node utf8_node(pa_agg* a, const char* name, bool nullable, const std::vector<std::pair<const uint8_t*, uint32_t>>& strs,
               const std::vector<uint8_t>* valid = nullptr, Ty ty = Ty::Utf8) {
  std::vector<int32_t> off(strs.size() + 1, 0);
  uint64_t tot = 0;
  for (size_t i = 0; i < strs.size(); i++) { tot += strs[i].second; off[i + 1] = (int32_t)tot; }
  std::vector<uint8_t> data(tot);
  for (size_t i = 0; i < strs.size(); i++) if (strs[i].second) memcpy(data.data() + off[i], strs[i].first, strs[i].second);
  Node n; n.ty = ty; n.name = name; n.nullable = nullable; n.length = (int64_t)strs.size();  // Utf8 and Binary share one layout
  n.bufs = {host_ref(a, off), BufRef::host(keep(a, std::move(data)).data(), tot)};
  if (valid) {
    std::vector<uint8_t> bits((strs.size() + 7) / 8, 0);
    int64_t nulls = 0;
    for (size_t i = 0; i < strs.size(); i++) { if ((*valid)[i]) bits[i >> 3] |= (uint8_t)(1u << (i & 7)); else nulls++; }
    n.null_count = nulls;
    if (nulls) { auto& k = keep(a, std::move(bits)); n.validity = BufRef::host(k.data(), k.size()); }
  }
  return n;
}
Node dict_node(const char* name, bool nullable, int64_t len, int64_t nulls, BufRef validity, BufRef indices, Node values) {
  Node n; n.ty = Ty::DictU32; n.name = name; n.nullable = nullable; n.length = len; n.null_count = nulls; n.validity = validity; n.bufs = {indices};
  n.dict.reset(new Node(std::move(values)));
  return n;
}
Node ree_node(const std::string& name, bool nullable, int64_t len, int64_t n_runs, BufRef run_ends, Node values) {
  Node n; n.ty = Ty::RunEnd; n.name = name; n.nullable = nullable; n.length = len;
  n.kids.push_back(int_node("run_ends", 32, true, false, n_runs, run_ends));
  values.name = "values"; values.nullable = true;
  n.kids.push_back(std::move(values));
  return n;
}

}  // namespace

static int d2h_vec(pa_agg* a, std::vector<uint32_t>& dst, const uint32_t* src, size_t n) {
  dst.resize(n);
  if (n) CK(cudaMemcpyAsync(dst.data(), src, n * 4, cudaMemcpyDeviceToHost, a->s_comp));
  return PA_OK;
}

// Buffers of a merged batch (mode B) that are spread over the shards: every shard holds the part that belongs to its rows /
// its runs / its range of the location-index stream. The plan only needs their total length; merge_impl.hpp copies each
// shard's part to (placement + part offset).
enum SliceKind : uint32_t { SL_TS = 1, SL_VALUE, SL_UUID, SL_STOFF, SL_STSIZE, SL_STREAM, SL_RUN_ENDS, SL_RUN_KEYS, SL_VALID, SL_TS_RUNS /* v1: int64 run values */ };
static BufRef sliced(uint32_t kind, uint32_t col, uint64_t len) { return BufRef{BufRef::SLICED, (const void*)(uintptr_t)(((uint64_t)kind << 16) | col), len}; }
struct MergeView {
  uint64_t NT;                                            // rows of the merged batch
  const std::vector<std::vector<uint32_t>>* kind_keys;    // run keys of the 8 kind-derived columns, all shards concatenated
};

// The v2 record's trailing columns — stacktrace_id, value, the eight kind-derived run-end columns, timestamp (arrow_v2.go:612-663
// order). Their sizes depend only on N and on the kind runs, which are known as soon as the label chain has run: a flush copies
// stacktrace_id / value / timestamp to the host while the frame ids are still uploading (early_copy_issue), at positions counted
// from the END of the stream, which is where these buffers sit.
static void append_tail_v2(pa_agg* a, const MergeView* mv, uint64_t N, const std::vector<std::vector<uint32_t>>& kind_keys, std::vector<Node>& cols) {
  auto rowbuf = [&](uint32_t kind, const void* p, uint64_t elem) { return mv ? sliced(kind, 0, N * elem) : BufRef::dev(p, N * elem); };
  auto runbuf = [&](uint32_t kind, uint32_t col, const void* p, uint64_t n, uint64_t elem) { return mv ? sliced(kind, col, n * elem) : BufRef::dev(p, n * elem); };
  const uint32_t nlab = a->n_label_cols;
  {
    Node id; id.ty = Ty::FixedBinary; id.name = "stacktrace_id"; id.byte_width = 16; id.length = (int64_t)N; id.bufs = {rowbuf(SL_UUID, a->d_uuid.p, 16)};
    id.metadata = {{"ARROW:extension:name", "arrow.uuid"}, {"ARROW:extension:metadata", ""}};
    cols.push_back(std::move(id));
  }
  cols.push_back(int_node("value", 64, true, false, (int64_t)N, rowbuf(SL_VALUE, a->d_value.p, 8)));
  // constant-ish columns: values per run built from the class of each run
  static const char* fixed_names[6] = {"producer", "sample_type", "sample_unit", "period_type", "period_unit", "temporality"};
  auto ree_run_ends = [&](uint32_t t) { return runbuf(SL_RUN_ENDS, nlab + t, a->cols[nlab + t].run_ends, mv ? (uint64_t)a->h_ctr.n_runs[nlab + t] : (uint64_t)kind_keys[t].size(), 4); };
  auto string_col = [&](uint32_t t) {
    const auto& keys = kind_keys[t];
    std::vector<std::pair<const uint8_t*, uint32_t>> strs;
    std::vector<uint8_t> valid(keys.size(), 1);
    for (size_t i = 0; i < keys.size(); i++) {
      if (keys[i] == kNull) { valid[i] = 0; strs.emplace_back(nullptr, 0); continue; }
      const std::string& s = a->kind_strings[t][keys[i]];
      strs.emplace_back((const uint8_t*)s.data(), (uint32_t)s.size());
    }
    return ree_node(fixed_names[t], t == 5, (int64_t)N, (int64_t)keys.size(), ree_run_ends(t), utf8_node(a, "values", true, strs, &valid));
  };
  for (uint32_t t = 0; t < 6; t++) cols.push_back(string_col(t));
  {
    std::vector<int64_t> pv; for (uint32_t k : kind_keys[6]) pv.push_back(a->period_vals[k]);
    std::vector<uint64_t> dv; for (uint32_t k : kind_keys[7]) dv.push_back(a->duration_vals[k]);
    cols.push_back(ree_node("period", false, (int64_t)N, (int64_t)pv.size(), ree_run_ends(6), int_node("values", 64, true, true, (int64_t)pv.size(), host_ref(a, pv))));
    cols.push_back(ree_node("duration", false, (int64_t)N, (int64_t)dv.size(), ree_run_ends(7), int_node("values", 64, false, true, (int64_t)dv.size(), host_ref(a, dv))));
  }
  {
    Node ts; ts.ty = Ty::TimestampNsUtc; ts.name = "timestamp"; ts.length = (int64_t)N; ts.bufs = {rowbuf(SL_TS, a->d_ts.p, 8)};
    cols.push_back(std::move(ts));
  }
}

// the record's columns as Nodes (device buffers are referenced, host-built ones are kept in a->hostbufs)
static int collect_nodes(pa_agg* a, const MergeView* mv, std::vector<Node>& cols, const std::function<int()>& after_small_copies = nullptr) {
  const uint64_t N = mv ? mv->NT : a->N;
  const Counters& c = a->h_ctr;
  auto rowbuf = [&](uint32_t kind, const void* p, uint64_t elem) { return mv ? sliced(kind, 0, N * elem) : BufRef::dev(p, N * elem); };
  auto runbuf = [&](uint32_t kind, uint32_t col, const void* p, uint64_t n, uint64_t elem) { return mv ? sliced(kind, col, n * elem) : BufRef::dev(p, n * elem); };
  auto validbuf = [&](uint32_t col, const void* p, uint64_t nr) { return mv ? sliced(SL_VALID, col, (nr + 7) / 8) : BufRef::dev(p, (nr + 7) / 8); };
  const uint32_t nlab = a->n_label_cols;
  const bool v1 = a->cfg.schema == PA_SCHEMA_V1;
  const Ty lab_ty = v1 ? Ty::Binary : Ty::Utf8;                 // v1 label dictionaries hold binary values (arrow.go:465-471)
  const std::string lab_prefix = v1 ? "labels." : "";           // v1: top-level columns "labels.<name>" (ColumnLabelsPrefix)
  const uint32_t n_loc = c.n_locations, n_lines = c.n_lines, n_fn = c.n_functions, n_idx = (uint32_t)c.n_indices64;

  const bool prof = getenv("PA_COLLECT_PROFILE") != nullptr;
  const double tp0 = now_ms();
  double tp1 = 0, tp2 = 0, tp3 = 0;
  // ---- small D2H: dictionary orders, constant-column run keys, function order
  std::vector<uint32_t> ord_type, ord_map, ord_bid, ord_file, ord_fn;
  std::vector<std::vector<uint32_t>> ord_lab(nlab), kind_keys(8);
  int rc;
  if ((rc = d2h_vec(a, ord_type, a->sd_order[0], c.n_dict_type)) || (rc = d2h_vec(a, ord_map, a->sd_order[1], c.n_dict_map)) ||
      (rc = d2h_vec(a, ord_bid, a->sd_order[2], c.n_dict_bid)) || (rc = d2h_vec(a, ord_file, a->sd_order[3], c.n_dict_file)) ||
      (rc = d2h_vec(a, ord_fn, a->fn_order, n_fn)))
    return rc;
  for (uint32_t i = 0; i < nlab; i++)
    if (c.last_nonnull_plus1[i] && (rc = d2h_vec(a, ord_lab[i], a->cols[i].order, c.n_dict[i]))) return rc;
  for (uint32_t t = v1 ? 6 : 0; t < 8; t++) {  // v1: the six string columns stay on the device as dictionary indices
    if (mv) { kind_keys[t] = (*mv->kind_keys)[t]; continue; }
    if ((rc = d2h_vec(a, kind_keys[t], a->cols[nlab + t].run_keys, c.n_runs[nlab + t]))) return rc;
  }
  std::vector<uint32_t> kind_order, n_kind_dict;
  if (v1 && ((rc = d2h_vec(a, kind_order, a->v1_kind_order, 64)) || (rc = d2h_vec(a, n_kind_dict, a->v1_n_kind_dict, 8)))) return rc;
  CK(cudaStreamSynchronize(a->s_comp));
  tp1 = now_ms();
  if (after_small_copies && (rc = after_small_copies())) return rc;  // (large copies that may run under the host work below)

  std::lock_guard<std::mutex> g(a->reg_mu);
  const StringPool& sp = a->sp;
  auto cstr = [&sp](uint32_t cid) { return std::make_pair(sp.ptr(cid), sp.len(cid)); };
  auto strs_of = [&](const std::vector<uint32_t>& ord) {
    std::vector<std::pair<const uint8_t*, uint32_t>> v;
    v.reserve(ord.size());
    for (uint32_t cid : ord) v.push_back(cstr(cid));
    return v;
  };

  // ---- label columns (sorted by name, slices.Sort in NewRecord arrow_v2.go:613-614)
  struct LabelOut { std::string name; Node node; };
  std::vector<LabelOut> labels;
  std::map<std::string, HostCol> touched;  // columns modified by external labels
  // resolve external labels (sid -> canonical id) now that all strings are registered
  std::vector<std::pair<std::string, std::string>> ext;
  for (auto& e : a->external) {
    if (e.first >= sp.sid2cid.size() || e.second >= sp.sid2cid.size()) return a->fail(PA_EINVAL, "external label refers to an unregistered string id");
    uint32_t n = sp.sid2cid[e.first], v = sp.sid2cid[e.second];
    ext.emplace_back(std::string((const char*)sp.ptr(n), sp.len(n)), std::string((const char*)sp.ptr(v), sp.len(v)));
  }
  auto label_dict_strings = [&](uint32_t i, std::vector<char>& decimals) {
    const ColPlan& cp = a->cols[i];
    std::vector<std::pair<const uint8_t*, uint32_t>> v;
    const auto& ord = ord_lab[i];
    v.reserve(ord.size());
    if (cp.type == COL_CPU || cp.type == COL_TID) {  // fmt.Sprint(cpu|tid) (:618,:621): decimal digits, formatted into one arena
      decimals.resize(ord.size() * 10);
      char* out = decimals.data();
      for (size_t k = 0; k < ord.size(); k++) {
        char tmp[10];
        int n = 0;
        uint32_t x = ord[k];
        do { tmp[n++] = (char)('0' + x % 10u); x /= 10u; } while (x);
        for (int d = 0; d < n; d++) out[d] = tmp[n - 1 - d];
        v.emplace_back((const uint8_t*)out, (uint32_t)n);
        out += n;
      }
    } else if (cp.type == COL_LS) {
      const std::vector<uint32_t>& vals = a->ls.vals[cp.ord];
      for (uint32_t local : ord) v.push_back(cstr(vals[local]));
    } else {
      for (uint32_t cid : ord) v.push_back(cstr(cid));
    }
    return v;
  };
  for (uint32_t i = 0; i < nlab; i++) {
    const ColPlan& cp = a->cols[i];
    if (!c.last_nonnull_plus1[i]) continue;  // no sample carried this label: the reference never created the builder
    bool is_ext = false;
    for (auto& e : ext) is_ext |= e.first == cp.name;
    std::vector<char> decimals;
    auto strs = label_dict_strings(i, decimals);
    if (is_ext && mv) return a->fail(PA_EINVAL, "merged batch: an external label may not share its name with a sample label");
    if (is_ext) {  // bring the column to the host; LabelAll is applied below
      HostCol hc;
      uint32_t nr = c.n_runs[i];
      std::vector<uint32_t> idx(nr), vw((nr + 31) / 32);
      hc.run_ends.resize(nr);
      CK(cudaMemcpy(hc.run_ends.data(), cp.run_ends, (size_t)nr * 4, cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(idx.data(), cp.run_keys, (size_t)nr * 4, cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(vw.data(), cp.validity, vw.size() * 4, cudaMemcpyDeviceToHost));
      hc.idx = idx;
      hc.valid.resize(nr);
      for (uint32_t k = 0; k < nr; k++) hc.valid[k] = (vw[k >> 5] >> (k & 31)) & 1u;
      for (auto& s : strs) hc.dict.emplace_back((const char*)s.first, s.second);
      // EnsureLength was only ever called up to the last row that carried the label: drop the
      // trailing one-row null runs the device produced beyond it (arrow_v2.go:550, :562)
      uint32_t len = c.last_nonnull_plus1[i];
      uint32_t trailing = (uint32_t)N - len;
      hc.run_ends.resize(nr - trailing); hc.idx.resize(nr - trailing); hc.valid.resize(nr - trailing);
      hc.len = len;
      touched.emplace(cp.name, std::move(hc));
      continue;
    }
    Node dictv = utf8_node(a, "values", true, strs, nullptr, lab_ty);
    uint32_t nr = c.n_runs[i];
    Node values = dict_node("values", true, nr, c.n_null[i], validbuf(i, cp.validity, nr), runbuf(SL_RUN_KEYS, i, cp.run_keys, nr, 4), std::move(dictv));
    labels.push_back(LabelOut{cp.name, ree_node(lab_prefix + cp.name, true, (int64_t)N, nr, runbuf(SL_RUN_ENDS, i, cp.run_ends, nr, 4), std::move(values))});
  }
  for (auto& e : ext) {  // LabelAll (arrow_v2.go:555-564), in flag order
    HostCol& hc = touched[e.first];
    // ree.Append(rows - len): finishRun closes the previous run at len (already stored as its run
    // end), then one run — possibly of length zero — covers [len, rows) with the external value
    hc.run_ends.push_back((int32_t)N);
    auto it = std::find(hc.dict.begin(), hc.dict.end(), e.second);
    if (it == hc.dict.end()) { hc.dict.push_back(e.second); it = hc.dict.end() - 1; }
    hc.idx.push_back((uint32_t)(it - hc.dict.begin()));
    hc.valid.push_back(1);
    hc.len = (int64_t)N;
  }
  for (auto& kv : touched) {
    HostCol& hc = kv.second;
    std::vector<std::pair<const uint8_t*, uint32_t>> strs;
    for (auto& s : hc.dict) strs.emplace_back((const uint8_t*)s.data(), (uint32_t)s.size());
    Node dictv = utf8_node(a, "values", true, strs, nullptr, lab_ty);
    int64_t nulls = 0;
    std::vector<uint8_t> bits((hc.valid.size() + 7) / 8, 0);
    for (size_t k = 0; k < hc.valid.size(); k++) { if (hc.valid[k]) bits[k >> 3] |= (uint8_t)(1u << (k & 7)); else nulls++; }
    BufRef vref = BufRef::none();
    if (nulls) { auto& kb = keep(a, std::move(bits)); vref = BufRef::host(kb.data(), kb.size()); }
    Node values = dict_node("values", true, (int64_t)hc.idx.size(), nulls, vref, host_ref(a, hc.idx), std::move(dictv));
    labels.push_back(LabelOut{kv.first, ree_node(lab_prefix + kv.first, true, (int64_t)N, (int64_t)hc.run_ends.size(), host_ref(a, hc.run_ends), std::move(values))});
  }
  std::sort(labels.begin(), labels.end(), [](const LabelOut& x, const LabelOut& y) { return x.name < y.name; });
  tp2 = now_ms();

  auto ree_run_ends_of = [&](uint32_t col) { return runbuf(SL_RUN_ENDS, col, a->cols[col].run_ends, c.n_runs[col], 4); };
  if (v1) {
    // ---- v1 sample record (reporter/arrow.go:274-316, ArrowSamplesField :484-503): label columns first, then the 11 fixed columns
    // (merged batch: the stacktrace_id dictionary is replicated on every shard, the run-end columns are sliced like the labels)
    for (auto& l : labels) cols.push_back(std::move(l.node));
    const uint32_t c_ord = nlab + 8, c_ts = nlab + 9, nu = c.n_unique;
    {
      Node ids; ids.ty = Ty::Binary; ids.name = "values"; ids.nullable = true; ids.length = nu;
      ids.bufs = {BufRef::dev(a->v1_id_off, ((uint64_t)nu + 1) * 4), BufRef::dev(a->v1_ids, (uint64_t)nu * 16)};
      uint32_t nr = c.n_runs[c_ord];  // run key == stack ordinal == dictionary index
      cols.push_back(ree_node("stacktrace_id", false, (int64_t)N, nr, ree_run_ends_of(c_ord),
                              dict_node("values", true, nr, 0, BufRef::none(), runbuf(SL_RUN_KEYS, c_ord, a->cols[c_ord].run_keys, nr, 4), std::move(ids))));
    }
    cols.push_back(int_node("value", 64, true, false, (int64_t)N, rowbuf(SL_VALUE, a->d_value.p, 8)));
    static const char* names[6] = {"producer", "sample_type", "sample_unit", "period_type", "period_unit", "temporality"};
    for (uint32_t t = 0; t < 6; t++) {
      std::vector<std::pair<const uint8_t*, uint32_t>> strs;
      for (uint32_t k = 0; k < n_kind_dict[t]; k++) {
        const std::string& sv = a->kind_strings[t][kind_order[t * 8 + k]];
        strs.emplace_back((const uint8_t*)sv.data(), (uint32_t)sv.size());
      }
      const ColPlan& cp = a->cols[nlab + t];
      uint32_t nr = c.n_runs[nlab + t];
      int64_t nulls = t == 5 ? (int64_t)c.n_null[nlab + t] : 0;  // memory samples carry a null temporality
      cols.push_back(ree_node(names[t], false, (int64_t)N, nr, ree_run_ends_of(nlab + t),
                              dict_node("values", true, nr, nulls, nulls ? validbuf(nlab + t, cp.validity, nr) : BufRef::none(),
                                        runbuf(SL_RUN_KEYS, nlab + t, cp.run_keys, nr, 4), utf8_node(a, "values", true, strs, nullptr, Ty::Binary))));
    }
    {
      std::vector<int64_t> pv; for (uint32_t k : kind_keys[6]) pv.push_back(a->period_vals[k]);
      std::vector<int64_t> dv; for (uint32_t k : kind_keys[7]) dv.push_back((int64_t)a->duration_vals[k]);
      cols.push_back(ree_node("period", false, (int64_t)N, (int64_t)pv.size(), ree_run_ends_of(nlab + 6), int_node("values", 64, true, true, (int64_t)pv.size(), host_ref(a, pv))));
      cols.push_back(ree_node("duration", false, (int64_t)N, (int64_t)dv.size(), ree_run_ends_of(nlab + 7), int_node("values", 64, true, true, (int64_t)dv.size(), host_ref(a, dv))));
    }
    {
      uint32_t nr = c.n_runs[c_ts];
      cols.push_back(ree_node("timestamp", false, (int64_t)N, nr, ree_run_ends_of(c_ts), int_node("values", 64, true, true, nr, runbuf(SL_TS_RUNS, c_ts, a->v1_ts_vals, nr, 8))));
    }
  } else {
  {
    Node ln; ln.ty = Ty::Struct; ln.name = "labels"; ln.nullable = false; ln.length = (int64_t)N;
    for (auto& l : labels) ln.kids.push_back(std::move(l.node));
    cols.push_back(std::move(ln));
  }

  // ---- stacktrace: ListView<Dict<u32, Location>> (arrow_v2.go:345-481)
  {
    // function dictionary values
    std::vector<uint8_t> views((size_t)n_fn * 16, 0), fvalid(n_fn, 1);
    std::vector<std::vector<uint8_t>> blocks;  // StringView data blocks: 32 KiB, first block with room wins
    std::vector<size_t> bcap;
    size_t cur = 0;
    int64_t sys_nulls = 0;
    for (uint32_t k = 0; k < n_fn; k++) {
      uint32_t sys = a->ft.fn_sys_cid[ord_fn[k]];
      if (sys == kNoId) { fvalid[k] = 0; sys_nulls++; continue; }
      const uint8_t* p = sp.ptr(sys);
      int32_t len = (int32_t)sp.len(sys);
      uint8_t* v = views.data() + (size_t)k * 16;
      memcpy(v, &len, 4);
      if (len <= 12) { memcpy(v + 4, p, (size_t)len); continue; }
      size_t need = (size_t)len;
      auto fresh = [&] { size_t cap = std::max<size_t>(need, 32 << 10); cap = (cap + 63) & ~(size_t)63; blocks.emplace_back(); blocks.back().reserve(cap); bcap.push_back(cap); cur = blocks.size() - 1; };
      if (blocks.empty()) fresh();
      else if (need > bcap[cur] - blocks[cur].size()) {
        bool found = false;
        for (size_t b = 0; b < blocks.size(); b++) if (need <= bcap[b] - blocks[b].size()) { cur = b; found = true; break; }
        if (!found) fresh();
      }
      int32_t bi = (int32_t)cur, of = (int32_t)blocks[cur].size();
      memcpy(v + 4, p, 4); memcpy(v + 8, &bi, 4); memcpy(v + 12, &of, 4);
      blocks[cur].insert(blocks[cur].end(), p, p + len);
    }
    Node sysn; sysn.ty = Ty::Utf8View; sysn.name = "system_name"; sysn.nullable = true; sysn.length = n_fn; sysn.null_count = sys_nulls;
    if (sys_nulls) {
      std::vector<uint8_t> bits((n_fn + 7) / 8, 0);
      for (uint32_t k = 0; k < n_fn; k++) if (fvalid[k]) bits[k >> 3] |= (uint8_t)(1u << (k & 7));
      auto& kb = keep(a, std::move(bits)); sysn.validity = BufRef::host(kb.data(), kb.size());
    }
    { auto& kv = keep(a, std::move(views)); sysn.bufs.push_back(BufRef::host(kv.data(), kv.size())); }
    for (auto& b : blocks) { size_t n = b.size(); auto& kb = keep(a, std::move(b)); sysn.bufs.push_back(BufRef::host(kb.data(), n)); }
    Node filen = dict_node("filename", true, n_fn, c.null_file, BufRef::dev(a->sd_valid[3], (n_fn + 7) / 8), BufRef::dev(a->sd_keys[3], (uint64_t)n_fn * 4),
                           utf8_node(a, "filename", true, strs_of(ord_file)));
    Node fstruct; fstruct.ty = Ty::Struct; fstruct.name = "function"; fstruct.length = n_fn;
    fstruct.kids.push_back(std::move(sysn));
    fstruct.kids.push_back(std::move(filen));
    fstruct.kids.push_back(int_node("start_line", 64, false, false, n_fn, BufRef::zeros((uint64_t)n_fn * 8)));
    Node fdict = dict_node("function", false, n_lines, 0, BufRef::none(), BufRef::dev(a->fn_keys, (uint64_t)n_lines * 4), std::move(fstruct));

    Node lstruct; lstruct.ty = Ty::Struct; lstruct.name = "item"; lstruct.nullable = true; lstruct.length = n_lines;
    lstruct.kids.push_back(int_node("line", 64, false, false, n_lines, BufRef::dev(a->lo.line_no, (uint64_t)n_lines * 8)));
    lstruct.kids.push_back(int_node("column", 64, false, false, n_lines, BufRef::zeros((uint64_t)n_lines * 8)));
    lstruct.kids.push_back(std::move(fdict));
    Node lines; lines.ty = Ty::ListView; lines.name = "lines"; lines.nullable = true; lines.length = n_loc; lines.null_count = (int64_t)n_loc - n_lines;
    lines.validity = BufRef::dev(a->lo.line_valid, (n_loc + 7) / 8);
    lines.bufs = {BufRef::dev(a->lo.line_off, (uint64_t)n_loc * 4), BufRef::dev(a->lo.line_size, (uint64_t)n_loc * 4)};
    lines.kids.push_back(std::move(lstruct));

    Node loc; loc.ty = Ty::Struct; loc.name = "item"; loc.nullable = true; loc.length = n_loc;
    loc.kids.push_back(int_node("address", 64, false, false, n_loc, BufRef::dev(a->lo.address, (uint64_t)n_loc * 8)));
    loc.kids.push_back(dict_node("frame_type", true, n_loc, 0, BufRef::none(), BufRef::dev(a->sd_keys[0], (uint64_t)n_loc * 4), utf8_node(a, "frame_type", true, strs_of(ord_type))));
    loc.kids.push_back(dict_node("mapping_file", true, n_loc, 0, BufRef::none(), BufRef::dev(a->sd_keys[1], (uint64_t)n_loc * 4), utf8_node(a, "mapping_file", true, strs_of(ord_map))));
    loc.kids.push_back(dict_node("mapping_build_id", true, n_loc, c.null_bid, BufRef::dev(a->sd_valid[2], (n_loc + 7) / 8), BufRef::dev(a->sd_keys[2], (uint64_t)n_loc * 4),
                                 utf8_node(a, "mapping_build_id", true, strs_of(ord_bid))));
    loc.kids.push_back(std::move(lines));
    Node locd = dict_node("item", true, n_idx, 0, BufRef::none(), mv ? sliced(SL_STREAM, 0, (uint64_t)n_idx * 4) : BufRef::dev(a->d_ustream.p, (uint64_t)n_idx * 4), std::move(loc));
    Node st; st.ty = Ty::ListView; st.name = "stacktrace"; st.nullable = true; st.length = (int64_t)N;
    st.bufs = {rowbuf(SL_STOFF, a->d_stoff.p, 4), rowbuf(SL_STSIZE, a->d_stsize.p, 4)};
    st.kids.push_back(std::move(locd));
    cols.push_back(std::move(st));
  }
  tp3 = now_ms();
  append_tail_v2(a, mv, N, kind_keys, cols);
  if (prof) fprintf(stderr, "collect_nodes: small copies %.3f ms, labels %.3f, stacktrace dictionaries %.3f, tail %.3f\n", tp1 - tp0, tp2 - tp1, tp3 - tp2, now_ms() - tp3);

  }

  return PA_OK;
}

// Called with the whole pass enqueued: wait for the label chain (it only needs the headers, so it finishes long before the ids are
// in), size the record's trailing columns, and start copying stacktrace_id / value / timestamp into their final places counted
// from the end of the output buffer: value and timestamp at once, stacktrace_id chunk by chunk as the hash kernel produces it.
static int early_copy_issue(pa_agg* a) {
  const uint32_t nlab = a->n_label_cols;
  CK(cudaEventSynchronize(a->ev_early));
  const Counters* ec = reinterpret_cast<const Counters*>(a->h_early);
  uint32_t* keys = reinterpret_cast<uint32_t*>(a->h_early + sizeof(Counters));
  uint32_t nr[8];
  for (uint32_t t = 0; t < 8; t++) {
    nr[t] = ec->n_runs[nlab + t];
    if (nr[t] > pa_agg::kEarlyMaxRuns) return PA_OK;  // a batch that alternates sample kinds: the ordinary copy-out handles it
    if (nr[t]) CK(cudaMemcpyAsync(keys + t * pa_agg::kEarlyMaxRuns, a->cols[nlab + t].run_keys, nr[t] * 4, cudaMemcpyDeviceToHost, a->s_aux));
  }
  CK(cudaStreamSynchronize(a->s_aux));
  std::vector<std::vector<uint32_t>> kind_keys(8);
  for (uint32_t t = 0; t < 8; t++) kind_keys[t].assign(keys + t * pa_agg::kEarlyMaxRuns, keys + t * pa_agg::kEarlyMaxRuns + nr[t]);
  std::vector<Node> tail;
  {
    std::lock_guard<std::mutex> g(a->reg_mu);
    append_tail_v2(a, nullptr, a->N, kind_keys, tail);
  }
  pa_agg::Early& e = a->early;
  for (auto& bd : StreamPlan::tail_distances(tail.data(), tail.size())) {
    if (bd.first.kind != BufRef::DEVICE) continue;
    if (bd.first.ptr == a->d_uuid.p) e.dist_uuid = bd.second;
    if (bd.first.ptr == a->d_value.p) e.dist_value = bd.second;
    if (bd.first.ptr == a->d_ts.p) e.dist_ts = bd.second;
  }
  e.out_end = a->out + (a->out_cap & ~63ull);
  if (!e.dist_uuid || !e.dist_value || !e.dist_ts || e.dist_uuid > (a->out_cap & ~63ull)) return PA_OK;
  const uint64_t N = a->N;
  CK(cudaStreamWaitEvent(a->s_d2h, a->ev_hdr_done, 0));
  CK(cudaMemcpyAsync(e.out_end - e.dist_ts, a->d_ts.p, N * 8, cudaMemcpyDeviceToHost, a->s_d2h));
  CK(cudaMemcpyAsync(e.out_end - e.dist_value, a->d_value.p, N * 8, cudaMemcpyDeviceToHost, a->s_d2h));
  for (size_t k = 0; k < a->chunk_rows.size(); k++) {
    const uint64_t r0 = a->chunk_rows[k].first, r1 = a->chunk_rows[k].second;
    CK(cudaStreamWaitEvent(a->s_d2h, a->hash_ev[k], 0));
    CK(cudaMemcpyAsync(e.out_end - e.dist_uuid + r0 * 16, a->d_uuid.as<uint8_t>() + r0 * 16, (r1 - r0) * 16, cudaMemcpyDeviceToHost, a->s_d2h));
  }
  CK(cudaEventRecord(a->ev_early_done, a->s_d2h));
  e.issued = true;
  return PA_OK;
}

// ---- PA_IPC_LZ4_FRAME_GPU, shared by single aggregators (lz4_gpu_stream below) and merge groups (merge_impl.hpp) --------
// The batch messages of `plan` (message 0 is the schema, copied verbatim): their metadata, and where each message's buffers
// start in a table of every buffer of messages 1.. in stream order.
static int lz4_read_messages(pa_agg* a, const StreamPlan& plan, std::vector<BatchMeta>* meta, std::vector<uint32_t>* buf0) {
  const size_t M = plan.messages.size();
  meta->assign(M, BatchMeta{});
  buf0->assign(M, 0);
  std::string why;
  uint32_t nbuf = 0;
  for (size_t m = 1; m < M; m++) {
    const StreamPlan::Message& g = plan.messages[m];
    const std::vector<uint8_t>& blob = plan.message_meta(m);
    if (!read_batch_meta(blob.data() + 8, (uint32_t)blob.size() - 8, &(*meta)[m], &why)) return a->fail(PA_EIO, why.c_str());
    if ((*meta)[m].buffers.size() != 2 * (g.p1 - g.p0)) return a->fail(PA_EIO, "stream plan and batch metadata disagree");
    (*buf0)[m] = nbuf;
    nbuf += (uint32_t)(g.p1 - g.p0);
  }
  return PA_OK;
}

// Host side of a block table: one Lz4Buf per buffer, the blocks it compresses (all of them, or one member's share of a merged
// buffer). A block's source is device memory, zeros (nullptr), or a place in the staging area, which starts with the host
// sources (`staged`, uploaded with one copy) and continues with room the caller fills on the device.
struct Lz4Table {
  std::vector<Lz4Blk> blks;
  std::vector<Lz4Buf> bufs;
  std::vector<uint8_t> staged;
  uint64_t staging = 0;                                  // staging bytes: staged.size() + device-filled room
  std::vector<std::pair<size_t, uint64_t>> at_staged;    // (block, offset of its source in the staging area)
  void buffer(uint64_t len) { bufs.push_back(Lz4Buf{len, (uint32_t)blks.size(), 0}); }
  void block(const uint8_t* src, uint32_t len) { blks.push_back(Lz4Blk{src, len, (uint32_t)bufs.size() - 1}); bufs.back().nblk++; }
  void block_staged(uint64_t off, uint32_t len) { at_staged.emplace_back(blks.size(), off); block(nullptr, len); }
  uint64_t stage_host(const void* p, uint64_t n) {  // offset of the copy in the staging area
    const uint64_t at = staged.size();
    staged.insert(staged.end(), (const uint8_t*)p, (const uint8_t*)p + n);
    staging = std::max<uint64_t>(staging, staged.size());
    return at;
  }
  uint64_t reserve(uint64_t n) { staging = std::max<uint64_t>(staging, staged.size()); const uint64_t at = staging; staging += n; return at; }
};
// Its device side, carved out of a->d_lz4: the table, per-block sizes and frame offsets, per-buffer frame sizes and destinations,
// the staging area, and one 64 KiB slot per block for k_lz4_compress.
struct Lz4Dev {
  Lz4Blk* blks = nullptr;
  Lz4Buf* bufs = nullptr;
  uint32_t* size = nullptr;
  uint64_t *off = nullptr, *frame = nullptr, *dst = nullptr;
  uint8_t *staging = nullptr, *slots = nullptr;
  size_t nb = 0, nbuf = 0;
};
// Sizes a->d_lz4 for `t` and points each staged block at its source. Then lz4_upload, the caller's device-side staging, and
// lz4_compress.
static int lz4_alloc(pa_agg* a, Lz4Table& t, Lz4Dev* d) {
  const size_t nb = t.blks.size(), nbuf = t.bufs.size();
  auto al = [](size_t v) { return (v + 255) & ~(size_t)255; };
  const size_t o_bufs = al(nb * sizeof(Lz4Blk)), o_size = o_bufs + al(nbuf * sizeof(Lz4Buf)), o_off = o_size + al(nb * 4), o_frame = o_off + al(nb * 8),
               o_dst = o_frame + al(nbuf * 8), o_staged = o_dst + al(nbuf * 8), o_slots = o_staged + al(t.staging), bytes = o_slots + nb * kLz4Block;
  CK(a->d_lz4.ensure(std::max<size_t>(bytes, 256)));
  uint8_t* p = a->d_lz4.as<uint8_t>();
  d->blks = (Lz4Blk*)p;
  d->bufs = (Lz4Buf*)(p + o_bufs);
  d->size = (uint32_t*)(p + o_size);
  d->off = (uint64_t*)(p + o_off); d->frame = (uint64_t*)(p + o_frame); d->dst = (uint64_t*)(p + o_dst);
  d->staging = p + o_staged; d->slots = p + o_slots;
  d->nb = nb; d->nbuf = nbuf;
  for (auto& hb : t.at_staged) t.blks[hb.first].src = d->staging + hb.second;
  return PA_OK;
}
// Uploads the table and the host sources.
static int lz4_upload(pa_agg* a, const Lz4Table& t, const Lz4Dev& d, cudaStream_t s) {
  if (d.nb) CK(cudaMemcpyAsync(d.blks, t.blks.data(), d.nb * sizeof(Lz4Blk), cudaMemcpyHostToDevice, s));
  if (d.nbuf) CK(cudaMemcpyAsync(d.bufs, t.bufs.data(), d.nbuf * sizeof(Lz4Buf), cudaMemcpyHostToDevice, s));
  if (!t.staged.empty()) CK(cudaMemcpyAsync(d.staging, t.staged.data(), t.staged.size(), cudaMemcpyHostToDevice, s));
  return PA_OK;
}
// k_lz4_compress + k_lz4_layout (timed as T_LZ4, which this call resets): per block its compressed size and offset inside its
// buffer's share of blocks, per buffer 11 + the bytes of those blocks (frame header, blocks with their sizes, EndMark).
static int lz4_compress(pa_agg* a, const Lz4Dev& d, cudaStream_t s) {
  Timer& tm = a->tm[T_LZ4];
  tm.launches = 0;
  CK(cudaEventRecord(tm.a, s));
  if (d.nb) { k_lz4_compress<<<(unsigned)((d.nb + kLz4Warps - 1) / kLz4Warps), kLz4Warps * 32, 0, s>>>(d.blks, (uint32_t)d.nb, d.slots, d.size); tm.launches++; }
  if (d.nbuf) { k_lz4_layout<<<(unsigned)((d.nbuf + kWarps - 1) / kWarps), kThreads, 0, s>>>(d.bufs, (uint32_t)d.nbuf, d.size, d.off, d.frame); tm.launches++; }
  CK(cudaGetLastError());
  CK(cudaEventRecord(tm.b, s));
  return PA_OK;
}

// Layout of an LZ4_FRAME stream from each buffer's length and whole frame size: a buffer is its int64 length and its frame, or -1
// and its raw bytes when the frame is not smaller than the buffer.
struct Lz4Layout {
  std::vector<std::vector<uint8_t>> metas;  // per message: encapsulated metadata (the schema's verbatim)
  std::vector<uint64_t> at, body_len;       // per message: offset in the stream, body bytes
  std::vector<uint64_t> buf_at, buf_size;   // per buffer: offset inside its message's body, bytes (prefix included; 0 = empty)
  std::vector<uint8_t> raw;                 // per buffer: stored raw
  uint64_t total = 0;                       // stream bytes, end-of-stream marker included
  uint64_t body_of(size_t m) const { return at[m] + metas[m].size(); }
};
static void lz4_layout(const StreamPlan& plan, const std::vector<BatchMeta>& meta, const std::vector<uint32_t>& buf0, const std::vector<uint64_t>& len,
                       const std::vector<uint64_t>& frame, Lz4Layout* L) {
  const size_t M = plan.messages.size();
  L->metas.assign(M, {});
  L->at.assign(M, 0); L->body_len.assign(M, 0);
  L->buf_at.assign(len.size(), 0); L->buf_size.assign(len.size(), 0); L->raw.assign(len.size(), 0);
  uint64_t total = 0;
  for (size_t m = 0; m < M; m++) {
    if (m == 0) {
      L->metas[m] = plan.message_meta(0);
    } else {
      const size_t n = plan.messages[m].p1 - plan.messages[m].p0;
      std::vector<int64_t> sizes(n), offs;
      for (size_t i = 0; i < n; i++) {
        const size_t b = buf0[m] + i;
        sizes[i] = len[b] ? 8 + (int64_t)std::min<uint64_t>(frame[b], len[b]) : 0;
        L->buf_size[b] = (uint64_t)sizes[i];
        L->raw[b] = len[b] && frame[b] >= len[b];
      }
      int64_t bl = 0;
      L->metas[m] = lz4_batch_message(meta[m], sizes, &offs, &bl);
      for (size_t i = 0; i < n; i++) L->buf_at[buf0[m] + i] = (uint64_t)offs[i];
      L->body_len[m] = (uint64_t)bl;
    }
    L->at[m] = total;
    total += L->metas[m].size() + L->body_len[m];
  }
  L->total = total + 8;
}

// PA_IPC_LZ4_FRAME_GPU: writes the stream `plan` describes to a->out with every record and dictionary batch body compressed
// on the device (the framing of ipc_compress_lz4; only the compressed bodies cross PCIe). The host assembles the metadata with
// the same rewrite as the host mode, from the per-buffer frame sizes. *d2h_ms: the copy-out of the bodies.
static int lz4_gpu_stream(pa_agg* a, const StreamPlan& plan, cudaStream_t s, uint64_t* out_len, float* d2h_ms) {
  const size_t M = plan.messages.size();
  std::vector<BatchMeta> meta;
  std::vector<uint32_t> buf0;
  if (int rc = lz4_read_messages(a, plan, &meta, &buf0)) return rc;
  Lz4Table t;
  std::vector<uint64_t> len;
  for (size_t m = 1; m < M; m++)
    for (size_t i = plan.messages[m].p0; i < plan.messages[m].p1; i++) {
      const BufRef& r = plan.placements[i].src;
      if (r.len && r.kind != BufRef::DEVICE && r.kind != BufRef::HOST && r.kind != BufRef::ZEROS) return a->fail(PA_EINVAL, "buffer without a source");
      t.buffer(r.len);
      len.push_back(r.len);
      const uint64_t h = r.kind == BufRef::HOST && r.len ? t.stage_host(r.ptr, r.len) : 0;
      for (uint64_t o = 0; o < r.len; o += kLz4Block) {
        const uint32_t n = (uint32_t)std::min<uint64_t>(kLz4Block, r.len - o);
        if (r.kind == BufRef::HOST) t.block_staged(h + o, n);
        else t.block(r.kind == BufRef::DEVICE ? (const uint8_t*)r.ptr + o : nullptr, n);
      }
    }
  Lz4Dev d;
  if (int rc = lz4_alloc(a, t, &d)) return rc;
  if (int rc = lz4_upload(a, t, d, s)) return rc;
  if (int rc = lz4_compress(a, d, s)) return rc;
  Timer& tm = a->tm[T_LZ4];
  const size_t nb = d.nb, nbuf = d.nbuf;
  std::vector<uint64_t> frame(nbuf);
  if (nbuf) CK(cudaMemcpyAsync(frame.data(), d.frame, nbuf * 8, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));

  Lz4Layout L;
  lz4_layout(plan, meta, buf0, len, frame, &L);
  std::vector<uint64_t> body_dev(M, 0), dst(nbuf, 0);
  uint64_t dev_total = 0;
  for (size_t m = 1; m < M; m++) {
    for (size_t i = 0; i < plan.messages[m].p1 - plan.messages[m].p0; i++) {
      const size_t b = buf0[m] + i;
      dst[b] = (dev_total + L.buf_at[b]) | (L.raw[b] ? 1ull << 63 : 0);
    }
    body_dev[m] = dev_total;
    dev_total += L.body_len[m];
  }
  const uint64_t total = L.total;
  CK(a->d_lz4_body.ensure(std::max<uint64_t>(dev_total, 256)));
  if (nbuf) CK(cudaMemcpyAsync(d.dst, dst.data(), nbuf * 8, cudaMemcpyHostToDevice, s));
  CK(cudaEventRecord(a->ev_lz4p0, s));
  if (nb) {
    k_lz4_pack<<<(unsigned)((nb + kWarps - 1) / kWarps), kThreads, 0, s>>>(d.blks, (uint32_t)nb, d.bufs, d.slots, d.size, d.off, d.frame, d.dst, a->d_lz4_body.as<uint8_t>());
    tm.launches++;
  }
  CK(cudaGetLastError());
  CK(cudaEventRecord(a->ev_lz4p1, s));
  if (total > a->out_cap) {
    CK(cudaStreamSynchronize(a->s_d2h));
    if (a->out) cudaFreeHost(a->out);
    a->out = nullptr;
    a->out_cap = 0;
    uint64_t want = total + total / 4 + 4096;
    if (cudaHostAlloc((void**)&a->out, want, cudaHostAllocDefault) != cudaSuccess) return a->fail(PA_ENOMEM, "pinned output allocation failed");
    a->out_cap = want;
  }
  CK(cudaEventRecord(a->ev_d2h0, s));
  for (size_t m = 0; m < M; m++)
    if (L.body_len[m]) CK(cudaMemcpyAsync(a->out + L.body_of(m), a->d_lz4_body.as<uint8_t>() + body_dev[m], L.body_len[m], cudaMemcpyDeviceToHost, s));
  CK(cudaEventRecord(a->ev_d2h1, s));
  for (size_t m = 0; m < M; m++) memcpy(a->out + L.at[m], L.metas[m].data(), L.metas[m].size());
  const uint32_t eos[2] = {0xFFFFFFFFu, 0u};
  memcpy(a->out + total - 8, eos, 8);
  CK(cudaStreamSynchronize(s));
  float ms = 0, pack = 0;
  cudaEventElapsedTime(&ms, tm.a, tm.b);
  cudaEventElapsedTime(&pack, a->ev_lz4p0, a->ev_lz4p1);
  tm.ms = (double)ms + pack;
  cudaEventElapsedTime(d2h_ms, a->ev_d2h0, a->ev_d2h1);
  *out_len = total;
  return PA_OK;
}

static int collect(pa_agg* a, pa_agg_result* res) {
  memset(res, 0, sizeof *res);
  if (!a->processed) return a->fail(PA_EINVAL, "collect before process");
  if (a->merged_part) return a->fail(PA_EINVAL, "this batch is one shard of a merged record: collect it through pa_merge_collect (or pa_agg_discard it)");
  CK(cudaSetDevice(a->device));
  const uint64_t N = a->N;
  a->hostbufs.clear();
  if (N == 0) { release_staged(a); return PA_OK; }  // reference skips empty batches (:1775-1778)
  double t0 = now_ms();
  const Counters& c = a->h_ctr;
  const bool v1 = a->cfg.schema == PA_SCHEMA_V1;
  auto second_wave = [&]() -> int {
    if (a->early.issued && a->early.out_end == a->out + (a->out_cap & ~63ull)) {
      // second wave of the early copy-out: with the pass finished the length of the location-index stream is known, and with it the
      // positions (from the end) of the three buffers in front of stacktrace_id. They leave on the copy-out stream while the host
      // assembles the dictionaries (collect_nodes); the plan below confirms the positions like those of the first wave.
      pa_agg::Early& e = a->early;
      const uint64_t nidx = c.n_indices64, pad = 7;
      e.dist_stream = e.dist_uuid + ((nidx * 4 + pad) & ~pad);
      e.dist_stsize = e.dist_stream + ((N * 4 + pad) & ~pad);
      e.dist_stoff = e.dist_stsize + ((N * 4 + pad) & ~pad);
      if (e.dist_stoff <= (a->out_cap & ~63ull)) {
        CK(cudaMemcpyAsync(e.out_end - e.dist_stoff, a->d_stoff.p, N * 4, cudaMemcpyDeviceToHost, a->s_d2h));
        CK(cudaMemcpyAsync(e.out_end - e.dist_stsize, a->d_stsize.p, N * 4, cudaMemcpyDeviceToHost, a->s_d2h));
        if (nidx) CK(cudaMemcpyAsync(e.out_end - e.dist_stream, a->d_ustream.p, nidx * 4, cudaMemcpyDeviceToHost, a->s_d2h));
        CK(cudaEventRecord(a->ev_early_done, a->s_d2h));
      } else {
        e.dist_stream = e.dist_stsize = e.dist_stoff = 0;
      }
    }
    return PA_OK;
  };
  std::vector<Node> cols;
  {
    int rcn = collect_nodes(a, nullptr, cols, second_wave);
    if (rcn) return rcn;
  }
  const double t_nodes = now_ms();
  const uint32_t n_loc = c.n_locations, n_fn = c.n_functions, n_idx = (uint32_t)c.n_indices64;

  // ---- plan the stream and fill it
  StreamPlan plan;
  plan.build(cols, {{"parca_write_schema_version", v1 ? "v1" : "v2"}}, (int64_t)N);
  const double t_plan = now_ms();
  if (a->cfg.ipc_compression == PA_IPC_LZ4_FRAME_GPU) {
    uint64_t len = 0;
    float d2h = 0, h2d = 0;
    if (int rc = lz4_gpu_stream(a, plan, a->s_comp, &len, &d2h)) return rc;
    cudaEventElapsedTime(&h2d, a->ev_h2d0, a->ev_h2d1);
    res->ipc = a->out; res->ipc_len = len; res->n_rows = N; res->n_unique_stacks = c.n_unique; res->n_locations = c.n_locations;
    res->n_functions = c.n_functions; res->n_location_indices = (uint32_t)c.n_indices64; res->gpu_launches = a->launches;
    res->h2d_ms = h2d; res->gpu_ms = a->tm[T_TOTAL].ms; res->d2h_ms = d2h; res->host_ms = std::max(0.0, now_ms() - t0 - d2h - a->tm[T_LZ4].ms);
    release_staged(a);
    return PA_OK;
  }
  if (plan.total > a->out_cap) {
    if (a->early.issued) { CK(cudaStreamSynchronize(a->s_d2h)); a->early.issued = false; }  // the early copies went into the buffer that is too small
    if (a->out) cudaFreeHost(a->out);
    a->out = nullptr;
    a->out_cap = 0;
    uint64_t want = plan.total + plan.total / 4 + 4096;
    if (cudaHostAlloc((void**)&a->out, want, cudaHostAllocDefault) != cudaSuccess) return a->fail(PA_ENOMEM, "pinned output allocation failed");
    a->out_cap = want;
  }
  double t1 = now_ms();
  // a stream whose tail was copied out early ends where those copies assumed it would
  const pa_agg::Early& e = a->early;
  const bool anchored = e.issued && e.out_end == a->out + (a->out_cap & ~63ull) && plan.total <= (a->out_cap & ~63ull);
  uint8_t* const base = anchored ? e.out_end - plan.total : a->out;
  cudaEvent_t d0 = a->ev_d2h0, d1 = a->ev_d2h1;
  CK(cudaEventRecord(d0, a->s_comp));
  auto placed_early = [&](const Placement& p) {
    const uint64_t dist = plan.total - p.at;
    return anchored && ((p.src.ptr == a->d_ts.p && dist == e.dist_ts) || (p.src.ptr == a->d_value.p && dist == e.dist_value) || (p.src.ptr == a->d_uuid.p && dist == e.dist_uuid) ||
                        (p.src.ptr == a->d_stoff.p && dist == e.dist_stoff) || (p.src.ptr == a->d_stsize.p && dist == e.dist_stsize) ||
                        (p.src.ptr == a->d_ustream.p && dist == e.dist_stream));
  };
  if (e.issued) {
    // an early copy that is NOT where the plan puts its buffer may still be landing somewhere in the output: let it finish before
    // anything else is written there (the ordinary copies below then overwrite whatever it hit)
    int hits = 0;
    for (auto& p : plan.placements) if (p.src.kind == BufRef::DEVICE && p.src.len && placed_early(p)) hits++;
    const int expected = 3 + (e.dist_stoff ? 2 : 0) + (e.dist_stream && c.n_indices64 ? 1 : 0);
    if (hits != expected) CK(cudaStreamSynchronize(a->s_d2h));
  }
  for (auto& p : plan.placements) {
    if (p.src.kind != BufRef::DEVICE || !p.src.len || placed_early(p)) continue;
    CK(cudaMemcpyAsync(base + p.at, p.src.ptr, p.src.len, cudaMemcpyDeviceToHost, a->s_comp));
  }
  CK(cudaEventRecord(d1, a->s_comp));
  if (e.issued) CK(cudaStreamWaitEvent(a->s_comp, a->ev_early_done, 0));
  const double t_enq = now_ms();
  plan.write_host_parts(base);  // metadata, host-built buffers, zero fills and padding overlap the D2H
  const double t_hostparts = now_ms();
  CK(cudaStreamSynchronize(a->s_comp));
  if (getenv("PA_COLLECT_PROFILE"))
    fprintf(stderr, "collect: nodes %.3f ms, plan %.3f, alloc+enqueue %.3f, host parts %.3f, wait for copies %.3f (anchored %d)\n", t_nodes - t0, t_plan - t_nodes,
            t_enq - t_plan, t_hostparts - t_enq, now_ms() - t_hostparts, (int)anchored);
  const uint8_t* stream = base;
  uint64_t stream_len = plan.total;
  if (a->cfg.ipc_compression == PA_IPC_LZ4_FRAME) {  // network-path framing (ipc.WithLZ4(), :1851); host work, counted in host_ms
    std::string why;
    if (!ipc_compress_lz4(base, plan.total, a->comp_out, &why)) return a->fail(PA_EIO, why.c_str());
    stream = a->comp_out.data();
    stream_len = a->comp_out.size();
  }
  double t2 = now_ms();
  float d2h = 0, h2d = 0;
  cudaEventElapsedTime(&d2h, d0, d1);
  cudaEventElapsedTime(&h2d, a->ev_h2d0, a->ev_h2d1);
  res->ipc = stream; res->ipc_len = stream_len; res->n_rows = N; res->n_unique_stacks = c.n_unique; res->n_locations = n_loc;
  res->n_functions = n_fn; res->n_location_indices = n_idx; res->gpu_launches = a->launches;
  res->h2d_ms = h2d; res->gpu_ms = a->tm[T_TOTAL].ms; res->d2h_ms = d2h; res->host_ms = (t1 - t0) + (t2 - t1) - d2h;
  release_staged(a);
  return PA_OK;
}

// ---------------------------------------------------------------------------------------------
// v1 stacktrace record: buildStacktraceRecord (parca_reporter.go:1545-1739) + LocationsWriter.NewRecord
// (arrow.go:230-254) + IPC. Off the per-interval hot path (it runs for the stacks the server asks for, or for
// the stacks not yet logged in offline mode), but the same building blocks: scans, gathers, first-occurrence ranks.
static int stacktraces(pa_agg* a, const uint8_t* ids, uint64_t n, pa_agg_result* res) {
  memset(res, 0, sizeof *res);
  if (a->cfg.schema != PA_SCHEMA_V1) return a->fail(PA_EINVAL, "pa_agg_stacktraces needs a PA_SCHEMA_V1 aggregator");
  if (a->staged >= 0) return a->fail(PA_EINVAL, "collect the staged batch before asking for stacktraces");
  if (n && !ids) return a->fail(PA_EINVAL, "null ids");
  if (n > 0x7FFFFFFFull / 16) return a->fail(PA_ERANGE, "stacktrace_id offsets exceed int32");
  CK(cudaSetDevice(a->device));
  const double t0 = now_ms();
  a->hostbufs.clear();
  int rc = upload_tables(a, false);  // frames may have been registered since the last flush
  if (rc) return rc;
  cudaStream_t s = a->s_comp;
  const uint32_t n32 = (uint32_t)n;
  const size_t Nn = std::max<size_t>(n, 1);
  Counters* ctr = a->d_ctr.as<Counters>();
  Timer tm{};

  // ---- phase 1: look the ids up, size the flattened location list
  uint8_t *d_ids = nullptr, *complete_b = nullptr, *listv_b = nullptr;
  uint32_t *q_slot = nullptr, *q_nloc = nullptr, *complete_w = nullptr, *listv_w = nullptr;
  int* loc_off = nullptr;
  {
    struct Req { void** pp; size_t bytes; };
    std::vector<Req> reqs;
    auto want = [&reqs](auto** pp, size_t bytes) { reqs.push_back(Req{(void**)pp, (bytes + 255) & ~(size_t)255}); };
    want(&d_ids, Nn * 16); want(&q_slot, Nn * 4); want(&q_nloc, Nn * 4); want(&loc_off, (Nn + 1) * 4); want(&complete_b, Nn); want(&listv_b, Nn);
    want(&complete_w, (Nn / 32 + 2) * 4); want(&listv_w, (Nn / 32 + 2) * 4);
    size_t tot = 0;
    for (auto& r : reqs) tot += r.bytes;
    CK(a->d_st1.ensure(tot));
    size_t off = 0;
    for (auto& r : reqs) { *r.pp = a->d_st1.as<uint8_t>() + off; off += r.bytes; }
  }
  // host copy: also the stacktrace_id column's data (the inner buffer stays put when hostbufs grows)
  const uint8_t* ids_host = keep(a, std::vector<uint8_t>(ids, ids + n * 16)).data();
  CK(cudaEventRecord(a->tm[T_TOTAL].a, s));
  CK(cudaMemsetAsync(ctr, 0, sizeof(Counters), s));
  if (n) CK(cudaMemcpyAsync(d_ids, ids_host, n * 16, cudaMemcpyHostToDevice, s));
  const StoreSlot* st = a->d_store.as<StoreSlot>();
  const uint32_t smask = (uint32_t)(a->store_slots - 1);
  a->store_epoch++;  // one tick of the LRU clock per request: its Gets are more recent than every access before it
  if (a->store_epoch >= (1ull << 32)) return a->fail(PA_ERANGE, "stack store: access clock overflow");
  k_st_lookup<<<small_grid(a, n), kThreads, 0, s>>>(d_ids, n32, st, smask, q_slot, q_nloc, a->d_store_stamp.as<unsigned long long>(), a->store_epoch << 32);
  launch_scan(a, StLocF{q_nloc, n32, loc_off, ctr}, 1, tm, small_grid(a, n), s, a->d_partial);
  tm.launches += 1;
  CK(cudaMemcpyAsync(a->h_ctr_pinned, ctr, sizeof(Counters), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  if (a->h_ctr_pinned->err & ERR_INDEX_OVERFLOW) return a->fail(PA_ERANGE, "flattened locations exceed int32 list offsets");
  const uint64_t L = a->h_ctr_pinned->n_locations;

  // ---- phase 2: per-location and per-line columns, run-end encoding, dictionaries
  const size_t Ln = std::max<size_t>(L, 1);
  uint32_t unknown_cid = a->cid_unknown;
  size_t S2;
  {
    std::lock_guard<std::mutex> g(a->reg_mu);
    if (a->cfg.unknown_frame_type_sid) {
      if (a->cfg.unknown_frame_type_sid >= a->sp.sid2cid.size()) return a->fail(PA_EINVAL, "unknown_frame_type_sid is not a registered string id");
      unknown_cid = a->sp.sid2cid[a->cfg.unknown_frame_type_sid];
    }
    S2 = std::max<uint32_t>(a->sp.count(), 1);
  }
  const uint32_t missing_cid = a->cid_missing;
  uint32_t* loc_fid = nullptr;
  StLocOut o{};
  uint32_t *hasline_w = nullptr, *run_key[4] = {}, *run_valid[4] = {}, *d_first[5] = {}, *d_rank[5] = {}, *d_order[5] = {}, *d_bits[5] = {}, *d_wp[5] = {};
  int* run_end[4] = {};
  size_t ff_bytes = 0;
  {
    struct Req { void** pp; size_t bytes; int cls; };
    std::vector<Req> reqs;
    auto want = [&reqs](auto** pp, size_t bytes, int cls = 1) { reqs.push_back(Req{(void**)pp, (bytes + 255) & ~(size_t)255, cls}); };
    for (int d = 0; d < 5; d++) want(&d_first[d], S2 * 4, 0);
    want(&loc_fid, Ln * 4); want(&o.address, Ln * 8); want(&o.type_key, Ln * 4); want(&o.map_key, Ln * 4); want(&o.bid_key, Ln * 4);
    want(&o.line_off, (Ln + 1) * 4); want(&o.has_line, Ln); want(&hasline_w, (Ln / 32 + 2) * 4); want(&o.line_no, Ln * 8); want(&o.column, Ln * 8);
    want(&o.fn_key, Ln * 4); want(&o.file_key, Ln * 4);
    for (int c = 0; c < 4; c++) { want(&run_key[c], Ln * 4); want(&run_end[c], Ln * 4); want(&run_valid[c], (Ln / 32 + 2) * 4); }
    for (int d = 0; d < 5; d++) { want(&d_rank[d], S2 * 4); want(&d_order[d], S2 * 4); want(&d_bits[d], (Ln / 32 + 2) * 4); want(&d_wp[d], (Ln / 32 + 2) * 4); }
    size_t cls_bytes[2] = {0, 0};
    for (auto& r : reqs) cls_bytes[r.cls] += r.bytes;
    CK(a->d_arena.ensure(cls_bytes[0] + cls_bytes[1]));
    size_t off[2] = {0, cls_bytes[0]};
    for (auto& r : reqs) { *r.pp = a->d_arena.as<uint8_t>() + off[r.cls]; off[r.cls] += r.bytes; }
    ff_bytes = cls_bytes[0];
  }
  std::vector<FoJob> jobs(5);
  const uint32_t* job_n[5] = {&ctr->n_runs[0], &ctr->n_runs[1], &ctr->n_runs[2], &ctr->n_runs[3], &ctr->n_lines};
  for (int d = 0; d < 5; d++) {
    FoJob j{};
    j.keys = d < 4 ? run_key[d] : o.fn_key; j.n_ptr = job_n[d]; j.first = d_first[d]; j.universe = (uint32_t)S2; j.rank = d_rank[d]; j.order = d_order[d];
    j.out = d < 4 ? run_key[d] : o.fn_key; j.validity = d < 4 ? run_valid[d] : nullptr; j.bitmap = d_bits[d]; j.wprefix = d_wp[d];
    j.n_unique = &ctr->n_dict[d]; j.n_null = d < 4 ? &ctr->n_null[d] : nullptr; j.nullable = d < 4 ? 1u : 0u; j.ctr = ctr;
    jobs[d] = j;
  }
  rc = upload_descriptors(a, jobs.data(), jobs.size() * sizeof(FoJob), nullptr, 0);
  if (rc) return rc;
  CK(cudaMemsetAsync(a->d_arena.p, 0xFF, ff_bytes, s));
  FrameTableV1 ft1{(const unsigned long long*)a->m_addr.ptr(), a->m_type.ptr(), a->m1_map.ptr(), a->m1_bid.ptr(), a->m1_fn.ptr(), a->m1_file.ptr(),
                   (const unsigned long long*)a->m1_line.ptr(), (const unsigned long long*)a->m1_col.ptr(), a->m1_complete.ptr()};
  k_st_expand<<<small_grid(a, std::max<uint64_t>(n * 32, L)), kThreads, 0, s>>>(n32, q_slot, loc_off, st, a->d_store_arena.as<uint32_t>(), ft1.complete, loc_fid,
                                                                                    complete_b, listv_b, ctr);
  k_pack_bits<<<small_grid(a, n), kThreads, 0, s>>>(complete_b, nullptr, n32, complete_w);
  k_pack_bits<<<small_grid(a, n), kThreads, 0, s>>>(listv_b, nullptr, n32, listv_w);
  launch_scan(a, StLinesF{ctr, ctr, loc_fid, ft1, o, unknown_cid, missing_cid}, 1, tm, small_grid(a, L), s, a->d_partial);
  k_pack_bits<<<small_grid(a, L), kThreads, 0, s>>>(o.has_line, &ctr->n_locations, 0, hasline_w);
  StRunF rf{};
  rf.c[0] = StRunCol{o.type_key, &ctr->n_locations, run_key[0], run_end[0]};
  rf.c[1] = StRunCol{o.map_key, &ctr->n_locations, run_key[1], run_end[1]};
  rf.c[2] = StRunCol{o.bid_key, &ctr->n_locations, run_key[2], run_end[2]};
  rf.c[3] = StRunCol{o.file_key, &ctr->n_lines, run_key[3], run_end[3]};
  rf.ctr_w = ctr;
  launch_scan(a, rf, 4, tm, small_grid(a, L), s, a->d_partial);
  run_fo_jobs(a, a->d_jobs.as<FoJob>(), 0, 5, true, tm, Ln, S2, true, s, a->d_partial);
  tm.launches += 4;
  CK(cudaMemcpyAsync(a->h_ctr_pinned, ctr, sizeof(Counters), cudaMemcpyDeviceToHost, s));
  CK(cudaEventRecord(a->tm[T_TOTAL].b, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  const Counters c = *a->h_ctr_pinned;
  const uint64_t NL = c.n_lines;

  // ---- phase 3: dictionary values (host strings in rank order) and the IPC stream
  std::vector<uint32_t> ord[5];
  for (int d = 0; d < 5; d++) if ((rc = d2h_vec(a, ord[d], d_order[d], c.n_dict[d]))) return rc;
  CK(cudaStreamSynchronize(s));
  std::lock_guard<std::mutex> g(a->reg_mu);
  const StringPool& sp = a->sp;
  auto strs_of = [&sp](const std::vector<uint32_t>& v) {
    std::vector<std::pair<const uint8_t*, uint32_t>> out;
    out.reserve(v.size());
    for (uint32_t cid : v) out.emplace_back(sp.ptr(cid), sp.len(cid));
    return out;
  };
  auto dict_ree = [&](const char* name, int d, uint64_t len) {
    uint32_t nr = c.n_runs[d];
    Node values = dict_node("values", true, nr, c.n_null[d], c.n_null[d] ? BufRef::dev(run_valid[d], (nr + 7) / 8) : BufRef::none(),
                            BufRef::dev(run_key[d], (uint64_t)nr * 4), utf8_node(a, "values", true, strs_of(ord[d]), nullptr, Ty::Binary));
    return ree_node(name, false, (int64_t)len, nr, BufRef::dev(run_end[d], (uint64_t)nr * 4), std::move(values));
  };
  auto zero_ree = [&](const char* name) {  // AppendN(0, numMappings) (arrow.go:231-238): one run over every location, or none
    std::vector<int32_t> re;
    if (L) re.push_back((int32_t)L);
    std::vector<uint64_t> zero{0};
    return ree_node(name, false, (int64_t)L, (int64_t)re.size(), host_ref(a, re), int_node("values", 64, false, true, 1, host_ref(a, zero)));
  };
  Node line; line.ty = Ty::Struct; line.name = "item"; line.nullable = true; line.length = (int64_t)NL;
  line.kids.push_back(int_node("line", 64, true, false, (int64_t)NL, BufRef::dev(o.line_no, NL * 8)));
  line.kids.push_back(int_node("column", 64, false, false, (int64_t)NL, BufRef::dev(o.column, NL * 8)));
  line.kids.push_back(dict_node("function_name", false, (int64_t)NL, 0, BufRef::none(), BufRef::dev(o.fn_key, NL * 4),
                                utf8_node(a, "values", true, strs_of(ord[4]), nullptr, Ty::Binary)));
  {
    std::vector<std::pair<const uint8_t*, uint32_t>> empty_name;
    if (NL) empty_name.emplace_back(sp.ptr(0), 0u);  // FunctionSystemName.AppendString("") for every line
    line.kids.push_back(dict_node("function_system_name", false, (int64_t)NL, 0, BufRef::none(), BufRef::zeros(NL * 4),
                                  utf8_node(a, "values", true, empty_name, nullptr, Ty::Binary)));
  }
  line.kids.push_back(dict_ree("function_filename", 3, NL));
  line.kids.push_back(int_node("function_start_line", 64, true, false, (int64_t)NL, BufRef::zeros(NL * 8)));
  Node lines; lines.ty = Ty::List; lines.name = "lines"; lines.nullable = false; lines.length = (int64_t)L; lines.null_count = (int64_t)(L - NL);
  lines.validity = BufRef::dev(hasline_w, (L + 7) / 8);
  lines.bufs = {BufRef::dev(o.line_off, (L + 1) * 4)};
  lines.kids.push_back(std::move(line));
  Node loc; loc.ty = Ty::Struct; loc.name = "item"; loc.nullable = true; loc.length = (int64_t)L;
  loc.kids.push_back(int_node("address", 64, false, false, (int64_t)L, BufRef::dev(o.address, L * 8)));
  loc.kids.push_back(dict_ree("frame_type", 0, L));
  loc.kids.push_back(zero_ree("mapping_start"));
  loc.kids.push_back(zero_ree("mapping_limit"));
  loc.kids.push_back(zero_ree("mapping_offset"));
  loc.kids.push_back(dict_ree("mapping_file", 1, L));
  loc.kids.push_back(dict_ree("mapping_build_id", 2, L));
  loc.kids.push_back(std::move(lines));
  Node locs; locs.ty = Ty::List; locs.name = "locations"; locs.nullable = false; locs.length = (int64_t)n; locs.null_count = c.st_null_lists;
  locs.validity = BufRef::dev(listv_w, (n + 7) / 8);
  locs.bufs = {BufRef::dev(loc_off, (n + 1) * 4)};
  locs.kids.push_back(std::move(loc));
  std::vector<Node> cols;
  {
    std::vector<int32_t> off(n + 1);
    for (uint64_t i = 0; i <= n; i++) off[i] = (int32_t)(16 * i);
    Node id; id.ty = Ty::Binary; id.name = "stacktrace_id"; id.nullable = false; id.length = (int64_t)n;
    id.bufs = {host_ref(a, off), BufRef::host(ids_host, n * 16)};
    cols.push_back(std::move(id));
  }
  {
    Node ic; ic.ty = Ty::Bool; ic.name = "is_complete"; ic.nullable = false; ic.length = (int64_t)n; ic.bufs = {BufRef::dev(complete_w, (n + 7) / 8)};
    cols.push_back(std::move(ic));
  }
  cols.push_back(std::move(locs));

  StreamPlan plan;
  plan.build(cols, {{"parca_write_schema_version", "v1"}}, (int64_t)n);
  if (a->cfg.ipc_compression == PA_IPC_LZ4_FRAME_GPU) {
    uint64_t len = 0;
    float d2h = 0, gpu = 0;
    if (int rc = lz4_gpu_stream(a, plan, s, &len, &d2h)) return rc;
    cudaEventElapsedTime(&gpu, a->tm[T_TOTAL].a, a->tm[T_TOTAL].b);
    res->ipc = a->out; res->ipc_len = len; res->n_rows = n; res->n_unique_stacks = n; res->n_locations = L; res->n_functions = c.n_dict[4];
    res->n_location_indices = NL; res->gpu_launches = tm.launches; res->gpu_ms = gpu; res->d2h_ms = d2h;
    res->host_ms = std::max(0.0, (now_ms() - t0) - gpu - d2h - a->tm[T_LZ4].ms);
    return PA_OK;
  }
  if (plan.total > a->out_cap) {
    CK(cudaStreamSynchronize(a->s_d2h));
    if (a->out) cudaFreeHost(a->out);
    a->out = nullptr;
    a->out_cap = 0;
    uint64_t want = plan.total + plan.total / 4 + 4096;
    if (cudaHostAlloc((void**)&a->out, want, cudaHostAllocDefault) != cudaSuccess) return a->fail(PA_ENOMEM, "pinned output allocation failed");
    a->out_cap = want;
  }
  const double t1 = now_ms();
  CK(cudaEventRecord(a->ev_d2h0, s));
  for (auto& p : plan.placements)
    if (p.src.kind == BufRef::DEVICE && p.src.len) CK(cudaMemcpyAsync(a->out + p.at, p.src.ptr, p.src.len, cudaMemcpyDeviceToHost, s));
  CK(cudaEventRecord(a->ev_d2h1, s));
  plan.write_host_parts(a->out);
  CK(cudaStreamSynchronize(s));
  const uint8_t* stream = a->out;
  uint64_t stream_len = plan.total;
  if (a->cfg.ipc_compression == PA_IPC_LZ4_FRAME) {
    std::string why;
    if (!ipc_compress_lz4(a->out, plan.total, a->comp_out, &why)) return a->fail(PA_EIO, why.c_str());
    stream = a->comp_out.data();
    stream_len = a->comp_out.size();
  }
  const double t2 = now_ms();
  float d2h = 0, gpu = 0;
  cudaEventElapsedTime(&d2h, a->ev_d2h0, a->ev_d2h1);
  cudaEventElapsedTime(&gpu, a->tm[T_TOTAL].a, a->tm[T_TOTAL].b);
  res->ipc = stream; res->ipc_len = stream_len; res->n_rows = n; res->n_unique_stacks = n; res->n_locations = L; res->n_functions = c.n_dict[4];
  res->n_location_indices = NL; res->gpu_launches = tm.launches; res->gpu_ms = gpu; res->d2h_ms = d2h; res->host_ms = (t2 - t0) - gpu - d2h;
  if (res->host_ms < 0) res->host_ms = 0;
  (void)t1;
  return PA_OK;
}

// ---------------------------------------------------------------------------------------------
// mode B building blocks (see include/parcaagg.h): export a processed shard, stage a merged batch from device memory
static const char kRegisteredUnsupported[] = "not supported with PA_CFG_REGISTERED_STACKS (rows name registered stacks, not frame ranges)";
static int stage_device(pa_agg* a, const pa_sample_hdr* hdr, uint64_t n_rows, const uint64_t* frames, uint64_t n_frames) {
  if (a->registered) return a->fail(PA_EINVAL, kRegisteredUnsupported);
  CK(cudaSetDevice(a->device));
  if (a->staged >= 0) return a->fail(PA_EINVAL, "the previously staged batch has not been collected");
  if (n_rows > a->cfg.max_samples || n_frames > a->cfg.max_frames) return a->fail(PA_ENOSPC, "device batch exceeds max_samples / max_frames");
  if ((n_rows && !hdr) || (n_frames && !frames)) return a->fail(PA_EINVAL, "null device buffer");
  if (a->idb != 8) return a->fail(PA_EINVAL, "device-staged batches carry uint64 frame ids: create the aggregator with frame_id_bytes = 8");
  CK(a->d_frames.ensure(std::max<uint64_t>(n_frames, 1) * 8));  // provided-hash aggregators do not own a frame buffer until now
  a->staged = a->active;  // no ring buffer is detached: ingest into the ring continues untouched
  a->src_frames = a->d_frames.as<unsigned long long>();
  a->N = n_rows;
  a->NF = n_frames;
  a->processed = false;
  a->chunk_rows.clear();
  a->chunk_frames_end.clear();
  CK(cudaEventRecord(a->ev_h2d0, a->s_copy));
  if (n_rows) CK(cudaMemcpyAsync(a->d_hdr.p, hdr, n_rows * 64, cudaMemcpyDeviceToDevice, a->s_copy));
  if (n_frames) CK(cudaMemcpyAsync(a->d_frames.p, frames, n_frames * 8, cudaMemcpyDeviceToDevice, a->s_copy));
  CK(cudaEventRecord(a->ev_h2d1, a->s_copy));
  CK(cudaStreamSynchronize(a->s_copy));
  return PA_OK;
}

static int stage_device_parts(pa_agg* a, const pa_device_part* parts, uint32_t n_parts, uint64_t n_total) {
  if (a->registered) return a->fail(PA_EINVAL, kRegisteredUnsupported);
  CK(cudaSetDevice(a->device));
  if (a->staged >= 0) return a->fail(PA_EINVAL, "the previously staged batch has not been collected");
  if (n_parts && !parts) return a->fail(PA_EINVAL, "null parts");
  uint64_t rows = 0, nfr = 0;
  for (uint32_t p = 0; p < n_parts; p++) {
    if ((parts[p].n_rows && (!parts[p].hdr || !parts[p].global_row)) || (parts[p].n_frames && !parts[p].frames)) return a->fail(PA_EINVAL, "null device buffer");
    rows += parts[p].n_rows;
    nfr += parts[p].n_frames;
  }
  if (rows != n_total) return a->fail(PA_EINVAL, "the parts do not add up to n_rows_total");
  if (a->idb != 8) return a->fail(PA_EINVAL, "device-staged batches carry uint64 frame ids: create the aggregator with frame_id_bytes = 8");
  if (n_total > a->cfg.max_samples || nfr > a->cfg.max_frames) return a->fail(PA_ENOSPC, "device batch exceeds max_samples / max_frames");
  CK(a->d_frames.ensure(std::max<uint64_t>(nfr, 1) * 8));
  CK(a->d_st1.ensure(256));
  uint32_t* bad = a->d_st1.as<uint32_t>();
  cudaStream_t s = a->s_copy;
  CK(cudaEventRecord(a->ev_h2d0, s));
  CK(cudaMemsetAsync(bad, 0, 4, s));
  uint64_t foff = 0;
  for (uint32_t p = 0; p < n_parts; p++) {
    if (parts[p].n_rows)
      k_scatter_rows<<<small_grid(a, parts[p].n_rows * 4), kThreads, 0, s>>>((const uint4*)parts[p].hdr, (const unsigned long long*)parts[p].global_row, parts[p].n_rows,
                                                                              n_total, a->d_hdr.as<uint4>(), bad);
    if (parts[p].n_frames) CK(cudaMemcpyAsync(a->d_frames.as<uint64_t>() + foff, parts[p].frames, parts[p].n_frames * 8, cudaMemcpyDeviceToDevice, s));
    foff += parts[p].n_frames;
  }
  uint32_t h_bad = 0;
  CK(cudaMemcpyAsync(&h_bad, bad, 4, cudaMemcpyDeviceToHost, s));
  CK(cudaEventRecord(a->ev_h2d1, s));
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  if (h_bad) return a->fail(PA_EINVAL, "global_row out of range");
  a->staged = a->active;
  a->src_frames = a->d_frames.as<unsigned long long>();
  a->N = n_total;
  a->NF = nfr;
  a->processed = false;
  a->chunk_rows.clear();
  a->chunk_frames_end.clear();
  return PA_OK;
}

static int shard_export(pa_agg* a, uint64_t frame_base, pa_sample_hdr* hdr_out, uint64_t* frames_out) {
  if (a->registered) return a->fail(PA_EINVAL, kRegisteredUnsupported);
  if (a->cfg.schema != PA_SCHEMA_V2) return a->fail(PA_EINVAL, "shard export needs a PA_SCHEMA_V2 aggregator (the v2 pipeline gathers the unique stacks)");
  if (a->staged < 0 || !a->processed) return a->fail(PA_EINVAL, "shard export needs a processed, not yet collected batch");
  if (!a->N) return PA_OK;
  if (!hdr_out || (a->h_ctr.n_indices64 && !frames_out)) return a->fail(PA_EINVAL, "null device buffer");
  CK(cudaSetDevice(a->device));
  cudaStream_t s = a->s_comp;
  k_shard_export_rows<<<a->G, kThreads, 0, s>>>((uint32_t)a->N, a->d_hdr.as<uint4>(), a->d_uuid.as<uint8_t>(), a->d_slot.as<uint32_t>(), a->d_table.as<StackSlot>(),
                                                frame_base, (uint4*)hdr_out);
  k_shard_export_frames<<<small_grid(a, a->h_ctr.n_indices64), kThreads, 0, s>>>(a->d_ctr.as<Counters>(), a->d_ustream.as<uint32_t>(), a->loc_order,
                                                                                   (unsigned long long*)frames_out);
  CK(cudaStreamSynchronize(s));
  CK(cudaGetLastError());
  return PA_OK;
}

// PA_CFG_RETIRE_STACKS: idle selection on the device (bitmap, popcount prefix, handles in slot order), then the host marks the
// retired stacks for freeing at the stage after their grace batch
static int retire_stacks(pa_agg* a, uint32_t idle, uint64_t* handles, uint64_t cap, uint64_t* n_retired) {
  if (!a->retire) return a->fail(PA_EINVAL, "pa_agg_retire_stacks needs an aggregator created with PA_CFG_RETIRE_STACKS");
  if (idle == 0) return a->fail(PA_EINVAL, "idle_batches must be at least 1");
  if (a->staged >= 0) return a->fail(PA_EINVAL, "collect the staged batch before retiring stacks");
  if (cap && !handles) return PA_EINVAL;
  if (n_retired) *n_retired = 0;
  // rs_stages and rs_dev_slots change only under flush_mu, which this thread holds; stacks registered since the last upload are
  // not on the device yet and are never idle (their last_use is the current stage count)
  const uint64_t ns = a->rs_dev_slots;
  if (a->rs_stages < idle || ns == 0 || cap == 0) return PA_OK;
  CK(cudaSetDevice(a->device));
  cudaStream_t s = a->s_comp;
  const uint32_t nw = (uint32_t)((ns + 31) / 32);
  const uint64_t nh = std::min<uint64_t>(cap, ns);
  CK(a->d_rs_tmp.ensure(nh * 8 + 2ull * nw * 4 + 64));
  unsigned long long* d_handles = a->d_rs_tmp.as<unsigned long long>();
  uint32_t* bits = (uint32_t*)(d_handles + nh);
  uint32_t* wprefix = bits + nw;
  uint32_t* total = wprefix + nw;
  const RegStack* recs = a->d_rs_recs.as<RegStack>();
  uint32_t* last = a->d_rs_last.as<uint32_t>();
  Timer t{};
  k_stack_idle_bits<<<small_grid(a, ns), kThreads, 0, s>>>(recs, last, (uint32_t)ns, (uint32_t)(a->rs_stages - idle), bits);
  launch_scan(a, WordsF{bits, wprefix, nw, total}, 1, t, small_grid(a, nw), s, a->d_partial);
  k_stack_idle_emit<<<small_grid(a, ns), kThreads, 0, s>>>(bits, wprefix, (uint32_t)ns, recs, nh, d_handles, last);
  uint32_t n_idle = 0;
  CK(cudaMemcpyAsync(&n_idle, total, 4, cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s));
  const uint64_t n = std::min<uint64_t>(n_idle, nh);
  if (n) CK(cudaMemcpy(handles, d_handles, n * 8, cudaMemcpyDeviceToHost));
  CK(cudaGetLastError());
  std::lock_guard<std::mutex> g(a->reg_mu);
  for (uint64_t i = 0; i < n; i++) {
    const uint32_t slot = (uint32_t)handles[i];
    a->rs_state[slot] = pa_agg::RS_RETIRING;
    a->rs_retiring.emplace_back(slot, a->rs_stages + 2);  // batch rs_stages + 1 is the grace batch
  }
  a->rs_retired += n;
  if (n_retired) *n_retired = n;
  return PA_OK;
}

extern "C" {

int pa_agg_retire_stacks(pa_agg* a, uint32_t idle_batches, uint64_t* handles, uint64_t cap, uint64_t* n_retired) {
  if (!a) return PA_EINVAL;
  if (a->group_retire) return a->fail(PA_EINVAL, "PA_CFG_GROUP_RETIRE: the merge group retires its stacks together, through pa_merge_retire_stacks");
  std::lock_guard<std::mutex> g(a->flush_mu);
  return retire_stacks(a, idle_batches, handles, cap, n_retired);
}

int pa_agg_shard_sizes(pa_agg* a, uint64_t* n_rows, uint64_t* n_frames) {
  if (!a || !n_rows || !n_frames) return PA_EINVAL;
  std::lock_guard<std::mutex> g(a->flush_mu);
  if (a->staged < 0 || !a->processed) return a->fail(PA_EINVAL, "shard sizes need a processed, not yet collected batch");
  *n_rows = a->N;
  *n_frames = a->N ? a->h_ctr.n_indices64 : 0;
  return PA_OK;
}
int pa_agg_shard_export(pa_agg* a, uint64_t frame_base, pa_sample_hdr* hdr_out, uint64_t* frames_out) {
  if (!a) return PA_EINVAL;
  std::lock_guard<std::mutex> g(a->flush_mu);
  return shard_export(a, frame_base, hdr_out, frames_out);
}
int pa_agg_stage_device_parts(pa_agg* a, const pa_device_part* parts, uint32_t n_parts, uint64_t n_rows_total) {
  if (!a) return PA_EINVAL;
  std::lock_guard<std::mutex> g(a->flush_mu);
  return stage_device_parts(a, parts, n_parts, n_rows_total);
}
int pa_agg_discard(pa_agg* a) {
  if (!a) return PA_EINVAL;
  std::lock_guard<std::mutex> g(a->flush_mu);
  CK(cudaSetDevice(a->device));
  CK(cudaStreamSynchronize(a->s_copy));
  CK(cudaStreamSynchronize(a->s_comp));
  release_staged(a);
  a->merged_part = false;
  return PA_OK;
}
int pa_agg_stage_device(pa_agg* a, const pa_sample_hdr* hdr, uint64_t n_rows, const uint64_t* frames, uint64_t n_frames) {
  if (!a) return PA_EINVAL;
  std::lock_guard<std::mutex> g(a->flush_mu);
  return stage_device(a, hdr, n_rows, frames, n_frames);
}

int pa_agg_stacktraces(pa_agg* a, const uint8_t* ids, uint64_t n_ids, pa_agg_result* out) {
  if (!a || !out) return PA_EINVAL;
  std::lock_guard<std::mutex> g(a->flush_mu);
  return stacktraces(a, ids, n_ids, out);
}
int pa_agg_last_stack_ids(pa_agg* a, uint8_t* out, uint64_t n) {
  if (!a || (n && !out)) return PA_EINVAL;
  std::lock_guard<std::mutex> g(a->flush_mu);
  if (a->cfg.schema != PA_SCHEMA_V1) return a->fail(PA_EINVAL, "pa_agg_last_stack_ids needs a PA_SCHEMA_V1 aggregator");
  if (n > a->last_unique) return a->fail(PA_EINVAL, "more ids requested than the last batch had unique stacks");
  CK(cudaSetDevice(a->device));
  if (n) CK(cudaMemcpy(out, a->d_v1_ids.p, n * 16, cudaMemcpyDeviceToHost));
  return PA_OK;
}

int pa_agg_stage(pa_agg* a) {
  if (!a) return PA_EINVAL;
  std::lock_guard<std::mutex> g(a->flush_mu);
  int rc = stage_async(a);
  if (rc) return rc;
  CK(cudaStreamSynchronize(a->s_copy));
  return PA_OK;
}
int pa_agg_process(pa_agg* a) {
  if (!a) return PA_EINVAL;
  std::lock_guard<std::mutex> g(a->flush_mu);
  return process(a);
}
int pa_agg_collect(pa_agg* a, pa_agg_result* out) {
  if (!a || !out) return PA_EINVAL;
  std::lock_guard<std::mutex> g(a->flush_mu);
  return collect(a, out);
}
int pa_agg_flush(pa_agg* a, pa_agg_result* out) {
  if (!a || !out) return PA_EINVAL;
  std::lock_guard<std::mutex> g(a->flush_mu);
  int rc = stage_async(a);  // copies keep running while process() consumes the chunks already resident
  if (rc) return rc;
  rc = process(a);
  if (rc) { cudaStreamSynchronize(a->s_copy); release_staged(a); return rc; }  // a failed flush drops the interval's data (:1218-1220)
  rc = collect(a, out);
  if (rc) release_staged(a);
  return rc;
}
void pa_agg_release(pa_agg* a, pa_agg_result* res) {
  if (!a || !res) return;
  std::lock_guard<std::mutex> g(a->flush_mu);
  a->hostbufs.clear();
  memset(res, 0, sizeof *res);
}
int pa_agg_last_kernel_ms(const pa_agg* a, const char* name, double* ms, uint32_t* launches) {
  if (!a || !name) return PA_EINVAL;
  for (int t = 0; t < T_COUNT; t++)
    if (!strcmp(name, kTimerNames[t])) {
      if (ms) *ms = a->tm[t].ms;
      if (launches) *launches = a->tm[t].launches;
      return PA_OK;
    }
  // the label column plan (ms is 0): labelset-derived columns planned for the last pass, and passes redone since creation
  // because the prediction missed a name the batch's rows used
  if (!strcmp(name, "label_columns") || !strcmp(name, "label_replans")) {
    if (ms) *ms = 0;
    if (launches) *launches = !strcmp(name, "label_columns") ? a->n_lscols : (uint32_t)std::min<uint64_t>(a->label_replans, 0xFFFFFFFFu);
    return PA_OK;
  }
  // PA_IPC_LZ4_FRAME_GPU merge groups (ms is 0): bytes of this member's parts that went to the owners of blocks crossing a part
  // border in the last pa_merge_plan
  if (!strcmp(name, "lz4_heads")) {
    if (ms) *ms = 0;
    if (launches) *launches = (uint32_t)std::min<uint64_t>(a->lz4_head_bytes, 0xFFFFFFFFu);
    return PA_OK;
  }
  // counters of the v1 stack store since creation (ms is 0): table compactions / eviction rounds
  if (!strcmp(name, "store_compactions") || !strcmp(name, "store_evictions")) {
    if (ms) *ms = 0;
    if (launches) *launches = (uint32_t)(name[6] == 'c' ? a->store_compactions : a->store_evictions);
    return PA_OK;
  }
  // PA_SCHEMA_V1 merge groups (ms is 0): frame ids (4 bytes each) this member sent to the other copies of the store in the last
  // store exchange of pa_merge_process
  if (!strcmp(name, "store_frames")) {
    if (ms) *ms = 0;
    if (launches) *launches = (uint32_t)std::min<uint64_t>(a->store_frames_sent, 0xFFFFFFFFu);
    return PA_OK;
  }
  // PA_CFG_RETIRE_STACKS (ms is 0): the stack registry's counters
  {
    static const char* kRegistryCounters[] = {"stacks_live", "stacks_free", "stack_frames_live", "stack_frames_dead", "stack_compactions", "stacks_retired"};
    for (int k = 0; k < 6; k++)
      if (!strcmp(name, kRegistryCounters[k])) {
        if (!a->retire) return PA_EINVAL;
        std::lock_guard<std::mutex> g(const_cast<pa_agg*>(a)->reg_mu);
        const uint64_t v[6] = {a->rs_live, a->rs_state.size() - a->rs_live, a->rs_frames_live, a->rs_frames_dead, a->rs_compactions, a->rs_retired};
        if (ms) *ms = 0;
        if (launches) *launches = (uint32_t)std::min<uint64_t>(v[k], 0xFFFFFFFFu);
        return PA_OK;
      }
  }
  if (!strcmp(name, "stack_compact")) {  // the last arena compaction: device time and launches
    if (!a->retire) return PA_EINVAL;
    if (ms) *ms = a->rs_tm.ms;
    if (launches) *launches = a->rs_tm.launches;
    return PA_OK;
  }
  // PA_SCHEMA_V1 merge groups of PA_CFG_GROUP_STACKS members (ms is 0): stack references (8-byte handles) this member sent
  // instead of frame ids in the last store exchange
  if (!strcmp(name, "store_refs")) {
    if (ms) *ms = 0;
    if (launches) *launches = (uint32_t)std::min<uint64_t>(a->store_refs_sent, 0xFFFFFFFFu);
    return PA_OK;
  }
  return PA_EINVAL;
}
int pa_agg_debug_stack_ids(pa_agg* a, uint8_t* out, uint64_t n_rows) {
  if (!a || !out || n_rows > a->N) return PA_EINVAL;
  CK(cudaSetDevice(a->device));
  CK(cudaMemcpy(out, a->d_uuid.p, n_rows * 16, cudaMemcpyDeviceToHost));
  return PA_OK;
}
int pa_agg_debug_stack_counts(pa_agg* a, uint32_t* out, uint64_t n) {
  if (!a || !out || n > a->h_ctr.n_unique || !a->N) return PA_EINVAL;
  std::lock_guard<std::mutex> g(a->flush_mu);
  CK(cudaSetDevice(a->device));
  // computed on demand from the staged batch (rows -> table slot -> first-occurrence ordinal)
  CK(cudaMemsetAsync(a->d_uniq_count.p, 0, (size_t)a->h_ctr.n_unique * 4, a->s_comp));
  k_count_stacks<<<a->G, kThreads, 0, a->s_comp>>>((uint32_t)a->N, a->d_slot.as<uint32_t>(), a->d_table.as<StackSlot>(), a->d_uniq_count.as<uint32_t>());
  CK(cudaMemcpyAsync(out, a->d_uniq_count.p, n * 4, cudaMemcpyDeviceToHost, a->s_comp));
  CK(cudaStreamSynchronize(a->s_comp));
  return PA_OK;
}

int pa_agg_debug_pair_counts(pa_agg* a, uint32_t* labelset_ids, uint32_t* stack_ordinals, uint32_t* counts, uint64_t cap, uint64_t* n_pairs) {
  if (!a || !n_pairs || (cap && (!labelset_ids || !stack_ordinals || !counts))) return PA_EINVAL;
  std::lock_guard<std::mutex> g(a->flush_mu);
  if (!a->processed) return a->fail(PA_EINVAL, "pair counts need a processed batch");
  *n_pairs = 0;
  const uint64_t N = a->N;
  if (!N) return PA_OK;
  CK(cudaSetDevice(a->device));
  cudaStream_t s = a->s_comp;
  // scratch of its own (the flush arena is still owned by the batch): pair table, first-row bitmap + prefix, outputs
  const uint64_t slots = pow2_at_least(2 * N), words = N / 32 + 2, ocap = std::min<uint64_t>(cap, N);
  DBuf scratch;
  const size_t b_tab = slots * sizeof(PairSlot), b_words = ((words * 4 + 255) & ~(size_t)255), b_out = ((std::max<uint64_t>(ocap, 1) * 4 + 255) & ~(size_t)255);
  CK(scratch.ensure(b_tab + 2 * b_words + 3 * b_out + 256));
  uint8_t* base = scratch.as<uint8_t>();
  PairSlot* pt = (PairSlot*)base;
  uint32_t* bits = (uint32_t*)(base + b_tab);
  uint32_t* wp = (uint32_t*)(base + b_tab + b_words);
  uint32_t* o_ls = (uint32_t*)(base + b_tab + 2 * b_words);
  uint32_t* o_st = (uint32_t*)(base + b_tab + 2 * b_words + b_out);
  uint32_t* o_ct = (uint32_t*)(base + b_tab + 2 * b_words + 2 * b_out);
  uint32_t* flags = (uint32_t*)(base + b_tab + 2 * b_words + 3 * b_out);  // [0] overflow, [1] distinct pairs
  int rc = PA_OK;
  auto run = [&]() -> int {
    CK(cudaMemsetAsync(base, 0, b_tab + b_words, s));
    CK(cudaMemsetAsync(flags, 0, 8, s));
    k_pair_count<<<a->G, kThreads, 0, s>>>((uint32_t)N, a->d_ls.as<uint32_t>(), a->d_slot.as<uint32_t>(), a->d_table.as<StackSlot>(), pt, (uint32_t)(slots - 1), flags);
    k_pair_bits<<<small_grid(a, slots), kThreads, 0, s>>>(pt, (uint32_t)slots, bits);
    Timer t{};
    launch_scan(a, WordsF{bits, wp, (uint32_t)((N + 31) / 32), flags + 1}, 1, t, small_grid(a, N / 32 + 1), s, a->d_partial);
    k_pair_emit<<<small_grid(a, slots), kThreads, 0, s>>>(pt, (uint32_t)slots, bits, wp, (uint32_t)ocap, o_ls, o_st, o_ct);
    uint32_t h[2] = {0, 0};
    CK(cudaMemcpyAsync(h, flags, 8, cudaMemcpyDeviceToHost, s));
    CK(cudaStreamSynchronize(s));
    CK(cudaGetLastError());
    if (h[0]) return a->fail(PA_ENOMEM, "pair table overflow");
    *n_pairs = h[1];
    const uint64_t m = std::min<uint64_t>(h[1], ocap);
    if (m) {
      CK(cudaMemcpy(labelset_ids, o_ls, m * 4, cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(stack_ordinals, o_st, m * 4, cudaMemcpyDeviceToHost));
      CK(cudaMemcpy(counts, o_ct, m * 4, cudaMemcpyDeviceToHost));
    }
    return PA_OK;
  };
  rc = run();
  scratch.release();
  return rc;
}

int pa_ipc_compress_lz4(const uint8_t* ipc, uint64_t len, uint8_t** out, uint64_t* out_len) {
  if (!ipc || !out || !out_len) return PA_EINVAL;
  std::vector<uint8_t> v;
  std::string why;
  if (!ipc_compress_lz4(ipc, len, v, &why)) return why.find("liblz4") != std::string::npos || why.find("LZ4F") != std::string::npos ? PA_EIO : PA_EINVAL;
  uint8_t* p = (uint8_t*)malloc(std::max<size_t>(v.size(), 1));
  if (!p) return PA_ENOMEM;
  memcpy(p, v.data(), v.size());
  *out = p;
  *out_len = v.size();
  return PA_OK;
}
void pa_ipc_free(uint8_t* p) { free(p); }

// ---- host helpers ------------------------------------------------------------------------------
static bool valid_utf8(const uint8_t* s, uint64_t n) {  // unicode/utf8.ValidString
  uint64_t i = 0;
  while (i < n) {
    uint8_t b = s[i];
    if (b < 0x80) { i++; continue; }
    int extra; uint32_t cp, lo;
    if (b >= 0xC2 && b <= 0xDF) { extra = 1; cp = b & 0x1Fu; lo = 0x80; }
    else if (b >= 0xE0 && b <= 0xEF) { extra = 2; cp = b & 0x0Fu; lo = 0x800; }
    else if (b >= 0xF0 && b <= 0xF4) { extra = 3; cp = b & 0x07u; lo = 0x10000; }
    else return false;
    if (i + (uint64_t)extra >= n) return false;
    for (int k = 1; k <= extra; k++) {
      uint8_t cb = s[i + k];
      if ((cb & 0xC0) != 0x80) return false;
      cp = (cp << 6) | (cb & 0x3Fu);
    }
    if (cp < lo || cp > 0x10FFFF || (cp >= 0xD800 && cp <= 0xDFFF)) return false;
    i += (uint64_t)extra + 1;
  }
  return true;
}
// maybeFixTruncation, reporter/parca_reporter.go:190-216
int64_t pa_fix_truncation(const uint8_t* s, uint64_t len, uint64_t max_len) {
  if (valid_utf8(s, len)) return (int64_t)len;
  if (len != max_len) return -1;
  for (uint64_t back = 1; back <= 2 && back <= len; back++) {
    uint64_t idx = max_len - back;
    if ((s[idx] & 0xC0) != 0x80) return valid_utf8(s, idx) ? (int64_t)idx : -1;
  }
  return -1;
}
uint64_t pa_xxh64(const void* data, uint64_t len, uint64_t seed) {
  const uint8_t* p = (const uint8_t*)data;
  const uint8_t* const end = p + len;
  auto rd64 = [](const uint8_t* q) { uint64_t v; memcpy(&v, q, 8); return v; };
  auto rot = [](uint64_t x, int r) { return (x << r) | (x >> (64 - r)); };
  const uint64_t P1 = 11400714785074694791ULL, P2 = 14029467366897019727ULL, P3 = 1609587929392839161ULL, P4 = 9650029242287828579ULL, P5 = 2870177450012600261ULL;
  uint64_t h;
  if (len >= 32) {
    uint64_t v[4] = {seed + P1 + P2, seed + P2, seed, seed - P1};
    for (; p + 32 <= end; p += 32)
      for (int k = 0; k < 4; k++) v[k] = rot(v[k] + rd64(p + 8 * k) * P2, 31) * P1;
    h = rot(v[0], 1) + rot(v[1], 7) + rot(v[2], 12) + rot(v[3], 18);
    for (int k = 0; k < 4; k++) h = (h ^ (rot(v[k] * P2, 31) * P1)) * P1 + P4;
  } else {
    h = seed + P5;
  }
  h += len;
  for (; p + 8 <= end; p += 8) h = rot(h ^ (rot(rd64(p) * P2, 31) * P1), 27) * P1 + P4;
  if (p + 4 <= end) { uint32_t w; memcpy(&w, p, 4); h = rot(h ^ (w * P1), 23) * P2 + P3; p += 4; }
  for (; p < end; p++) h = rot(h ^ (*p * P5), 11) * P1;
  h ^= h >> 33; h *= P2; h ^= h >> 29; h *= P3; h ^= h >> 32;
  return h;
}

}  // extern "C"

#include "merge_impl.hpp"
