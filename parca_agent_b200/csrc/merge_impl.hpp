// merge_impl.hpp — multi-GPU mode B inside the library: ONE record batch out of several pid-hash shards, with an
// O(unique keys) dictionary exchange (SURVEY section 8e). Textually included at the end of agg.cu (one translation unit:
// the kernels live in a header).
//
// Definition of the merged batch: the reference's record (reporter/parca_reporter.go:1742-1790) for the sample stream
// [shard 0's rows, shard 1's rows, ...] — every GPU owns a ring (north_star: samples are sharded by pid hash), and the
// merged stream is the rings in rank order. Rows, and everything that is per row or per run, stay on the GPU that
// ingested them and go to the host over that GPU's own PCIe link; only dictionary keys cross NVLink:
//   all-to-all   (id128, global first row, depth) of each shard's unique stacks to the id's owner     U_local x 24 B
//   all-gather   the owners' deduplicated lists (every shard then ranks them identically)             U x 24 B
//   all-reduce   min over the frame-indexed first-position table and the direct label tables          (P + L + 64k + S) x 4 B
//   all-gather   thread-id lists, per-column run edges (count, first / last key)                      T x 8 B + cols x 40 B
//   v1 groups (replicated known-stacks store): all-reduce(min) of each merged stack's inverted last row  U x 4 B
//                and all-gather-v of the frames of the stacks the store lacks                          4 B per frame (0 in steady state)
//                (PA_CFG_GROUP_STACKS members: of one arena offset per such stack instead)             8 B per stack
//                (PA_CFG_GROUP_RETIRE members: of the stack's handle instead)                          8 B per stack
//   PA_CFG_GROUP_RETIRE groups, in pa_merge_retire_stacks: all-gather of the call's arguments and state   32 B
//                and all-reduce(min) of the inverted last_use of every registry slot                   4 B per slot
// Invariants reproduced: first-occurrence order of every dictionary (arrow_v2.go:191, :302; parca_reporter.go:425),
// run merging across shard borders (arrow.go:97-131).
//
// Transport: NCCL (dlopen'ed, so single-GPU users need no NCCL) with one communicator per member, members in one or in
// several processes; or, when every member lives on ONE device of one process (tests, and hosts that feed one GPU from
// several rings), plain device copies on a shared stream.
#pragma once
#include <dlfcn.h>
#include <fcntl.h>
#include <nccl.h>
#include <sched.h>
#include <sys/mman.h>
#include <sys/stat.h>

#include <atomic>

namespace pa {

struct NcclApi {
  void* h = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*AllReduce)(const void*, void*, size_t, ncclDataType_t, ncclRedOp_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Send)(const void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char* (*GetErrorString)(ncclResult_t) = nullptr;
  std::string why;
};
static NcclApi* nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    const char* env = getenv("PA_NCCL_LIB");
    const char* names[] = {env, "libnccl.so.2", "libnccl.so", "/usr/lib/x86_64-linux-gnu/libnccl.so.2"};
    // a copy that is already mapped (e.g. the one torch ships) wins: two NCCL instances in one process do not mix
    api.h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);
    for (const char* n : names) { if (api.h) break; if (n && *n) api.h = dlopen(n, RTLD_NOW | RTLD_GLOBAL); }
    if (!api.h) { api.why = "libnccl.so.2 not found (set PA_NCCL_LIB)"; return; }
    auto sym = [&](const char* n) { void* p = dlsym(api.h, n); if (!p && api.why.empty()) api.why = std::string("missing NCCL symbol ") + n; return p; };
    api.GetUniqueId = (decltype(api.GetUniqueId))sym("ncclGetUniqueId");
    api.CommInitRank = (decltype(api.CommInitRank))sym("ncclCommInitRank");
    api.CommDestroy = (decltype(api.CommDestroy))sym("ncclCommDestroy");
    api.AllGather = (decltype(api.AllGather))sym("ncclAllGather");
    api.AllReduce = (decltype(api.AllReduce))sym("ncclAllReduce");
    api.Broadcast = (decltype(api.Broadcast))sym("ncclBroadcast");
    api.Send = (decltype(api.Send))sym("ncclSend");
    api.Recv = (decltype(api.Recv))sym("ncclRecv");
    api.GroupStart = (decltype(api.GroupStart))sym("ncclGroupStart");
    api.GroupEnd = (decltype(api.GroupEnd))sym("ncclGroupEnd");
    api.GetErrorString = (decltype(api.GetErrorString))sym("ncclGetErrorString");
    if (!api.why.empty()) api.h = nullptr;
  });
  return api.h ? &api : nullptr;
}

// per-member device buffers of the merge (grown on demand, kept across intervals)
struct MergeBufs {
  DBuf ctl;        // MergeCtl + owner-table control words + merged-table control words + per-owner counters / cursors
  DBuf send, recv, otab, oclaimed, ouniq, glist, gtab, gclaimed, g_uniq_row, g_uniq_slot, g_uniq_size;
  DBuf tid_list, tid_all, edges, edges_all, mcols, mcols_all, gather_scratch, kind_all, vwords, vwords_all;
  // v1 groups only: stacktrace_id offsets, and the replicated store's update (last rows, frames exchange) and requests
  DBuf v1_off, v1_last, v1_need, v1_foff, v1_bounds, v1_send, v1_frames, v1_ids_req;
  void release() {
    DBuf* all[] = {&ctl, &send, &recv, &otab, &oclaimed, &ouniq, &glist, &gtab, &gclaimed, &g_uniq_row, &g_uniq_slot, &g_uniq_size,
                   &tid_list, &tid_all, &edges, &edges_all, &mcols, &mcols_all, &gather_scratch, &kind_all, &vwords, &vwords_all,
                   &v1_off, &v1_last, &v1_need, &v1_foff, &v1_bounds, &v1_send, &v1_frames, &v1_ids_req};
    for (DBuf* b : all) b->release();
  }
};
// layout of MergeBufs::ctl (uint32 words)
enum { CTL_MERGE = 0 /* MergeCtl: 8 words */, CTL_OWNER = 8 /* n_claimed, zero_claimed, err */, CTL_MERGED = 12, CTL_CNT = 16 /* [kMaxWorld] */,
       CTL_CURSOR = CTL_CNT + kMaxWorld + 2 /* cnt is followed by two scalars in the size exchange */, CTL_WORDS = CTL_CURSOR + kMaxWorld };

}  // namespace pa

namespace pa {
// Shared-memory transport (pa_merge_create_shm): ONE POSIX shm segment that every process of the group maps and page-locks.
// A collective is: every rank DMAs its block from its GPU into its own mailbox (over its own PCIe link), a process-shared
// barrier, every rank DMAs the blocks it needs out of the others' mailboxes into its GPU, another barrier. No NCCL, no
// sockets; payloads larger than a mailbox go in rounds. Header first, then `world` mailboxes of mailbox_bytes each.
struct ShmHeader {
  std::atomic<uint32_t> ready;     // rank 0 has initialised the segment
  uint32_t world;
  uint64_t mailbox_bytes;
  std::atomic<uint32_t> arrive, gen;  // barrier: arrival counter + generation
  std::atomic<uint32_t> failed;    // a rank gave up (timeout / error): everybody leaves the barrier with an error
  uint64_t desc[kMaxWorld][2 * kMaxWorld + 2];  // per rank: scounts | sdispls | total of the all-to-all in flight
};
constexpr size_t kShmHeaderBytes = (sizeof(ShmHeader) + 4095) & ~(size_t)4095;
}  // namespace pa

struct pa_merge {
  std::vector<pa_agg*> members;   // the shards this process drives
  std::vector<uint32_t> ranks;    // their ranks in the group
  uint32_t world = 0;
  bool use_nccl = false;        // one stream per member, collectives order them (NCCL, or the caller's host transport)
  std::vector<ncclComm_t> comms;
  const pa_merge_host_transport* host = nullptr;  // non-null: collectives go through the caller's callbacks on host buffers
  pa_merge_host_transport host_copy{};
  uint8_t *h_xs = nullptr, *h_xr = nullptr;       // pinned staging of the host transport
  size_t h_xs_cap = 0, h_xr_cap = 0;
  // shared-memory transport
  uint8_t* shm = nullptr;
  size_t shm_len = 0;
  std::string shm_name;
  bool shm_owner = false, shm_registered = false;
  DBuf shm_scratch;                               // device scratch of the all-reduce
  std::vector<MergeBufs> mb;
  std::vector<cudaStream_t> saved_streams;
  std::string err;
  uint8_t* h_pin = nullptr;       // pinned staging for the small host exchanges
  size_t h_pin_cap = 0;
  // ---- the batch last processed
  bool processed = false;
  uint64_t NT = 0, NFT = 0;
  std::vector<uint64_t> n_rows, row_base, nf;   // per rank
  std::vector<MergeCol> cols_all;               // [world][ncols]
  std::vector<MergeCtl> mctl;                   // per local member
  uint32_t ncols = 0;
  uint32_t retry_err = 0;                       // why merge_process_once asked for a redo: ERR_TABLE_FULL and / or ERR_LABEL_PLAN
  double ms_total = 0, ms_exchange_wait = 0;
  uint64_t nvlink_bytes = 0;                    // payload this process's members sent to other ranks during the last process()
  // ---- the stream last planned
  bool planned = false;
  std::vector<Node> nodes;
  StreamPlan plan;
  std::vector<std::vector<uint32_t>> kind_keys;
  std::vector<uint32_t> vwords_all;             // [world][ncols][2] first / last validity word of every shard's part
  uint8_t* out = nullptr;                       // library-owned output (local groups)
  uint64_t out_cap = 0;
  void* registered = nullptr;                   // caller's shared output buffer, page-locked by us
  uint64_t registered_len = 0;
  // ---- PA_IPC_LZ4_FRAME_GPU groups (every member in that mode): LZ4_FRAME bodies on the whole buffers' 64 KiB block grid
  bool lz4 = false;
  // ---- PA_CFG_GROUP_STACKS groups (every member in that mode): rows name stacks of identical registries, no ring frames
  bool group_stacks = false;
  bool group_retire = false;  // PA_CFG_GROUP_RETIRE groups (every member in that mode): stacks are retired by the group
  struct Lz4Share {                             // one local member's blocks, from pa_merge_plan to pa_merge_collect
    Lz4Table t;
    Lz4Dev d;
    std::vector<uint64_t> contrib, prefix;      // per buffer: bytes of my blocks (4 + size each); of lower ranks' blocks in front
    std::vector<const uint8_t*> part;           // per buffer: device source of my part of a sliced buffer (raw fallback)
    uint64_t send = 0, recv = 0;                // my heads, everybody's heads: offsets in the staging area
  };
  std::vector<Lz4Share> lzs;
  std::vector<uint32_t> lz_msg;                 // per buffer (messages 1.., stream order): its message
  std::vector<size_t> lz_place;                 // per buffer: its placement
  std::vector<std::vector<std::pair<uint64_t, uint64_t>>> lz_parts;  // per buffer: [world] (offset, bytes) of each part; empty = root only
  std::vector<uint64_t> lz_frame;               // per buffer: whole frame bytes
  Lz4Layout lz;

  int fail(int code, const std::string& what) { err = what; return code; }
};

namespace pa {

#define MCK(expr)                                                                              \
  do {                                                                                         \
    cudaError_t e_ = (expr);                                                                   \
    if (e_ != cudaSuccess) return g->fail(PA_EIO, std::string(#expr) + ": " + cudaGetErrorString(e_)); \
  } while (0)
#define NCK(expr)                                                                              \
  do {                                                                                         \
    ncclResult_t r_ = (expr);                                                                  \
    if (r_ != ncclSuccess) return g->fail(PA_EIO, std::string(#expr) + ": " + nccl_api()->GetErrorString(r_)); \
  } while (0)

// A group builds LZ4_FRAME records when every member was created with PA_IPC_LZ4_FRAME_GPU, plain ones when none was; a group
// that mixes the two is refused (at creation in one process, in pa_merge_process across processes).
static bool lz4_gpu_member(const pa_agg* m) { return m->cfg.ipc_compression == PA_IPC_LZ4_FRAME_GPU; }
static const char kLz4Mixed[] = "a merge group builds LZ4_FRAME records only when every member uses PA_IPC_LZ4_FRAME_GPU, and plain ones when none does: "
                                "this group mixes PA_IPC_LZ4_FRAME_GPU members with other members";
// Registered stacks join a group only with group-wide ids (PA_CFG_GROUP_STACKS), and only groups where every member has them.
static bool group_stacks_member(const pa_agg* m) { return m->group_stacks; }
static const char kStacksMixed[] = "a merge group of PA_CFG_GROUP_STACKS members takes no other members: this group mixes PA_CFG_GROUP_STACKS members "
                                   "with ring members or with plain PA_CFG_REGISTERED_STACKS members";
static const char kStacksMismatch[] = "the members of a PA_CFG_GROUP_STACKS merge group must register identical stacks in the same order: "
                                      "their number of stacks, frame arena length or stack digest differ";
// PA_CFG_GROUP_RETIRE members retire together: a group of them takes no other members, and they stay in lockstep
static const char kRetireMixed[] = "a merge group of PA_CFG_GROUP_RETIRE members takes no other members: this group mixes PA_CFG_GROUP_RETIRE members "
                                   "with members that do not retire stacks as a group";
static const char kRetireMismatch[] = "the members of a PA_CFG_GROUP_RETIRE merge group must register identical stacks in the same order, and stage "
                                      "and retire only as a group: their slot count, live stack frames, stage count or registry digest differ "
                                      "(a member staged or flushed on its own has left the group)";
// Every member of a group uses the same schema; v1 members also need the same store size, since each holds a full copy of the
// group's store (refused like a mixed LZ4 mode).
static const char kSchemaMixed[] = "a merge group builds one record schema: this group mixes PA_SCHEMA_V1 and PA_SCHEMA_V2 members";
static const char kStoreMismatch[] = "the members of a PA_SCHEMA_V1 merge group each hold a copy of the group's known-stacks store: "
                                     "their stack_cache_entries / stack_cache_frames must be equal (left at 0, both follow max_samples: "
                                     "members with different rings then need explicit, equal sizes)";
static cudaStream_t mstream(pa_merge* g, size_t i) { return g->members[i]->s_comp; }
// An in-process group on one device runs every member on ONE stream while a merge call is active, so that every copy between
// members is stream-ordered (NCCL groups keep one stream per member: the collectives order them).
struct StreamShare {
  pa_merge* g;
  explicit StreamShare(pa_merge* g_) : g(g_) {
    g->saved_streams.clear();
    if (g->use_nccl) return;
    for (pa_agg* a : g->members) { cudaStreamSynchronize(a->s_comp); g->saved_streams.push_back(a->s_comp); }
    for (pa_agg* a : g->members) a->s_comp = g->saved_streams[0];
  }
  ~StreamShare() {
    if (g->use_nccl) return;
    for (size_t i = 0; i < g->members.size(); i++) g->members[i]->s_comp = g->saved_streams[i];
  }
};
static int msync(pa_merge* g) {
  for (size_t i = 0; i < g->members.size(); i++) { MCK(cudaSetDevice(g->members[i]->device)); MCK(cudaStreamSynchronize(mstream(g, i))); }
  return PA_OK;
}
static int pin_room(pa_merge* g, size_t bytes) {
  if (bytes <= g->h_pin_cap) return PA_OK;
  if (g->h_pin) cudaFreeHost(g->h_pin);
  g->h_pin = nullptr; g->h_pin_cap = 0;
  MCK(cudaHostAlloc((void**)&g->h_pin, bytes * 2, cudaHostAllocDefault));
  g->h_pin_cap = bytes * 2;
  return PA_OK;
}

// ---- shared-memory transport ---------------------------------------------------------------------------------------------
static ShmHeader* shm_hdr(pa_merge* g) { return reinterpret_cast<ShmHeader*>(g->shm); }
static uint8_t* shm_box(pa_merge* g, uint32_t r) { return g->shm + kShmHeaderBytes + (size_t)r * shm_hdr(g)->mailbox_bytes; }
static int shm_barrier(pa_merge* g) {
  ShmHeader* h = shm_hdr(g);
  const uint32_t gen = h->gen.load(std::memory_order_acquire);
  if (h->arrive.fetch_add(1, std::memory_order_acq_rel) + 1 == h->world) {
    h->arrive.store(0, std::memory_order_relaxed);
    h->gen.fetch_add(1, std::memory_order_release);
    return PA_OK;
  }
  const double t0 = now_ms();
  uint32_t spins = 0;
  while (h->gen.load(std::memory_order_acquire) == gen) {
    if (h->failed.load(std::memory_order_relaxed)) return g->fail(PA_EIO, "shared-memory transport: another rank failed");
    if ((++spins & 0x3FF) == 0) {
      sched_yield();
      if (now_ms() - t0 > 120000.0) { h->failed.store(1); return g->fail(PA_EIO, "shared-memory transport: barrier timed out (a rank of the group is gone)"); }
    }
  }
  return PA_OK;
}
#define SBAR() do { int rcb_ = shm_barrier(g); if (rcb_) return rcb_; } while (0)
// rank r's block `src` (bytes[r] bytes) lands at dst + displ[r] on every rank
static int shm_allgatherv(pa_merge* g, const void* src, void* dst, const std::vector<uint64_t>& count, const std::vector<uint64_t>& displ) {
  const uint32_t W = g->world, me = g->ranks[0];
  const uint64_t M = shm_hdr(g)->mailbox_bytes;
  cudaStream_t s = mstream(g, 0);
  uint64_t maxc = 0;
  for (uint32_t r = 0; r < W; r++) maxc = std::max(maxc, count[r]);
  for (uint64_t off = 0; off < maxc; off += M) {
    const uint64_t mine = count[me] > off ? std::min<uint64_t>(M, count[me] - off) : 0;
    if (mine) MCK(cudaMemcpyAsync(shm_box(g, me), (const uint8_t*)src + off, mine, cudaMemcpyDeviceToHost, s));
    MCK(cudaStreamSynchronize(s));
    SBAR();
    for (uint32_t r = 0; r < W; r++) {
      const uint64_t n = count[r] > off ? std::min<uint64_t>(M, count[r] - off) : 0;
      if (n) MCK(cudaMemcpyAsync((uint8_t*)dst + displ[r] + off, shm_box(g, r), n, cudaMemcpyHostToDevice, s));
    }
    MCK(cudaStreamSynchronize(s));
    SBAR();  // nobody overwrites its mailbox before everybody has read it
  }
  g->nvlink_bytes += count[me] * (W - 1);
  return PA_OK;
}
static int shm_alltoallv(pa_merge* g, const void* send, const std::vector<uint64_t>& sc, const std::vector<uint64_t>& sd, void* recv, const std::vector<uint64_t>& rd) {
  const uint32_t W = g->world, me = g->ranks[0];
  ShmHeader* h = shm_hdr(g);
  const uint64_t M = h->mailbox_bytes;
  cudaStream_t s = mstream(g, 0);
  uint64_t tot = 0;
  for (uint32_t r = 0; r < W; r++) { h->desc[me][r] = sc[r]; h->desc[me][W + r] = sd[r]; tot = std::max(tot, sd[r] + sc[r]); }
  h->desc[me][2 * W] = tot;
  SBAR();
  uint64_t maxtot = 0;
  for (uint32_t r = 0; r < W; r++) maxtot = std::max<uint64_t>(maxtot, h->desc[r][2 * W]);
  for (uint64_t off = 0; off < maxtot; off += M) {  // round: bytes [off, off + M) of every rank's flat send buffer
    const uint64_t mine = tot > off ? std::min<uint64_t>(M, tot - off) : 0;
    if (mine) MCK(cudaMemcpyAsync(shm_box(g, me), (const uint8_t*)send + off, mine, cudaMemcpyDeviceToHost, s));
    MCK(cudaStreamSynchronize(s));
    SBAR();
    for (uint32_t j = 0; j < W; j++) {  // what rank j has for me in this round
      const uint64_t b0 = h->desc[j][W + me], b1 = b0 + h->desc[j][me];
      const uint64_t lo = std::max<uint64_t>(b0, off), hi = std::min<uint64_t>(b1, off + M);
      if (hi > lo) MCK(cudaMemcpyAsync((uint8_t*)recv + rd[j] + (lo - b0), shm_box(g, j) + (lo - off), hi - lo, cudaMemcpyHostToDevice, s));
    }
    MCK(cudaStreamSynchronize(s));
    SBAR();
  }
  for (uint32_t r = 0; r < W; r++) if (r != me) g->nvlink_bytes += sc[r];
  return PA_OK;
}
// all-reduce(min) as reduce-scatter + all-gather through the mailboxes: every rank reduces ITS slice of the round (1/W of the
// elements, pulled from the W-1 other mailboxes), publishes the reduced slice, and pulls the other reduced slices — 2(W-1)/W of the
// buffer per rank over PCIe instead of (W-1) times the buffer
static int shm_allreduce_min(pa_merge* g, uint32_t* buf, size_t count) {
  const uint32_t W = g->world, me = g->ranks[0];
  const uint64_t M = shm_hdr(g)->mailbox_bytes & ~(uint64_t)3;
  cudaStream_t s = mstream(g, 0);
  const uint64_t bytes = (uint64_t)count * 4;
  if (W == 1) return PA_OK;
  for (uint64_t off = 0; off < bytes; off += M) {
    const uint64_t n = std::min<uint64_t>(M, bytes - off), ne = n / 4;
    const uint64_t per = (ne + W - 1) / W;
    auto slice = [&](uint32_t r, uint64_t* e0, uint64_t* e1) { *e0 = std::min<uint64_t>((uint64_t)r * per, ne); *e1 = std::min<uint64_t>(*e0 + per, ne); };
    uint32_t* round = (uint32_t*)((uint8_t*)buf + off);
    uint64_t m0, m1;
    slice(me, &m0, &m1);
    MCK(g->shm_scratch.ensure(std::max<uint64_t>((m1 - m0) * 4, 256)));
    // phase 1: everybody's round into its own mailbox; each rank reduces its slice
    MCK(cudaMemcpyAsync(shm_box(g, me), round, n, cudaMemcpyDeviceToHost, s));
    MCK(cudaStreamSynchronize(s));
    SBAR();
    if (m1 > m0) {
      const int grid = (int)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)g->members[0]->G, (m1 - m0 + 2047) / 2048));
      for (uint32_t r = 0; r < W; r++) {
        if (r == me) continue;
        MCK(cudaMemcpyAsync(g->shm_scratch.p, shm_box(g, r) + m0 * 4, (m1 - m0) * 4, cudaMemcpyHostToDevice, s));
        k_min_u32<<<grid, kThreads, 0, s>>>(round + m0, g->shm_scratch.as<uint32_t>(), m1 - m0);
      }
    }
    MCK(cudaStreamSynchronize(s));
    SBAR();  // every mailbox has been read: it may be overwritten
    // phase 2: publish the reduced slice, fetch the others
    if (m1 > m0) MCK(cudaMemcpyAsync(shm_box(g, me) + m0 * 4, round + m0, (m1 - m0) * 4, cudaMemcpyDeviceToHost, s));
    MCK(cudaStreamSynchronize(s));
    SBAR();
    for (uint32_t r = 0; r < W; r++) {
      if (r == me) continue;
      uint64_t r0, r1;
      slice(r, &r0, &r1);
      if (r1 > r0) MCK(cudaMemcpyAsync(round + r0, shm_box(g, r) + r0 * 4, (r1 - r0) * 4, cudaMemcpyHostToDevice, s));
    }
    MCK(cudaStreamSynchronize(s));
    SBAR();
  }
  g->nvlink_bytes += bytes * 2 * (W - 1) / W;
  return PA_OK;
}

// host transport: device buffers are staged through pinned memory around the caller's collective (one member per process)
static int xroom(pa_merge* g, size_t send_bytes, size_t recv_bytes) {
  auto grow = [&](uint8_t*& p, size_t& cap, size_t need) -> int {
    if (need <= cap) return PA_OK;
    if (p) cudaFreeHost(p);
    p = nullptr; cap = 0;
    MCK(cudaHostAlloc((void**)&p, need * 2 + 256, cudaHostAllocDefault));
    cap = need * 2 + 256;
    return PA_OK;
  };
  int rc = grow(g->h_xs, g->h_xs_cap, send_bytes);
  return rc ? rc : grow(g->h_xr, g->h_xr_cap, recv_bytes);
}
#define HCK(expr)                                                                            \
  do {                                                                                       \
    if ((expr) != 0) return g->fail(PA_EIO, std::string("host transport callback failed: ") + #expr); \
  } while (0)

// ---- collectives over the members of the group (every call is made for all local members at once) -------------------
// all-gather `bytes` from every rank's device buffer into every member's `dst` (world x bytes)
static int t_allgather(pa_merge* g, const std::vector<const void*>& src, const std::vector<void*>& dst, size_t bytes) {
  const size_t L = g->members.size();
  if (g->shm) {
    const double th0 = now_ms();
    std::vector<uint64_t> cnt(g->world, bytes), dsp(g->world);
    for (uint32_t r = 0; r < g->world; r++) dsp[r] = (uint64_t)r * bytes;
    int rc = shm_allgatherv(g, src[0], dst[0], cnt, dsp);
    g->ms_exchange_wait += now_ms() - th0;
    return rc;
  }
  if (g->host) {
    const double th0 = now_ms();
    int rc = xroom(g, bytes, (size_t)g->world * bytes);
    if (rc) return rc;
    cudaStream_t s = mstream(g, 0);
    MCK(cudaMemcpyAsync(g->h_xs, src[0], bytes, cudaMemcpyDeviceToHost, s));
    MCK(cudaStreamSynchronize(s));
    HCK(g->host->allgather(g->host->user, g->h_xs, g->h_xr, bytes));
    MCK(cudaMemcpyAsync(dst[0], g->h_xr, (size_t)g->world * bytes, cudaMemcpyHostToDevice, s));
    MCK(cudaStreamSynchronize(s));
    g->nvlink_bytes += bytes * (g->world - 1);
    g->ms_exchange_wait += now_ms() - th0;  // host transport: the stream idles while the caller's collective runs
  } else if (g->use_nccl) {
    NcclApi* n = nccl_api();
    NCK(n->GroupStart());
    for (size_t i = 0; i < L; i++) NCK(n->AllGather(src[i], dst[i], bytes, ncclChar, g->comms[i], mstream(g, i)));
    NCK(n->GroupEnd());
    g->nvlink_bytes += (uint64_t)L * bytes * (g->world - 1);
  } else {
    for (size_t i = 0; i < L; i++)
      for (size_t j = 0; j < L; j++) MCK(cudaMemcpyAsync((uint8_t*)dst[i] + (size_t)g->ranks[j] * bytes, src[j], bytes, cudaMemcpyDeviceToDevice, mstream(g, i)));
  }
  return PA_OK;
}
// the same, landing in host memory (out: world x bytes); synchronises
static int t_allgather_host(pa_merge* g, const std::vector<const void*>& src, size_t bytes, std::vector<uint8_t>& out) {
  const size_t L = g->members.size();
  if (g->shm && bytes <= shm_hdr(g)->mailbox_bytes) {  // small control blocks: straight out of the mailboxes, no trip back through the device
    const double th0 = now_ms();
    cudaStream_t s = mstream(g, 0);
    if (bytes) MCK(cudaMemcpyAsync(shm_box(g, g->ranks[0]), src[0], bytes, cudaMemcpyDeviceToHost, s));
    MCK(cudaStreamSynchronize(s));
    SBAR();
    out.resize((size_t)g->world * bytes);
    for (uint32_t r = 0; r < g->world; r++) memcpy(out.data() + (size_t)r * bytes, shm_box(g, r), bytes);
    SBAR();
    g->ms_exchange_wait += now_ms() - th0;
    return PA_OK;
  }
  std::vector<void*> dst(L);
  for (size_t i = 0; i < L; i++) {
    MCK(cudaSetDevice(g->members[i]->device));
    MCK(g->mb[i].gather_scratch.ensure(std::max<size_t>((size_t)g->world * bytes, 256)));
    dst[i] = g->mb[i].gather_scratch.p;
  }
  int rc = t_allgather(g, src, dst, bytes);
  if (rc) return rc;
  if ((rc = pin_room(g, (size_t)g->world * bytes))) return rc;
  MCK(cudaSetDevice(g->members[0]->device));
  MCK(cudaMemcpyAsync(g->h_pin, dst[0], (size_t)g->world * bytes, cudaMemcpyDeviceToHost, mstream(g, 0)));
  const double t0 = now_ms();
  if ((rc = msync(g))) return rc;
  g->ms_exchange_wait += now_ms() - t0;
  out.assign(g->h_pin, g->h_pin + (size_t)g->world * bytes);
  return PA_OK;
}
// all-gather with per-rank byte counts; dst holds rank r's block at displ[r]
static int t_allgatherv(pa_merge* g, const std::vector<const void*>& src, const std::vector<void*>& dst, const std::vector<uint64_t>& count, const std::vector<uint64_t>& displ) {
  const size_t L = g->members.size();
  if (g->shm) {
    const double th0 = now_ms();
    int rc = shm_allgatherv(g, src[0], dst[0], count, displ);
    g->ms_exchange_wait += now_ms() - th0;
    return rc;
  }
  if (g->host) {
    const double th0 = now_ms();
    uint64_t total = 0;
    for (uint32_t r = 0; r < g->world; r++) total = std::max<uint64_t>(total, displ[r] + count[r]);
    const uint64_t mine = count[g->ranks[0]];
    int rc = xroom(g, std::max<uint64_t>(mine, 1), std::max<uint64_t>(total, 1));
    if (rc) return rc;
    cudaStream_t s = mstream(g, 0);
    if (mine) MCK(cudaMemcpyAsync(g->h_xs, src[0], mine, cudaMemcpyDeviceToHost, s));
    MCK(cudaStreamSynchronize(s));
    HCK(g->host->allgatherv(g->host->user, g->h_xs, g->h_xr, count.data(), displ.data()));
    if (total) MCK(cudaMemcpyAsync(dst[0], g->h_xr, total, cudaMemcpyHostToDevice, s));
    MCK(cudaStreamSynchronize(s));
    g->nvlink_bytes += mine * (g->world - 1);
    g->ms_exchange_wait += now_ms() - th0;  // host transport: the stream idles while the caller's collective runs
  } else if (g->use_nccl) {
    NcclApi* n = nccl_api();
    NCK(n->GroupStart());
    for (size_t i = 0; i < L; i++)
      for (uint32_t r = 0; r < g->world; r++) {
        if (!count[r]) continue;
        void* at = (uint8_t*)dst[i] + displ[r];
        NCK(n->Broadcast(r == g->ranks[i] ? src[i] : at, at, count[r], ncclChar, (int)r, g->comms[i], mstream(g, i)));
      }
    NCK(n->GroupEnd());
    for (size_t i = 0; i < L; i++) g->nvlink_bytes += count[g->ranks[i]] * (g->world - 1);
  } else {
    for (size_t i = 0; i < L; i++)
      for (size_t j = 0; j < L; j++)
        if (count[g->ranks[j]]) MCK(cudaMemcpyAsync((uint8_t*)dst[i] + displ[g->ranks[j]], src[j], count[g->ranks[j]], cudaMemcpyDeviceToDevice, mstream(g, i)));
  }
  return PA_OK;
}
// all-to-all with byte counts: member i sends scount[i][r] bytes at sdispl[i][r] to rank r, receives rcount[i][r] at rdispl[i][r]
static int t_alltoallv(pa_merge* g, const std::vector<const void*>& send, const std::vector<std::vector<uint64_t>>& scount, const std::vector<std::vector<uint64_t>>& sdispl,
                       const std::vector<void*>& recv, const std::vector<std::vector<uint64_t>>& rcount, const std::vector<std::vector<uint64_t>>& rdispl) {
  const size_t L = g->members.size();
  if (g->shm) {
    const double th0 = now_ms();
    int rc = shm_alltoallv(g, send[0], scount[0], sdispl[0], recv[0], rdispl[0]);
    g->ms_exchange_wait += now_ms() - th0;
    return rc;
  }
  if (g->host) {
    const double th0 = now_ms();
    uint64_t stot = 0, rtot = 0;
    for (uint32_t r = 0; r < g->world; r++) { stot = std::max<uint64_t>(stot, sdispl[0][r] + scount[0][r]); rtot = std::max<uint64_t>(rtot, rdispl[0][r] + rcount[0][r]); }
    int rc = xroom(g, std::max<uint64_t>(stot, 1), std::max<uint64_t>(rtot, 1));
    if (rc) return rc;
    cudaStream_t s = mstream(g, 0);
    if (stot) MCK(cudaMemcpyAsync(g->h_xs, send[0], stot, cudaMemcpyDeviceToHost, s));
    MCK(cudaStreamSynchronize(s));
    HCK(g->host->alltoallv(g->host->user, g->h_xs, scount[0].data(), sdispl[0].data(), g->h_xr, rcount[0].data(), rdispl[0].data()));
    if (rtot) MCK(cudaMemcpyAsync(recv[0], g->h_xr, rtot, cudaMemcpyHostToDevice, s));
    MCK(cudaStreamSynchronize(s));
    for (uint32_t r = 0; r < g->world; r++) if (r != g->ranks[0]) g->nvlink_bytes += scount[0][r];
    g->ms_exchange_wait += now_ms() - th0;  // host transport: the stream idles while the caller's collective runs
  } else if (g->use_nccl) {
    NcclApi* n = nccl_api();
    for (size_t i = 0; i < L; i++) {  // the part that stays on the shard
      const uint32_t me = g->ranks[i];
      if (scount[i][me]) { MCK(cudaSetDevice(g->members[i]->device)); MCK(cudaMemcpyAsync((uint8_t*)recv[i] + rdispl[i][me], (const uint8_t*)send[i] + sdispl[i][me], scount[i][me], cudaMemcpyDeviceToDevice, mstream(g, i))); }
    }
    NCK(n->GroupStart());
    for (size_t i = 0; i < L; i++)
      for (uint32_t r = 0; r < g->world; r++) {
        if (r == g->ranks[i]) continue;
        if (scount[i][r]) { NCK(n->Send((const uint8_t*)send[i] + sdispl[i][r], scount[i][r], ncclChar, (int)r, g->comms[i], mstream(g, i))); g->nvlink_bytes += scount[i][r]; }
        if (rcount[i][r]) NCK(n->Recv((uint8_t*)recv[i] + rdispl[i][r], rcount[i][r], ncclChar, (int)r, g->comms[i], mstream(g, i)));
      }
    NCK(n->GroupEnd());
  } else {
    for (size_t i = 0; i < L; i++)     // receiver
      for (size_t j = 0; j < L; j++) {  // sender
        const uint32_t ri = g->ranks[i], rj = g->ranks[j];
        if (scount[j][ri]) MCK(cudaMemcpyAsync((uint8_t*)recv[i] + rdispl[i][rj], (const uint8_t*)send[j] + sdispl[j][ri], scount[j][ri], cudaMemcpyDeviceToDevice, mstream(g, i)));
      }
  }
  return PA_OK;
}
static int t_allreduce_min(pa_merge* g, const std::vector<uint32_t*>& buf, size_t count) {
  const size_t L = g->members.size();
  if (!count) return PA_OK;
  if (g->shm) {
    const double th0 = now_ms();
    int rc = shm_allreduce_min(g, buf[0], count);
    g->ms_exchange_wait += now_ms() - th0;
    return rc;
  }
  if (g->host) {
    const double th0 = now_ms();
    int rc = xroom(g, count * 4, 1);
    if (rc) return rc;
    cudaStream_t s = mstream(g, 0);
    MCK(cudaMemcpyAsync(g->h_xs, buf[0], count * 4, cudaMemcpyDeviceToHost, s));
    MCK(cudaStreamSynchronize(s));
    HCK(g->host->allreduce_min_u32(g->host->user, (uint32_t*)g->h_xs, (uint64_t)count));
    MCK(cudaMemcpyAsync(buf[0], g->h_xs, count * 4, cudaMemcpyHostToDevice, s));
    MCK(cudaStreamSynchronize(s));
    g->nvlink_bytes += (uint64_t)count * 4 * 2 * (g->world - 1) / g->world;
    g->ms_exchange_wait += now_ms() - th0;  // host transport: the stream idles while the caller's collective runs
  } else if (g->use_nccl) {
    NcclApi* n = nccl_api();
    NCK(n->GroupStart());
    for (size_t i = 0; i < L; i++) NCK(n->AllReduce(buf[i], buf[i], count, ncclUint32, ncclMin, g->comms[i], mstream(g, i)));
    NCK(n->GroupEnd());
    g->nvlink_bytes += (uint64_t)L * count * 4 * 2 * (g->world - 1) / g->world;  // ring-equivalent volume
  } else {
    cudaStream_t s = mstream(g, 0);
    const int grid = (int)std::max<size_t>(1, std::min<size_t>((size_t)g->members[0]->G, (count + 2047) / 2048));
    for (size_t j = 1; j < L; j++) k_min_u32<<<grid, kThreads, 0, s>>>(buf[0], buf[j], count);
    for (size_t j = 1; j < L; j++) MCK(cudaMemcpyAsync(buf[j], buf[0], count * 4, cudaMemcpyDeviceToDevice, s));
  }
  return PA_OK;
}

// ---------------------------------------------------------------------------------------------------------------------
static int merge_process_once(pa_merge* g, bool* retry) {
  const size_t L = g->members.size();
  const uint32_t W = g->world;
  *retry = false;
  g->nvlink_bytes = 0;
  g->ms_exchange_wait = 0;
  int rc;
  // ---- plan + local front (header split, XXH64 + local dedup) on every member
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    MCK(cudaSetDevice(a->device));
    MergeBufs& mb = g->mb[i];
    MCK(mb.ctl.ensure(CTL_WORDS * 4));
    MergeDims md;
    md.world = W; md.rank = g->ranks[i]; md.row_base = g->row_base[g->ranks[i]]; md.n_total = g->NT; md.nf_total = g->NFT;
    md.slice_len_ptr = mb.ctl.as<uint32_t>() + CTL_MERGE + 3;  // MergeCtl::slice_len
    if ((rc = pass_plan(a, &md))) return g->fail(rc, a->err);
    a->P.jobs[a->P.j_loc].n_map_ptr = md.slice_len_ptr;  // this shard maps only its range of the stream
    if ((rc = upload_descriptors(a, a->P.jobs.data(), a->P.jobs.size() * sizeof(FoJob), a->P.rc.data(), a->P.rc.size() * sizeof(ReeCol)))) return g->fail(rc, a->err);
    MCK(cudaMemsetAsync(mb.ctl.p, 0, CTL_WORDS * 4, a->s_comp));
    if ((rc = pass_front(a))) return g->fail(rc, a->err);
  }
  // ---- stacks: count per owner, thread-id list; sizes to the host (sync 1)
  std::vector<const void*> csrc(L);
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    MCK(cudaSetDevice(a->device));
    cudaStream_t s = a->s_comp;
    MergeBufs& mb = g->mb[i];
    uint32_t* ctl = mb.ctl.as<uint32_t>();
    Counters* ctr = a->d_ctr.as<Counters>();
    MCK(cudaEventRecord(a->tm[T_RANK].a, s));
    const int Gu = small_grid(a, std::min<uint64_t>(std::max<uint64_t>(a->N, 1), a->P.cap / 2));
    k_owner_count<<<Gu, kThreads, 0, s>>>(a->d_table.as<StackSlot>(), a->P.claimed, &ctr->n_claimed, W, ctl + CTL_CNT);
    if (a->tid_slots) {
      MCK(mb.tid_list.ensure(std::max<uint64_t>(std::min<uint64_t>(a->P.tcap, std::max<uint64_t>(a->N, 1)), 32) * 8));
      k_tid_pack<<<small_grid(a, a->P.tcap), kThreads, 0, s>>>(a->tid_slots, a->tid_mask, ctl + CTL_MERGE + 4 /* MergeCtl::n_tids */, mb.tid_list.as<unsigned long long>());
    }
    // [cnt[0..W) | n_tids | local err] in one block: cnt lives at CTL_CNT; copy the two scalars behind it
    MCK(cudaMemcpyAsync(ctl + CTL_CNT + W, ctl + CTL_MERGE + 4, 4, cudaMemcpyDeviceToDevice, s));
    MCK(cudaMemcpyAsync(ctl + CTL_CNT + W + 1, &ctr->err, 4, cudaMemcpyDeviceToDevice, s));
    a->tm[T_RANK].launches += 2;
    csrc[i] = ctl + CTL_CNT;
  }
  std::vector<uint8_t> hb;
  const size_t cw = (size_t)W + 2;
  if ((rc = t_allgather_host(g, csrc, cw * 4, hb))) return rc;
  const uint32_t* hc = (const uint32_t*)hb.data();  // [rank][W+2]
  auto cnt_of = [&](uint32_t from, uint32_t to) { return (uint64_t)hc[(size_t)from * cw + to]; };
  for (uint32_t r = 0; r < W; r++)
    if (hc[(size_t)r * cw + W + 1] & ERR_TABLE_FULL) { *retry = true; }
  if (*retry) { g->retry_err = ERR_TABLE_FULL; return PA_OK; }  // some shard's local table was too small: every member redoes the batch with larger ones
  if (g->group_retire) {  // a stale handle is seen only by the shard whose rows carry it: every rank stops here, before the exchange
    uint32_t e = 0;
    for (uint32_t r = 0; r < W; r++) e |= hc[(size_t)r * cw + W + 1];
    if (e & ERR_BAD_STACK_ID) {
      for (size_t i = 0; i < L; i++) g->members[i]->h_ctr.err = e;
      return PA_OK;
    }
  }
  // ---- pack by owner, all-to-all
  std::vector<const void*> sendp(L);
  std::vector<void*> recvp(L);
  std::vector<std::vector<uint64_t>> sc(L, std::vector<uint64_t>(W)), sd(L, std::vector<uint64_t>(W)), rcn(L, std::vector<uint64_t>(W)), rd(L, std::vector<uint64_t>(W));
  std::vector<uint64_t> n_recv(L);
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    MCK(cudaSetDevice(a->device));
    cudaStream_t s = a->s_comp;
    MergeBufs& mb = g->mb[i];
    const uint32_t me = g->ranks[i];
    uint32_t* ctl = mb.ctl.as<uint32_t>();
    Counters* ctr = a->d_ctr.as<Counters>();
    OwnerOffsets oo{};
    uint64_t tot_s = 0, tot_r = 0;
    for (uint32_t r = 0; r < W; r++) {
      oo.off[r] = (uint32_t)tot_s;
      sc[i][r] = cnt_of(me, r) * sizeof(StackEntry); sd[i][r] = tot_s * sizeof(StackEntry); tot_s += cnt_of(me, r);
      rcn[i][r] = cnt_of(r, me) * sizeof(StackEntry); rd[i][r] = tot_r * sizeof(StackEntry); tot_r += cnt_of(r, me);
    }
    oo.off[W] = (uint32_t)tot_s;
    n_recv[i] = tot_r;
    MCK(mb.send.ensure(std::max<uint64_t>(tot_s, 1) * sizeof(StackEntry)));
    MCK(mb.recv.ensure(std::max<uint64_t>(tot_r, 1) * sizeof(StackEntry)));
    const int Gu = small_grid(a, std::max<uint64_t>(tot_s, 1));
    k_owner_pack<<<Gu, kThreads, 0, s>>>(a->d_table.as<StackSlot>(), a->P.claimed, &ctr->n_claimed, W, oo, ctl + CTL_CURSOR, (uint32_t)a->P.row_base, a->d_nfr.as<uint16_t>(), mb.send.as<StackEntry>());
    a->tm[T_RANK].launches++;
    sendp[i] = mb.send.p; recvp[i] = mb.recv.p;
  }
  if ((rc = t_alltoallv(g, sendp, sc, sd, recvp, rcn, rd))) return rc;
  // ---- thread ids: all-gather the lists, insert the others' entries
  {
    std::vector<uint64_t> tcount(W), tdispl(W);
    uint64_t ttot = 0;
    for (uint32_t r = 0; r < W; r++) { tcount[r] = (uint64_t)hc[(size_t)r * cw + W] * 8; tdispl[r] = ttot; ttot += tcount[r]; }
    bool any_tid = false;
    for (size_t i = 0; i < L; i++) any_tid |= g->members[i]->tid_slots != nullptr;
    if (any_tid && ttot) {
      std::vector<const void*> ts(L);
      std::vector<void*> td(L);
      for (size_t i = 0; i < L; i++) {
        MCK(cudaSetDevice(g->members[i]->device));
        MCK(g->mb[i].tid_all.ensure(ttot));
        ts[i] = g->mb[i].tid_list.p; td[i] = g->mb[i].tid_all.p;
      }
      if ((rc = t_allgatherv(g, ts, td, tcount, tdispl))) return rc;
      for (size_t i = 0; i < L; i++) {
        pa_agg* a = g->members[i];
        MCK(cudaSetDevice(a->device));
        k_tid_insert<<<small_grid(a, ttot / 8), kThreads, 0, a->s_comp>>>(g->mb[i].tid_all.as<unsigned long long>(), (uint32_t)(ttot / 8), a->tid_slots, a->tid_mask, a->d_ctr.as<Counters>());
        a->tm[T_RANK].launches++;
      }
    }
  }
  // ---- owners: keep the minimum row per id; list of owned ids; sizes to the host (sync 2)
  std::vector<uint64_t> ocap(L);
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    MCK(cudaSetDevice(a->device));
    cudaStream_t s = a->s_comp;
    MergeBufs& mb = g->mb[i];
    uint32_t* ctl = mb.ctl.as<uint32_t>();
    ocap[i] = std::max<uint64_t>(pow2_at_least(2 * std::max<uint64_t>(n_recv[i], 1)), 1024);
    MCK(mb.otab.ensure((ocap[i] + 2) * sizeof(StackSlot)));
    MCK(mb.oclaimed.ensure((std::max<uint64_t>(n_recv[i], 1) + 1) * 4));
    MCK(mb.ouniq.ensure(std::max<uint64_t>(n_recv[i], 1) * sizeof(StackEntry)));
    MCK(cudaMemsetAsync(mb.otab.p, 0, (ocap[i] + 2) * sizeof(StackSlot), s));
    const int Gr = small_grid(a, std::max<uint64_t>(n_recv[i], 1));
    k_entries_insert<<<Gr, kThreads, 0, s>>>(mb.recv.as<StackEntry>(), (uint32_t)n_recv[i], mb.otab.as<StackSlot>(), (uint32_t)(ocap[i] - 1), ctl + CTL_OWNER, mb.oclaimed.as<uint32_t>());
    k_entries_compact<<<Gr, kThreads, 0, s>>>(mb.otab.as<StackSlot>(), mb.oclaimed.as<uint32_t>(), ctl + CTL_OWNER, mb.ouniq.as<StackEntry>());
    a->tm[T_RANK].launches += 2;
    csrc[i] = ctl + CTL_OWNER;
  }
  if ((rc = t_allgather_host(g, csrc, 4, hb))) return rc;
  std::vector<uint64_t> ucount(W), udispl(W);
  uint64_t U = 0;
  for (uint32_t r = 0; r < W; r++) { ucount[r] = (uint64_t)((const uint32_t*)hb.data())[r] * sizeof(StackEntry); udispl[r] = U * sizeof(StackEntry); U += ((const uint32_t*)hb.data())[r]; }
  // ---- merged dictionary on every shard: all-gather the owners' lists, insert, rank by global first row
  {
    std::vector<const void*> us(L);
    std::vector<void*> ud(L);
    for (size_t i = 0; i < L; i++) {
      MCK(cudaSetDevice(g->members[i]->device));
      MergeBufs& mb = g->mb[i];
      MCK(mb.glist.ensure(std::max<uint64_t>(U, 1) * sizeof(StackEntry)));
      us[i] = mb.ouniq.p; ud[i] = mb.glist.p;
    }
    if ((rc = t_allgatherv(g, us, ud, ucount, udispl))) return rc;
  }
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    MCK(cudaSetDevice(a->device));
    cudaStream_t s = a->s_comp;
    MergeBufs& mb = g->mb[i];
    Pass& P = a->P;
    uint32_t* ctl = mb.ctl.as<uint32_t>();
    Counters* ctr = a->d_ctr.as<Counters>();
    const uint64_t gcap = std::max<uint64_t>(pow2_at_least(2 * std::max<uint64_t>(U, 1)), 1024), Un = std::max<uint64_t>(U, 1);
    MCK(mb.gtab.ensure((gcap + 2) * sizeof(StackSlot)));
    MCK(mb.gclaimed.ensure((Un + 1) * 4)); MCK(mb.g_uniq_row.ensure(Un * 4)); MCK(mb.g_uniq_slot.ensure(Un * 4)); MCK(mb.g_uniq_size.ensure(Un * 4));
    StackSlot* gtab = mb.gtab.as<StackSlot>();
    const uint32_t gmask = (uint32_t)(gcap - 1);
    uint32_t *gclaimed = mb.gclaimed.as<uint32_t>(), *urow = mb.g_uniq_row.as<uint32_t>(), *uslot = mb.g_uniq_slot.as<uint32_t>(), *usize = mb.g_uniq_size.as<uint32_t>();
    MCK(cudaMemsetAsync(gtab, 0, (gcap + 2) * sizeof(StackSlot), s));
    const int Gu = small_grid(a, Un), Gw = small_grid(a, g->NT / 32 + 1);
    k_entries_insert<<<Gu, kThreads, 0, s>>>(mb.glist.as<StackEntry>(), (uint32_t)U, gtab, gmask, ctl + CTL_MERGED, gclaimed);
    k_merged_unpack<<<Gu, kThreads, 0, s>>>(gtab, gclaimed, ctl + CTL_MERGED);
    k_stack_bits<<<Gu, kThreads, 0, s>>>(gtab, gclaimed, ctl + CTL_MERGED, P.rowbits);
    launch_scan(a, WordsF{P.rowbits, P.row_wprefix, (uint32_t)((g->NT + 31) / 32), &ctr->n_unique}, 1, a->tm[T_RANK], Gw, s, a->d_partial);
    k_stack_assign<<<Gu, kThreads, 0, s>>>(gtab, gclaimed, ctl + CTL_MERGED, P.rowbits, P.row_wprefix, nullptr, urow, uslot, usize);
    launch_scan(a, UniqOffsetF{ctr, ctr, usize, uslot, gtab}, 1, a->tm[T_RANK], Gu, s, a->d_partial);
    // every local stack adopts the merged (ordinal, offset, size); rows pick them up; this shard's range of the stream
    const int Gl = small_grid(a, std::min<uint64_t>(std::max<uint64_t>(a->N, 1), P.cap / 2));
    k_local_adopt<<<Gl, kThreads, 0, s>>>(a->d_table.as<StackSlot>(), P.claimed, &ctr->n_claimed, gtab, gmask, ctl + CTL_MERGED, &ctr->err);
    k_rows_materialize<<<a->G, kThreads, 0, s>>>((uint32_t)a->N, a->d_slot.as<uint32_t>(), a->d_table.as<StackSlot>(), a->d_stoff.as<int>(), a->d_stsize.as<int>(),
                                                 P.v1 ? a->v1_ord : nullptr);
    // (v1 has no location-index stream: the won range only tells which stacks' frames this shard sends to the store update)
    const uint64_t ucap = P.v1 ? 0x7FFFFFFFull : std::min<uint64_t>(a->d_ustream.cap / 4, 0x7FFFFFFFull);
    k_won_range<<<1, 32, 0, s>>>(urow, uslot, gtab, ctr, (uint32_t)P.row_base, (uint32_t)a->N, (uint32_t)ucap, (MergeCtl*)(ctl + CTL_MERGE), ctr);
    if (P.v1) {  // the stacktrace_id dictionary, replicated: every shard writes the merged ids from the merged table
      MCK(a->d_v1_ids.ensure(Un * 16));
      MCK(mb.v1_off.ensure((Un + 1) * 4));
      a->v1_ids = a->d_v1_ids.as<uint8_t>();
      a->v1_id_off = mb.v1_off.as<int>();
      k_merged_ids<<<small_grid(a, Un + 1), kThreads, 0, s>>>(ctr, gtab, uslot, a->v1_ids, a->v1_id_off);
    } else {
      k_gather_won<<<a->G, kThreads, 0, s>>>((const MergeCtl*)(ctl + CTL_MERGE), urow, uslot, gtab, (uint32_t)P.row_base, a->src_frames, a->d_foff.as<unsigned long long>(),
                                             P.n_frames, a->d_ustream.as<uint32_t>(), a->loc_first, ctr, a->idb == 4 ? 1u : 0u);
    }
    a->tm[T_RANK].launches += 8;
    MCK(cudaEventRecord(a->tm[T_RANK].b, s));
  }
  // ---- first positions of frames (v2) / first rows of label values (v1: and of sample kinds): one all-reduce(min) each
  const bool v1 = g->members[0]->P.v1;
  {
    std::vector<uint32_t*> lf(L), rb(L);
    for (size_t i = 0; i < L; i++) { lf[i] = g->members[i]->loc_first; rb[i] = g->members[i]->P.red_block; }
    if (!v1 && (rc = t_allreduce_min(g, lf, g->members[0]->P.Pn))) return rc;
    if ((rc = t_allreduce_min(g, rb, g->members[0]->P.red_count))) return rc;
  }
  // ---- dictionaries (identical on every shard), run counts, run edges
  std::vector<const void*> esrc(L);
  std::vector<void*> edst(L);
  const uint32_t ncols = g->ncols;
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    MCK(cudaSetDevice(a->device));
    cudaStream_t s = a->s_comp;
    MergeBufs& mb = g->mb[i];
    if (!v1 && (rc = pass_locations(a))) return g->fail(rc, a->err);  // (the v1 record has no location or function dictionaries)
    if ((rc = pass_labels_count(a, s))) return g->fail(rc, a->err);
    MCK(mb.edges.ensure(std::max<size_t>((size_t)ncols * sizeof(EdgeCol), 256)));
    MCK(mb.edges_all.ensure(std::max<size_t>((size_t)W * ncols * sizeof(EdgeCol), 256)));
    MCK(mb.mcols.ensure(std::max<size_t>((size_t)ncols * sizeof(MergeCol), 256)));
    MCK(mb.mcols_all.ensure(std::max<size_t>((size_t)W * ncols * sizeof(MergeCol), 256)));
    k_edges_pack<<<1, kThreads, 0, s>>>(a->d_ctr.as<Counters>(), a->P.edge_keys, ncols, (uint32_t)a->P.row_base, (uint32_t)a->N, mb.edges.as<EdgeCol>());
    a->tm[T_LABELS].launches++;
    esrc[i] = mb.edges.p; edst[i] = mb.edges_all.p;
  }
  if ((rc = t_allgather(g, esrc, edst, (size_t)ncols * sizeof(EdgeCol)))) return rc;
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    MCK(cudaSetDevice(a->device));
    cudaStream_t s = a->s_comp;
    MergeBufs& mb = g->mb[i];
    k_merge_cols<<<1, kThreads, 0, s>>>(mb.edges_all.as<EdgeCol>(), W, g->ranks[i], ncols, mb.mcols.as<MergeCol>(), mb.mcols_all.as<MergeCol>(), a->d_ctr.as<Counters>());
    a->tm[T_LABELS].launches++;
    a->P.ra.mc = mb.mcols.as<MergeCol>();
    if ((rc = pass_label_dicts(a, s, a->d_partial))) return g->fail(rc, a->err);
    if ((rc = pass_labels_emit(a, s))) return g->fail(rc, a->err);
  }
  // ---- results to the host
  g->cols_all.assign((size_t)W * ncols, MergeCol{});
  g->mctl.assign(L, MergeCtl{});
  if ((rc = pin_room(g, (size_t)W * ncols * sizeof(MergeCol) + L * sizeof(MergeCtl) + 64))) return rc;
  MergeCol* h_cols = (MergeCol*)g->h_pin;
  MergeCtl* h_ctl = (MergeCtl*)(g->h_pin + (((size_t)W * ncols * sizeof(MergeCol) + 63) & ~(size_t)63));
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    MCK(cudaSetDevice(a->device));
    if (i == 0 && ncols) MCK(cudaMemcpyAsync(h_cols, g->mb[i].mcols_all.p, (size_t)W * ncols * sizeof(MergeCol), cudaMemcpyDeviceToHost, a->s_comp));
    MCK(cudaMemcpyAsync(h_ctl + i, g->mb[i].ctl.as<uint32_t>() + CTL_MERGE, sizeof(MergeCtl), cudaMemcpyDeviceToHost, a->s_comp));
    if ((rc = pass_finish(a))) return g->fail(rc, a->err);
  }
  if (ncols) memcpy(g->cols_all.data(), h_cols, (size_t)W * ncols * sizeof(MergeCol));
  for (size_t i = 0; i < L; i++) g->mctl[i] = h_ctl[i];
  // ---- every member must agree on the outcome (sync 3)
  for (size_t i = 0; i < L; i++) csrc[i] = &g->members[i]->d_ctr.as<Counters>()->err;
  if ((rc = t_allgather_host(g, csrc, 4, hb))) return rc;
  uint32_t err_any = 0;
  for (uint32_t r = 0; r < W; r++) err_any |= ((const uint32_t*)hb.data())[r];
  // (a label-plan miss is the same on every member: k_ls_plan ran on the all-reduced first_ls, so each member's used-name
  // bitmap is the union of every shard's, and every member replans the same columns)
  if (err_any & (ERR_TABLE_FULL | ERR_LABEL_PLAN)) { *retry = true; g->retry_err = err_any; return PA_OK; }
  for (size_t i = 0; i < L; i++) g->members[i]->h_ctr.err |= err_any;
  return PA_OK;
}

// ---- v1 groups: every member holds a full copy of the group's known-stacks store ---------------------------------------
// A group of v1 members behaves like ONE v1 aggregator fed [shard 0's rows, shard 1's rows, ...]: each member applies the
// merged batch's accesses to its copy (v1_store_update's steps, over merged ordinals), so the copies stay identical and each
// one stays a valid store of its own member. Exchanged per interval: the global last row of every merged stack (all-reduce(min)
// over U words), and the frames of the stacks the store lacks, each sent by the shard that holds its global first occurrence
// (all-gather-v; near zero in steady state). Every decision below depends only on replicated state, so every rank takes it.

// the frames the insert may need (k_store_need on the store as it is now), gathered into every member's v1_frames; in
// PA_CFG_GROUP_STACKS groups one handle per such stack instead (v1_foff then indexes references, not frames)
static int store_frames_exchange(pa_merge* g, uint32_t min_last_p1) {
  const size_t L = g->members.size();
  const uint32_t W = g->world;
  const uint64_t U = g->members[0]->h_ctr.n_unique;
  const bool refs = g->group_stacks;
  const uint64_t unit = refs ? 8 : 4;
  std::vector<std::vector<uint64_t>> bounds(L, std::vector<uint64_t>(W + 1));
  RankRows rr{};
  for (uint32_t r = 0; r <= W; r++) rr.base[r] = (uint32_t)g->row_base[r];
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    MCK(cudaSetDevice(a->device));
    cudaStream_t s = a->s_comp;
    MergeBufs& mb = g->mb[i];
    Counters* ctr = a->d_ctr.as<Counters>();
    MCK(mb.v1_need.ensure(std::max<uint64_t>(U, 1) * 4));
    MCK(mb.v1_foff.ensure((U + 1) * 8));
    MCK(mb.v1_bounds.ensure((W + 1) * 8));
    k_store_need<<<small_grid(a, U), kThreads, 0, s>>>(ctr, mb.gtab.as<StackSlot>(), mb.g_uniq_slot.as<uint32_t>(), mb.v1_last.as<uint32_t>(), min_last_p1,
                                                       a->d_store.as<StoreSlot>(), (uint32_t)(a->store_slots - 1), a->d_store_stamp.as<unsigned long long>(),
                                                       mb.v1_need.as<uint32_t>());
    if (refs) launch_scan(a, StoreRefsF{ctr, mb.v1_need.as<uint32_t>(), mb.v1_foff.as<unsigned long long>()}, 1, a->tm[T_RANK], small_grid(a, U), s, a->d_partial);
    else launch_scan(a, StoreFramesF{ctr, mb.v1_need.as<uint32_t>(), mb.v1_foff.as<unsigned long long>()}, 1, a->tm[T_RANK], small_grid(a, U), s, a->d_partial);
    k_rank_bounds<<<1, kMaxWorld + 32, 0, s>>>(ctr, mb.g_uniq_row.as<uint32_t>(), mb.v1_foff.as<unsigned long long>(), rr, W, mb.v1_bounds.as<unsigned long long>());
    MCK(cudaMemcpyAsync(bounds[i].data(), mb.v1_bounds.p, (W + 1) * 8, cudaMemcpyDeviceToHost, s));
  }
  int rc = msync(g);
  if (rc) return rc;
  const std::vector<uint64_t>& b = bounds[0];  // identical on every member
  std::vector<uint64_t> count(W), displ(W);
  for (uint32_t r = 0; r < W; r++) { displ[r] = b[r] * unit; count[r] = (b[r + 1] - b[r]) * unit; }
  std::vector<const void*> src(L);
  std::vector<void*> dst(L);
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    MCK(cudaSetDevice(a->device));
    MergeBufs& mb = g->mb[i];
    const uint32_t me = g->ranks[i];
    MCK(mb.v1_send.ensure(std::max<uint64_t>(count[me], 256)));
    MCK(mb.v1_frames.ensure(std::max<uint64_t>(b[W] * unit, 256)));
    if (refs) {
      static_assert(sizeof(pa_sample_hdr) == 64, "k_store_pack_refs reads the handles 8 words apart");
      k_store_pack_refs<<<small_grid(a, U), kThreads, 0, a->s_comp>>>((const MergeCtl*)(mb.ctl.as<uint32_t>() + CTL_MERGE), mb.g_uniq_row.as<uint32_t>(),
                                                                      (uint32_t)g->row_base[me], mb.v1_need.as<uint32_t>(), mb.v1_foff.as<unsigned long long>(),
                                                                      a->d_hdr.as<unsigned long long>() + offsetof(pa_sample_hdr, frame_off) / 8,
                                                                      mb.v1_send.as<unsigned long long>());
      a->store_refs_sent += count[me] / 8;
      src[i] = mb.v1_send.p; dst[i] = mb.v1_frames.p;
      continue;
    }
    k_store_pack<<<a->G, kThreads, 0, a->s_comp>>>((const MergeCtl*)(mb.ctl.as<uint32_t>() + CTL_MERGE), mb.g_uniq_row.as<uint32_t>(), (uint32_t)g->row_base[me],
                                                   mb.v1_need.as<uint32_t>(), mb.v1_foff.as<unsigned long long>(), a->src_frames, a->d_foff.as<unsigned long long>(),
                                                   a->P.n_frames, a->idb == 4 ? 1u : 0u, mb.v1_send.as<uint32_t>(), a->d_ctr.as<Counters>());
    a->store_frames_sent += count[me] / 4;
    src[i] = mb.v1_send.p; dst[i] = mb.v1_frames.p;
  }
  return b[W] ? t_allgatherv(g, src, dst, count, displ) : PA_OK;
}

// v1_store_update for every member's copy, after the merged pass (h_ctr holds the merged counters)
static int merge_store_update(pa_merge* g) {
  const size_t L = g->members.size();
  const uint64_t U = g->members[0]->h_ctr.n_unique, C = g->members[0]->store_entries;
  int rc;
  // ---- global last row of every merged stack
  std::vector<uint32_t*> last(L);
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    MCK(cudaSetDevice(a->device));
    MergeBufs& mb = g->mb[i];
    if (++a->store_epoch >= (1ull << 32)) return g->fail(a->fail(PA_ERANGE, "stack store: access clock overflow"), a->err);
    a->store_frames_sent = 0; a->store_refs_sent = 0;
    MCK(mb.v1_last.ensure(std::max<uint64_t>(U, 1) * 4));
    MCK(cudaMemsetAsync(mb.v1_last.p, 0xFF, U * 4, a->s_comp));
    k_merged_last_rows<<<a->G, kThreads, 0, a->s_comp>>>((uint32_t)a->N, a->d_slot.as<uint32_t>(), a->d_table.as<StackSlot>(), (uint32_t)a->P.row_base, mb.v1_last.as<uint32_t>());
    last[i] = mb.v1_last.as<uint32_t>();
  }
  if ((rc = t_allreduce_min(g, last, U))) return rc;
  // ---- room: the U >= C batch keeps its C stacks seen last (the store starts over), otherwise compaction when needed
  uint32_t min_last_p1 = 0;
  bool cleared = U >= C;
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    MCK(cudaSetDevice(a->device));
    if (cleared) {  // select keys in v1_foff: it is (U + 1) x 8 bytes, and the frames exchange below only starts filling it
      MergeBufs& mb = g->mb[i];
      MCK(mb.v1_foff.ensure((U + 1) * 8));
      k_merged_stamps<<<small_grid(a, U), kThreads, 0, a->s_comp>>>(a->d_ctr.as<Counters>(), last[i], mb.v1_foff.as<unsigned long long>());
      unsigned long long t = 0;
      if ((rc = select_kth_largest(a, mb.v1_foff.as<unsigned long long>(), U, C, &t)) || (rc = store_clear(a))) return g->fail(rc, a->err);
      min_last_p1 = (uint32_t)t;
      a->store_evictions++;
    } else {
      StoreCtl ctl{};
      if ((rc = store_ctl_read(a, &ctl))) return g->fail(rc, a->err);
      const uint64_t phys = a->store_slots - a->store_slots / 4;
      if (ctl.entries > ctl.live && (ctl.entries + U > phys || ctl.used_frames + a->h_ctr.n_indices64 > a->store_frames) && (rc = store_compact(a))) return g->fail(rc, a->err);
    }
  }
  if ((rc = store_frames_exchange(g, min_last_p1))) return rc;
  // ---- insert; out of slots or frame space: compaction, then a clear (which needs every stack's frames again)
  StoreCtl ctl{};
  for (int attempt = 0; attempt < 3; attempt++) {
    bool overflow = false;
    for (size_t i = 0; i < L; i++) {
      pa_agg* a = g->members[i];
      MCK(cudaSetDevice(a->device));
      MergeBufs& mb = g->mb[i];
      Counters* ctr = a->d_ctr.as<Counters>();
      MCK(cudaMemsetAsync(&ctr->store_overflow, 0, 4, a->s_comp));
      StoreInsertArgs sa = store_insert_args(a, min_last_p1);
      sa.gtab = mb.gtab.as<StackSlot>(); sa.g_slot = mb.g_uniq_slot.as<uint32_t>(); sa.g_last_inv = last[i];
      sa.g_frames = mb.v1_frames.as<uint32_t>(); sa.g_foff = mb.v1_foff.as<unsigned long long>();
      if (g->group_stacks) {
        sa.g_refs = mb.v1_frames.as<unsigned long long>(); sa.g_recs = (const uint4*)a->d_rs_recs.p; sa.n_recs = a->P.n_stacks;
        k_store_insert<true, true><<<a->G, kThreads, 0, a->s_comp>>>(sa);
      } else k_store_insert<true><<<a->G, kThreads, 0, a->s_comp>>>(sa);
      MCK(cudaMemcpyAsync(a->h_ctr_pinned, ctr, sizeof(Counters), cudaMemcpyDeviceToHost, a->s_comp));
      if ((rc = store_ctl_read(a, &ctl))) return g->fail(rc, a->err);
      MCK(cudaGetLastError());
      a->h_ctr.err |= a->h_ctr_pinned->err;
      overflow |= a->h_ctr_pinned->store_overflow != 0;
    }
    if (!overflow || attempt == 2) break;
    const bool compact = ctl.entries > ctl.live && !cleared && attempt == 0;
    for (size_t i = 0; i < L; i++) {
      pa_agg* a = g->members[i];
      MCK(cudaSetDevice(a->device));
      if (compact) { if ((rc = store_compact(a))) return g->fail(rc, a->err); }
      else { if ((rc = store_clear(a))) return g->fail(rc, a->err); a->store_evictions++; }
    }
    if (!compact) {
      cleared = true;
      if ((rc = store_frames_exchange(g, min_last_p1))) return rc;
    }
  }
  // ---- evict everything but the C entries accessed last
  if (ctl.live > C) {
    for (size_t i = 0; i < L; i++) {
      pa_agg* a = g->members[i];
      MCK(cudaSetDevice(a->device));
      unsigned long long t = 0;
      if ((rc = select_kth_largest(a, a->d_store_stamp.as<unsigned long long>(), a->store_slots + 2, C, &t))) return g->fail(rc, a->err);
      k_store_kill<<<small_grid(a, a->store_slots + 2), kThreads, 0, a->s_comp>>>(a->d_store_stamp.as<unsigned long long>(), a->store_slots + 2, t, a->d_store_ctl.as<StoreCtl>());
      MCK(cudaStreamSynchronize(a->s_comp));
      MCK(cudaGetLastError());
      a->store_evictions++;
    }
  }
  // ---- every rank must agree on the outcome: a bad frame id is seen only by the shard that packs that stack's frames
  std::vector<const void*> esrc(L);
  for (size_t i = 0; i < L; i++) esrc[i] = &g->members[i]->d_ctr.as<Counters>()->err;
  std::vector<uint8_t> hb;
  if ((rc = t_allgather_host(g, esrc, 4, hb))) return rc;
  uint32_t err_any = 0;
  for (uint32_t r = 0; r < g->world; r++) err_any |= ((const uint32_t*)hb.data())[r];
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    a->last_unique = U;
    a->h_ctr.err |= err_any;
    if ((rc = check_batch_errors(a, a->h_ctr.err))) return g->fail(rc, a->err);
  }
  return PA_OK;
}

static int merge_process(pa_merge* g) {
  const size_t L = g->members.size();
  const uint32_t W = g->world;
  g->processed = false;
  g->planned = false;
  int rc;
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    if (a->staged < 0) return g->fail(PA_EINVAL, "every member needs a staged batch (pa_agg_stage) before pa_merge_process");
    MCK(cudaSetDevice(a->device));
    a->processed = false;
    a->merged_part = true;
    if ((rc = upload_tables(a, true))) return g->fail(rc, a->err);
  }
  StreamShare share(g);
  auto restore = [] {};
  // ---- rows of every shard -> global row ranges; registrations must be identical (ids are global)
  // (group stacks: n_stack_frames is the frames of the stacks not yet freed, since dead frames make arena lengths differ)
  struct Dims { uint64_t n, nf, store_entries, store_frames, n_stack_frames, stack_digest, stages;
                uint64_t plan_digest;  // the label column plan each member predicted (upload_tables)
                uint32_t n_sample_cols, n_tail_cols, n_names, n_frames, n_cstr, n_labelsets, n_funcs, lz4, schema, group_stacks, n_stacks, group_retire; };
  std::vector<const void*> src(L);
  std::vector<uint8_t> hb;
  rc = PA_OK;
  for (size_t i = 0; i < L && !rc; i++) {
    pa_agg* a = g->members[i];
    cudaSetDevice(a->device);
    Dims d{a->N, a->NF, a->store_entries, a->store_frames, a->P.stack_frames_live, a->P.stack_digest,
           a->group_retire ? a->rs_stages : 0, a->plan_digest, a->n_label_cols - a->n_lscols, (uint32_t)a->cols.size() - a->n_label_cols, a->P.n_names,
           a->P.n_frames, a->P.n_cstr, a->P.n_labelsets, a->P.n_funcs,
           g->lz4 ? 1u : 0u, (uint32_t)a->cfg.schema, a->group_stacks ? 1u : 0u, a->P.n_stacks, a->group_retire ? 1u : 0u};
    if (g->mb[i].gather_scratch.ensure(std::max<size_t>((size_t)(W + 1) * sizeof(Dims), 256)) != cudaSuccess) { rc = g->fail(PA_ENOMEM, "device allocation failed"); break; }
    // staged through the tail of the gather scratch (the head receives the gathered block)
    uint8_t* mine = g->mb[i].gather_scratch.as<uint8_t>() + (size_t)W * sizeof(Dims);
    if (cudaMemcpyAsync(mine, &d, sizeof d, cudaMemcpyHostToDevice, a->s_comp) != cudaSuccess || cudaStreamSynchronize(a->s_comp) != cudaSuccess) { rc = g->fail(PA_EIO, "dims upload failed"); break; }
    src[i] = mine;
  }
  if (!rc) rc = t_allgather_host(g, src, sizeof(Dims), hb);
  if (rc) { restore(); return rc; }
  const Dims* dims = (const Dims*)hb.data();
  for (uint32_t r = 0; r < W; r++) {  // one member per process: the group's modes are settled here, before any work
    if (dims[r].lz4 != dims[0].lz4) { restore(); return g->fail(PA_EINVAL, kLz4Mixed); }
    if (dims[r].schema != dims[0].schema) { restore(); return g->fail(PA_EINVAL, kSchemaMixed); }
    const bool differ = dims[r].n_stacks != dims[0].n_stacks || dims[r].n_stack_frames != dims[0].n_stack_frames || dims[r].stack_digest != dims[0].stack_digest;
    const char* why = dims[r].group_stacks != dims[0].group_stacks ? kStacksMixed
                    : dims[r].group_retire != dims[0].group_retire ? kRetireMixed
                    : dims[0].group_retire && (differ || dims[r].stages != dims[0].stages) ? kRetireMismatch
                    : dims[0].group_stacks && differ ? kStacksMismatch : nullptr;
    if (why) {  // (also where the caller of each local member looks for it)
      restore();
      for (pa_agg* m : g->members) m->fail(PA_EINVAL, why);
      return g->fail(PA_EINVAL, why);
    }
    if (dims[0].schema == PA_SCHEMA_V1 && (dims[r].store_entries != dims[0].store_entries || dims[r].store_frames != dims[0].store_frames)) {
      restore();
      return g->fail(PA_EINVAL, kStoreMismatch);
    }
  }
  const bool v1 = dims[0].schema == PA_SCHEMA_V1;
  g->group_stacks = dims[0].group_stacks != 0;
  g->group_retire = dims[0].group_retire != 0;
  g->n_rows.assign(W, 0); g->nf.assign(W, 0); g->row_base.assign(W + 1, 0);
  g->NT = 0; g->NFT = 0;
  for (uint32_t r = 0; r < W; r++) {
    g->n_rows[r] = dims[r].n; g->nf[r] = dims[r].nf; g->row_base[r] = g->NT; g->NT += dims[r].n; g->NFT += dims[r].nf;
    if (dims[r].n_sample_cols != dims[0].n_sample_cols || dims[r].n_tail_cols != dims[0].n_tail_cols || dims[r].n_names != dims[0].n_names ||
        dims[r].n_frames != dims[0].n_frames || dims[r].n_cstr != dims[0].n_cstr || dims[r].n_labelsets != dims[0].n_labelsets || dims[r].n_funcs != dims[0].n_funcs) {
      restore();
      return g->fail(PA_EINVAL, "the shards of a merged batch must carry identical string / frame / labelset registrations");
    }
  }
  g->row_base[W] = g->NT;
  // group stacks: the rings hold no frames; the merged location-index stream, and each shard's slice of it, is bounded by the
  // frames of the (identical) registered stacks not yet freed, which every stack a row may name belongs to
  if (g->group_stacks) g->NFT = dims[0].n_stack_frames;
  // The label column plan must be the same on every member: the edge / run exchanges pair columns by index. Members predict it
  // from their own last batch, which differs when one of them flushed alone since the last merged batch; then all plan cold.
  bool same_plan = true;
  for (uint32_t r = 0; r < W; r++) same_plan &= dims[r].plan_digest == dims[0].plan_digest;
  for (size_t i = 0; i < L && !same_plan; i++)
    if ((rc = plan_cold(g->members[i]))) { restore(); return g->fail(rc, g->members[i]->err); }
  g->ncols = (uint32_t)g->members[0]->cols.size();
  if (g->NT > 0x7FFFFFFFull) { restore(); return g->fail(PA_ERANGE, "merged batch exceeds the int32 row limit of run ends / ListView offsets"); }
  if (g->NT == 0) {  // (like one aggregator's empty batch: no access to the store, and the label column prediction stands)
    for (size_t i = 0; i < L; i++) {
      pa_agg* a = g->members[i];
      a->plan_pending = false;
      a->processed = true; a->last_unique = 0; a->store_frames_sent = 0; a->store_refs_sent = 0;
      memset(&a->h_ctr, 0, sizeof(Counters));
    }
    restore();
    g->processed = true;
    return PA_OK;
  }
  const double t0 = now_ms();
  bool retry = false;
  for (int attempt = 0; attempt < 6; attempt++) {
    rc = merge_process_once(g, &retry);
    if (rc || !retry) break;
    for (size_t i = 0; i < L && !rc; i++) {
      pa_agg* a = g->members[i];
      if (g->retry_err & ERR_TABLE_FULL) { a->retry_cap = a->table_cap * 4; a->retry_tcap = a->tid_cap * 4; }
      if ((g->retry_err & ERR_LABEL_PLAN) && (rc = replan_labels(a))) rc = g->fail(rc, a->err);
    }
    if (rc) break;
    g->ncols = (uint32_t)g->members[0]->cols.size();
  }
  restore();
  if (rc) return rc;
  if (retry && (g->retry_err & ERR_TABLE_FULL)) return g->fail(PA_ENOMEM, "stack / thread-id table overflow");
  if (retry) return g->fail(check_batch_errors(g->members[0], g->retry_err), g->members[0]->err);  // (the label plan still missed)
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    if ((rc = check_batch_errors(a, a->h_ctr.err))) return g->fail(rc, a->err);
  }
  if (v1 && (rc = merge_store_update(g))) return rc;
  g->ms_total = now_ms() - t0;
  for (size_t i = 0; i < L; i++) { remember_sizes(g->members[i]); g->members[i]->processed = true; }
  g->processed = true;
  return PA_OK;
}

static int merge_plan_lz4(pa_merge* g);

// ---------------------------------------------------------------------------------------------------------------------
// Output. Every process builds the same plan (all inputs are replicated: merged counters, dictionary orders, run keys of the
// kind-derived columns); each member then copies ITS part of every sliced buffer to (placement + part offset) in the
// shared output, the root (rank 0) adds the replicated device buffers, the host-built buffers and the metadata.
static int merge_plan(pa_merge* g, uint64_t* ipc_len) {
  if (!g->processed) return g->fail(PA_EINVAL, "pa_merge_plan before pa_merge_process");
  const size_t L = g->members.size();
  const uint32_t W = g->world, ncols = g->ncols;
  g->planned = false;
  g->nodes.clear();
  if (g->NT == 0) { *ipc_len = 0; g->planned = true; return PA_OK; }
  pa_agg* a0 = g->members[0];
  const uint32_t nlab = a0->n_label_cols;
  int rc;
  StreamShare share(g);
  // ---- run keys of the 8 kind-derived columns from every shard (their values are host-built strings / integers), and the
  // first / last validity word of every shard's part of the nullable label columns (parts meet inside a byte)
  std::vector<uint64_t> kcount(W, 0), kdispl(W, 0);
  uint64_t ktot = 0;
  for (uint32_t r = 0; r < W; r++) {
    for (uint32_t t = 0; t < 8; t++) kcount[r] += (uint64_t)g->cols_all[(size_t)r * ncols + nlab + t].keep * 4;
    kdispl[r] = ktot; ktot += kcount[r];
  }
  std::vector<const void*> ksrc(L), vsrc(L);
  std::vector<void*> kdst(L);
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    MCK(cudaSetDevice(a->device));
    MergeBufs& mb = g->mb[i];
    const uint32_t me = g->ranks[i];
    MCK(mb.kind_all.ensure(std::max<uint64_t>(ktot + kcount[me], 256)));
    MCK(mb.vwords.ensure(std::max<size_t>((size_t)ncols * 8, 256)));
    MCK(cudaMemsetAsync(mb.vwords.p, 0, std::max<size_t>((size_t)ncols * 8, 256), a->s_comp));
    uint8_t* mine = mb.kind_all.as<uint8_t>() + ktot;  // packed behind the gathered block
    uint64_t off = 0;
    for (uint32_t t = 0; t < 8; t++) {
      const uint64_t n = (uint64_t)g->cols_all[(size_t)me * ncols + nlab + t].keep * 4;
      if (n) MCK(cudaMemcpyAsync(mine + off, a->cols[nlab + t].run_keys, n, cudaMemcpyDeviceToDevice, a->s_comp));
      off += n;
    }
    for (uint32_t c = 0; c < ncols; c++) {  // the label columns, and v1's temporality
      const MergeCol mc = g->cols_all[(size_t)me * ncols + c];
      if (!a->cols[c].validity || !mc.keep) continue;
      const uint32_t last = (mc.vshift + mc.keep - 1) >> 5;
      MCK(cudaMemcpyAsync(mb.vwords.as<uint32_t>() + 2 * c, a->cols[c].validity, 4, cudaMemcpyDeviceToDevice, a->s_comp));
      MCK(cudaMemcpyAsync(mb.vwords.as<uint32_t>() + 2 * c + 1, a->cols[c].validity + last, 4, cudaMemcpyDeviceToDevice, a->s_comp));
    }
    ksrc[i] = mine; kdst[i] = mb.kind_all.p; vsrc[i] = mb.vwords.p;
  }
  if ((rc = t_allgatherv(g, ksrc, kdst, kcount, kdispl))) return rc;
  std::vector<uint8_t> hv;
  if ((rc = t_allgather_host(g, vsrc, (size_t)std::max<uint32_t>(ncols, 1) * 8, hv))) return rc;
  g->vwords_all.assign((const uint32_t*)hv.data(), (const uint32_t*)hv.data() + (size_t)W * std::max<uint32_t>(ncols, 1) * 2);
  std::vector<uint32_t> kall(ktot / 4);
  if (ktot) { MCK(cudaSetDevice(a0->device)); MCK(cudaMemcpy(kall.data(), g->mb[0].kind_all.p, ktot, cudaMemcpyDeviceToHost)); }
  g->kind_keys.assign(8, {});
  for (uint32_t r = 0; r < W; r++) {
    uint64_t off = kdispl[r] / 4;
    for (uint32_t t = 0; t < 8; t++) {
      const uint32_t n = g->cols_all[(size_t)r * ncols + nlab + t].keep;
      g->kind_keys[t].insert(g->kind_keys[t].end(), kall.begin() + off, kall.begin() + off + n);
      off += n;
    }
  }
  // ---- nodes + layout (member 0's replicated state stands for everybody's)
  a0->hostbufs.clear();
  MCK(cudaSetDevice(a0->device));
  MergeView mv{g->NT, &g->kind_keys};
  if ((rc = collect_nodes(a0, &mv, g->nodes))) return g->fail(rc, a0->err);
  g->plan.build(g->nodes, {{"parca_write_schema_version", a0->cfg.schema == PA_SCHEMA_V1 ? "v1" : "v2"}}, (int64_t)g->NT);
  if (g->lz4 && (rc = merge_plan_lz4(g))) return rc;
  *ipc_len = g->lz4 ? g->lz.total : g->plan.total;
  g->planned = true;
  return PA_OK;
}

// Member i's validity words of label column `col` (host copy of `nwords` words; word 0 is the global word runbase / 32), with its
// border words completed by the other shards' first / last words: every byte from ceil(runbase / 8) up to
// ceil((runbase + keep) / 8) is then the merged bitmap's.
static void complete_valid_words(const pa_merge* g, size_t i, uint32_t col, uint32_t* host, uint32_t nwords) {
  const uint32_t W = g->world, ncols = g->ncols, me = g->ranks[i];
  const MergeCol mc = g->cols_all[(size_t)me * ncols + col];
  const uint64_t gw0 = mc.runbase >> 5;  // global index of my word 0
  for (uint32_t r = 0; r < W; r++) {
    if (r == me) continue;
    const MergeCol o = g->cols_all[(size_t)r * ncols + col];
    if (!o.keep) continue;
    const uint64_t ow0 = o.runbase >> 5, ow1 = ((uint64_t)o.runbase + o.keep - 1) >> 5;
    const uint32_t* ov = g->vwords_all.data() + ((size_t)r * std::max<uint32_t>(ncols, 1) + col) * 2;
    if (ow0 >= gw0 && ow0 < gw0 + nwords) host[ow0 - gw0] |= ov[0];
    if (ow1 != ow0 && ow1 >= gw0 && ow1 < gw0 + nwords) host[ow1 - gw0] |= ov[1];
  }
}

// part of a sliced buffer that member i holds: device pointer, byte offset inside the buffer, bytes
static void slice_of(const pa_merge* g, size_t i, uintptr_t tag, const void** ptr, uint64_t* at, uint64_t* len) {
  const pa_agg* a = g->members[i];
  const uint32_t kind = (uint32_t)(tag >> 16), col = (uint32_t)(tag & 0xFFFFu), me = g->ranks[i];
  const uint64_t base = g->row_base[me], n = a->N;
  *ptr = nullptr; *at = 0; *len = 0;
  switch (kind) {
    case SL_TS: *ptr = a->d_ts.p; *at = base * 8; *len = n * 8; break;
    case SL_VALUE: *ptr = a->d_value.p; *at = base * 8; *len = n * 8; break;
    case SL_UUID: *ptr = a->d_uuid.p; *at = base * 16; *len = n * 16; break;
    case SL_STOFF: *ptr = a->d_stoff.p; *at = base * 4; *len = n * 4; break;
    case SL_STSIZE: *ptr = a->d_stsize.p; *at = base * 4; *len = n * 4; break;
    case SL_STREAM: *ptr = a->d_ustream.p; *at = (uint64_t)g->mctl[i].off0 * 4; *len = (uint64_t)g->mctl[i].slice_len * 4; break;
    case SL_RUN_ENDS: case SL_RUN_KEYS: {
      const MergeCol mc = g->cols_all[(size_t)me * g->ncols + col];
      *ptr = kind == SL_RUN_ENDS ? (const void*)a->cols[col].run_ends : (const void*)a->cols[col].run_keys;
      *at = (uint64_t)mc.runbase * 4; *len = (uint64_t)mc.keep * 4;
      break;
    }
    case SL_TS_RUNS: {
      const MergeCol mc = g->cols_all[(size_t)me * g->ncols + col];
      *ptr = a->v1_ts_vals; *at = (uint64_t)mc.runbase * 8; *len = (uint64_t)mc.keep * 8;
      break;
    }
    default: break;  // SL_VALID is assembled bit-wise (below)
  }
}

// ---- PA_IPC_LZ4_FRAME_GPU groups ----------------------------------------------------------------------------------------
// The merged stream is, byte for byte, the stream one PA_IPC_LZ4_FRAME_GPU aggregator makes from the concatenated rows: every
// buffer is cut on ITS 64 KiB block grid, and a block's encoding depends on its bytes alone. Block k of a sliced buffer belongs
// to the member whose part holds the block's first byte. A block that runs past that part's end needs the heads of the
// following parts (their bytes up to the next grid boundary); every member publishes its heads in one all-gather, and each owner
// assembles its crossing blocks in its staging area. The root compresses the replicated, host-built and zero buffers alone. One
// all-gather of every member's compressed bytes per buffer then gives every rank the same layout, and with it the same ipc_len.
static int merge_plan_lz4(pa_merge* g) {
  const size_t L = g->members.size();
  const uint32_t W = g->world, ncols = g->ncols;
  const StreamPlan& plan = g->plan;
  const size_t M = plan.messages.size();
  pa_agg* a0 = g->members[0];
  int rc;
  std::vector<BatchMeta> meta;
  std::vector<uint32_t> buf0;
  if ((rc = lz4_read_messages(a0, plan, &meta, &buf0))) return g->fail(rc, a0->err);
  // ---- every rank's extent of the location-index stream (the other part extents follow from replicated state)
  std::vector<const void*> csrc(L);
  for (size_t i = 0; i < L; i++) csrc[i] = g->mb[i].ctl.as<uint32_t>() + CTL_MERGE;
  std::vector<uint8_t> hc;
  if ((rc = t_allgather_host(g, csrc, sizeof(MergeCtl), hc))) return rc;
  const MergeCtl* ctl_all = (const MergeCtl*)hc.data();
  auto extent = [&](uint32_t r, uintptr_t tag) -> std::pair<uint64_t, uint64_t> {
    const uint32_t kind = (uint32_t)(tag >> 16), col = (uint32_t)(tag & 0xFFFFu);
    const uint64_t rb = g->row_base[r], n = g->n_rows[r];
    switch (kind) {
      case SL_TS: case SL_VALUE: return {rb * 8, n * 8};
      case SL_UUID: return {rb * 16, n * 16};
      case SL_STOFF: case SL_STSIZE: return {rb * 4, n * 4};
      case SL_STREAM: return {(uint64_t)ctl_all[r].off0 * 4, (uint64_t)ctl_all[r].slice_len * 4};
      case SL_RUN_ENDS: case SL_RUN_KEYS: { const MergeCol mc = g->cols_all[(size_t)r * ncols + col]; return {(uint64_t)mc.runbase * 4, (uint64_t)mc.keep * 4}; }
      case SL_TS_RUNS: { const MergeCol mc = g->cols_all[(size_t)r * ncols + col]; return {(uint64_t)mc.runbase * 8, (uint64_t)mc.keep * 8}; }
      case SL_VALID: {
        const MergeCol mc = g->cols_all[(size_t)r * ncols + col];
        const uint64_t b0 = ((uint64_t)mc.runbase + 7) / 8, b1 = ((uint64_t)mc.runbase + mc.keep + 7) / 8;
        return {b0, b1 - b0};
      }
      default: return {0, 0};
    }
  };
  // ---- buffers, their parts, and the heads every rank publishes (rank r's heads back to back, in buffer order)
  g->lz_msg.clear(); g->lz_place.clear(); g->lz_parts.clear();
  std::vector<uint64_t> len;
  for (size_t m = 1; m < M; m++)
    for (size_t p = plan.messages[m].p0; p < plan.messages[m].p1; p++) {
      const BufRef& r = plan.placements[p].src;
      g->lz_msg.push_back((uint32_t)m); g->lz_place.push_back(p); len.push_back(r.len);
      g->lz_parts.emplace_back();
      if (!r.len || r.kind != BufRef::SLICED) continue;
      auto& parts = g->lz_parts.back();
      uint64_t pos = 0;
      for (uint32_t q = 0; q < W; q++) {
        parts.push_back(extent(q, (uintptr_t)r.ptr));
        if (!parts.back().second) continue;
        if (parts.back().first != pos) return g->fail(PA_EIO, "the shards' parts of a merged buffer do not follow each other");
        pos += parts.back().second;
      }
      if (pos != r.len) return g->fail(PA_EIO, "the shards' parts of a merged buffer do not cover it");
    }
  const size_t nbuf = len.size();
  auto head_of = [&](size_t b, uint32_t q) -> uint64_t {  // bytes of part q in front of the first grid boundary inside it
    if (g->lz_parts[b].empty()) return 0;
    const auto [at, n] = g->lz_parts[b][q];
    if (!n || at % kLz4Block == 0) return 0;
    return std::min<uint64_t>(at + n, (at / kLz4Block + 1) * kLz4Block) - at;
  };
  std::vector<std::vector<uint64_t>> head_at(nbuf, std::vector<uint64_t>(W, 0));
  std::vector<uint64_t> hcount(W, 0), hdispl(W, 0);
  uint64_t htot = 0;
  for (uint32_t q = 0; q < W; q++) {
    for (size_t b = 0; b < nbuf; b++) { head_at[b][q] = hcount[q]; hcount[q] += head_of(b, q); }
    hdispl[q] = htot;
    htot += hcount[q];
  }
  // ---- per member: validity parts completed on the host, the block table, the staging area
  struct Copy { const uint8_t* src; int64_t staged_src; uint64_t dst_staged, n; };  // staged_src >= 0: source in the staging area
  std::vector<std::vector<Copy>> pre(L), post(L);  // before the heads exchange (my heads out), after it (crossing blocks)
  g->lzs.assign(L, pa_merge::Lz4Share{});
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    MCK(cudaSetDevice(a->device));
    const uint32_t me = g->ranks[i];
    pa_merge::Lz4Share& sh = g->lzs[i];
    Lz4Table& t = sh.t;
    std::vector<const uint8_t*> psrc(nbuf, nullptr);
    std::vector<int64_t> pstaged(nbuf, -1);
    std::vector<uint64_t> hoff(nbuf, 0);
    // host sources first (they open the staging area): validity parts, and the root's host-built buffers
    for (size_t b = 0; b < nbuf; b++) {
      const BufRef& r = plan.placements[g->lz_place[b]].src;
      if (!r.len) continue;
      if (r.kind == BufRef::HOST && me == 0) hoff[b] = t.stage_host(r.ptr, r.len);
      if (r.kind != BufRef::SLICED || ((uintptr_t)r.ptr >> 16) != SL_VALID || !g->lz_parts[b][me].second) continue;
      const uint32_t col = (uint32_t)((uintptr_t)r.ptr & 0xFFFFu);
      const MergeCol mc = g->cols_all[(size_t)me * ncols + col];
      const uint32_t nw = (mc.vshift + mc.keep + 31) >> 5;
      std::vector<uint32_t> words(nw);
      MCK(cudaMemcpyAsync(words.data(), a->cols[col].validity, (size_t)nw * 4, cudaMemcpyDeviceToHost, a->s_comp));
      MCK(cudaStreamSynchronize(a->s_comp));
      complete_valid_words(g, i, col, words.data(), nw);
      const uint64_t gw0 = mc.runbase >> 5, b0 = g->lz_parts[b][me].first;
      pstaged[b] = (int64_t)t.stage_host((const uint8_t*)words.data() + (b0 - gw0 * 4), g->lz_parts[b][me].second);
    }
    const uint64_t send = sh.send = t.reserve(std::max<uint64_t>(hcount[me], 1)), recv = sh.recv = t.reserve(std::max<uint64_t>(htot, 1));
    sh.part.assign(nbuf, nullptr);
    for (size_t b = 0; b < nbuf; b++) {
      const BufRef& r = plan.placements[g->lz_place[b]].src;
      t.buffer(r.len);
      if (!r.len) continue;
      if (r.kind != BufRef::SLICED) {  // the root's alone
        if (me != 0) continue;
        if (r.kind != BufRef::DEVICE && r.kind != BufRef::HOST && r.kind != BufRef::ZEROS) return g->fail(PA_EINVAL, "buffer without a source");
        for (uint64_t o = 0; o < r.len; o += kLz4Block) {
          const uint32_t n = (uint32_t)std::min<uint64_t>(kLz4Block, r.len - o);
          if (r.kind == BufRef::HOST) t.block_staged(hoff[b] + o, n);
          else t.block(r.kind == BufRef::DEVICE ? (const uint8_t*)r.ptr + o : nullptr, n);
        }
        continue;
      }
      const auto [at, n] = g->lz_parts[b][me];
      if (!n) continue;
      if (pstaged[b] < 0) {
        const void* ptr; uint64_t at2, n2;
        slice_of(g, i, (uintptr_t)r.ptr, &ptr, &at2, &n2);
        if (at2 != at || n2 != n) return g->fail(PA_EIO, "a shard's part of a merged buffer changed between its exchange and its use");
        psrc[b] = (const uint8_t*)ptr;
      }
      if (const uint64_t h = head_of(b, me)) pre[i].push_back(Copy{psrc[b], pstaged[b], send + head_at[b][me], h});
      for (uint64_t k = (at + kLz4Block - 1) / kLz4Block; k * kLz4Block < at + n; k++) {
        const uint64_t s0 = k * kLz4Block, e = std::min<uint64_t>(s0 + kLz4Block, r.len);
        if (e <= at + n) {  // inside my part
          if (pstaged[b] >= 0) t.block_staged((uint64_t)pstaged[b] + (s0 - at), (uint32_t)(e - s0));
          else t.block(psrc[b] + (s0 - at), (uint32_t)(e - s0));
          continue;
        }
        // crossing block: my tail, then the heads of the parts that start before its end
        const uint64_t off = t.reserve(e - s0);
        t.block_staged(off, (uint32_t)(e - s0));
        post[i].push_back(Copy{pstaged[b] >= 0 ? nullptr : psrc[b] + (s0 - at), pstaged[b] >= 0 ? pstaged[b] + (int64_t)(s0 - at) : -1, off, at + n - s0});
        for (uint32_t q = me + 1; q < W; q++) {
          const auto [qat, qn] = g->lz_parts[b][q];
          if (!qn || qat >= e) continue;
          post[i].push_back(Copy{nullptr, (int64_t)(recv + hdispl[q] + head_at[b][q]), off + (qat - s0), head_of(b, q)});
        }
      }
    }
    if ((rc = lz4_alloc(a, t, &sh.d))) return g->fail(rc, a->err);
    if ((rc = lz4_upload(a, t, sh.d, a->s_comp))) return g->fail(rc, a->err);
    for (size_t b = 0; b < nbuf; b++) sh.part[b] = pstaged[b] >= 0 ? sh.d.staging + pstaged[b] : psrc[b];
    for (const Copy& c : pre[i])
      MCK(cudaMemcpyAsync(sh.d.staging + c.dst_staged, c.staged_src >= 0 ? sh.d.staging + c.staged_src : c.src, c.n, cudaMemcpyDeviceToDevice, a->s_comp));
    a->lz4_head_bytes = hcount[me];
  }
  // ---- the heads exchange
  if (htot) {
    std::vector<const void*> hs(L);
    std::vector<void*> hd(L);
    for (size_t i = 0; i < L; i++) { hs[i] = g->lzs[i].d.staging + g->lzs[i].send; hd[i] = g->lzs[i].d.staging + g->lzs[i].recv; }
    if ((rc = t_allgatherv(g, hs, hd, hcount, hdispl))) return rc;
  }
  // ---- crossing blocks, compression, and every rank's compressed bytes per buffer
  std::vector<const void*> fsrc(L);
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    MCK(cudaSetDevice(a->device));
    pa_merge::Lz4Share& sh = g->lzs[i];
    for (const Copy& c : post[i])
      MCK(cudaMemcpyAsync(sh.d.staging + c.dst_staged, c.staged_src >= 0 ? sh.d.staging + c.staged_src : c.src, c.n, cudaMemcpyDeviceToDevice, a->s_comp));
    if ((rc = lz4_compress(a, sh.d, a->s_comp))) return g->fail(rc, a->err);
    fsrc[i] = sh.d.frame;
  }
  std::vector<uint8_t> hf;
  if (nbuf && (rc = t_allgather_host(g, fsrc, nbuf * 8, hf))) return rc;
  const uint64_t* fr = (const uint64_t*)hf.data();  // [rank][buffer]: 11 + that rank's bytes of the buffer's blocks
  g->lz_frame.assign(nbuf, 11);
  for (size_t i = 0; i < L; i++) { g->lzs[i].contrib.assign(nbuf, 0); g->lzs[i].prefix.assign(nbuf, 0); }
  for (size_t b = 0; b < nbuf; b++)
    for (uint32_t q = 0; q < W; q++) {
      const uint64_t c = fr[(size_t)q * nbuf + b] - 11;
      for (size_t i = 0; i < L; i++) {
        if (g->ranks[i] == q) g->lzs[i].contrib[b] = c;
        if (g->ranks[i] > q) g->lzs[i].prefix[b] += c;
      }
      g->lz_frame[b] += c;
    }
  lz4_layout(plan, meta, buf0, len, g->lz_frame, &g->lz);
  return PA_OK;
}


// PA_IPC_LZ4_FRAME_GPU groups: every member packs its blocks and copies each share of a frame to its place in `base` (or, for a
// buffer stored raw, its part of the buffer); the root writes the metadata, length prefixes, frame headers, EndMarks, padding,
// the buffers it alone holds when they are stored raw, and the end-of-stream marker. *d2h: the longest member's copy-out.
static int merge_collect_lz4(pa_merge* g, uint8_t* base, bool root, float* d2h) {
  const size_t L = g->members.size(), nbuf = g->lz_frame.size();
  const Lz4Layout& lz = g->lz;
  const StreamPlan& plan = g->plan;
  auto buf_at = [&](size_t b) { return lz.body_of(g->lz_msg[b]) + lz.buf_at[b]; };  // its length prefix, in the stream
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    MCK(cudaSetDevice(a->device));
    cudaStream_t s = a->s_comp;
    pa_merge::Lz4Share& sh = g->lzs[i];
    const uint32_t me = g->ranks[i];
    std::vector<uint64_t> dst(nbuf, 0);
    uint64_t seg = 0;
    for (size_t b = 0; b < nbuf; b++) {
      if (lz.raw[b]) { dst[b] = 1ull << 63; continue; }
      dst[b] = seg;
      seg += sh.contrib[b];
    }
    MCK(a->d_lz4_body.ensure(std::max<uint64_t>(seg, 256)));
    if (nbuf) MCK(cudaMemcpyAsync(sh.d.dst, dst.data(), nbuf * 8, cudaMemcpyHostToDevice, s));
    MCK(cudaEventRecord(a->ev_lz4p0, s));
    if (sh.d.nb) {
      k_lz4_pack_parts<<<(unsigned)((sh.d.nb + kWarps - 1) / kWarps), kThreads, 0, s>>>(sh.d.blks, (uint32_t)sh.d.nb, sh.d.slots, sh.d.size, sh.d.off, sh.d.dst,
                                                                                       a->d_lz4_body.as<uint8_t>());
      a->tm[T_LZ4].launches++;
    }
    MCK(cudaGetLastError());
    MCK(cudaEventRecord(a->ev_lz4p1, s));
    MCK(cudaEventRecord(a->ev_d2h0, s));
    for (size_t b = 0; b < nbuf; b++) {
      const BufRef& r = plan.placements[g->lz_place[b]].src;
      if (!r.len) continue;
      if (!lz.raw[b]) {
        if (sh.contrib[b]) MCK(cudaMemcpyAsync(base + buf_at(b) + 8 + 7 + sh.prefix[b], a->d_lz4_body.as<uint8_t>() + dst[b], sh.contrib[b], cudaMemcpyDeviceToHost, s));
      } else if (r.kind == BufRef::SLICED) {
        const auto [at, n] = g->lz_parts[b][me];
        if (n) MCK(cudaMemcpyAsync(base + buf_at(b) + 8 + at, sh.part[b], n, cudaMemcpyDeviceToHost, s));
      } else if (r.kind == BufRef::DEVICE && me == 0) {
        MCK(cudaMemcpyAsync(base + buf_at(b) + 8, r.ptr, r.len, cudaMemcpyDeviceToHost, s));
      }
    }
    MCK(cudaEventRecord(a->ev_d2h1, s));
  }
  if (root) {  // overlaps the copies: none of these bytes is written by a member
    for (size_t m = 0; m < lz.metas.size(); m++) memcpy(base + lz.at[m], lz.metas[m].data(), lz.metas[m].size());
    static const uint8_t kHdr[7] = {0x04, 0x22, 0x4D, 0x18, 0x60, 0x40, 0x82};
    for (size_t b = 0; b < nbuf; b++) {
      const BufRef& r = plan.placements[g->lz_place[b]].src;
      if (!r.len) continue;
      uint8_t* o = base + buf_at(b);
      const int64_t prefix = lz.raw[b] ? -1 : (int64_t)r.len;
      memcpy(o, &prefix, 8);
      if (!lz.raw[b]) {
        memcpy(o + 8, kHdr, 7);
        memset(o + 8 + g->lz_frame[b] - 4, 0, 4);  // EndMark
      } else if (r.kind == BufRef::HOST) {
        memcpy(o + 8, r.ptr, r.len);
      } else if (r.kind == BufRef::ZEROS) {
        memset(o + 8, 0, r.len);
      }
      const uint64_t n = lz.buf_size[b];
      memset(o + n, 0, ((n + 7) & ~7ull) - n);
    }
    const uint32_t eos[2] = {0xFFFFFFFFu, 0u};
    memcpy(base + lz.total - 8, eos, 8);
  }
  int rc = msync(g);
  if (rc) return rc;
  *d2h = 0;
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    float ms = 0, pack = 0, copy = 0;
    cudaEventElapsedTime(&ms, a->tm[T_LZ4].a, a->tm[T_LZ4].b);
    cudaEventElapsedTime(&pack, a->ev_lz4p0, a->ev_lz4p1);
    cudaEventElapsedTime(&copy, a->ev_d2h0, a->ev_d2h1);
    a->tm[T_LZ4].ms = (double)ms + pack;
    *d2h = std::max(*d2h, copy);
  }
  return PA_OK;
}

template <class Done>
static int merge_result(pa_merge* g, uint8_t* base, bool root, uint64_t total, double t0, float d2h, pa_agg_result* res, Done& done) {
  const double t1 = now_ms();
  const size_t L = g->members.size();
  pa_agg* a0 = g->members[0];
  const Counters& c = a0->h_ctr;
  res->ipc = root ? base : nullptr; res->ipc_len = total; res->n_rows = g->NT; res->n_unique_stacks = c.n_unique; res->n_locations = c.n_locations;
  res->n_functions = c.n_functions; res->n_location_indices = (uint32_t)c.n_indices64;
  res->gpu_launches = 0;
  for (size_t i = 0; i < L; i++) res->gpu_launches += g->members[i]->launches;
  res->gpu_ms = a0->tm[T_TOTAL].ms; res->d2h_ms = d2h; res->host_ms = std::max(0.0, (t1 - t0) - d2h);
  float h2d = 0;
  cudaEventElapsedTime(&h2d, a0->ev_h2d0, a0->ev_h2d1);
  res->h2d_ms = h2d;
  done();
  return PA_OK;
}

static int merge_collect(pa_merge* g, uint8_t* base, uint64_t cap, pa_agg_result* res) {
  memset(res, 0, sizeof *res);
  if (!g->planned) return g->fail(PA_EINVAL, "pa_merge_collect before pa_merge_plan");
  const size_t L = g->members.size();
  const uint32_t W = g->world, ncols = g->ncols;
  auto done = [&] { for (size_t i = 0; i < L; i++) { release_staged(g->members[i]); g->members[i]->merged_part = false; } g->planned = false; g->processed = false; };
  if (g->NT == 0) { done(); return PA_OK; }
  const double t0 = now_ms();
  const uint64_t total = g->lz4 ? g->lz.total : g->plan.total;
  StreamShare share(g);
  bool root = false;
  for (size_t i = 0; i < L; i++) root |= g->ranks[i] == 0;
  if (!base) {
    if (L != W) return g->fail(PA_EINVAL, "members in several processes need a caller-provided output buffer shared by all of them");
    if (total > g->out_cap) {
      if (g->out) cudaFreeHost(g->out);
      g->out = nullptr; g->out_cap = 0;
      const uint64_t want = total + total / 4 + 4096;
      if (cudaHostAlloc((void**)&g->out, want, cudaHostAllocPortable) != cudaSuccess) return g->fail(PA_ENOMEM, "pinned output allocation failed");
      g->out_cap = want;
    }
    base = g->out;
  } else {
    if (cap < total) return g->fail(PA_ENOSPC, "output buffer smaller than the planned stream");
    if (g->registered != base || g->registered_len < total) {  // page-lock the caller's (shared) buffer once so the copies run at link speed
      if (g->registered) cudaHostUnregister(g->registered);
      g->registered = nullptr;
      if (cudaHostRegister(base, cap, cudaHostRegisterPortable) == cudaSuccess) { g->registered = base; g->registered_len = cap; }
      else cudaGetLastError();  // not fatal: pageable copies are slower but correct
    }
  }
  float d2h = 0;
  if (g->lz4) {
    if (int rc = merge_collect_lz4(g, base, root, &d2h)) return rc;
    return merge_result(g, base, root, total, t0, d2h, res, done);
  }
  // ---- device -> host: every member its parts; the root also the replicated buffers
  struct BitJob { size_t member; uint32_t col; uint64_t at; uint32_t* host; uint32_t nwords; };
  std::vector<BitJob> bits;
  size_t vbytes = 0;
  for (auto& p : g->plan.placements)
    if (p.src.kind == BufRef::SLICED && ((uintptr_t)p.src.ptr >> 16) == SL_VALID)
      for (size_t i = 0; i < L; i++) {
        const uint32_t col = (uint32_t)((uintptr_t)p.src.ptr & 0xFFFFu);
        const MergeCol mc = g->cols_all[(size_t)g->ranks[i] * ncols + col];
        if (!mc.keep) continue;
        const uint32_t nw = ((mc.vshift + mc.keep + 31) >> 5);
        bits.push_back(BitJob{i, col, p.at, nullptr, nw});
        vbytes += (size_t)nw * 4;
      }
  int rc = pin_room(g, std::max<size_t>(vbytes, 64));
  if (rc) return rc;
  {
    size_t off = 0;
    for (auto& b : bits) { b.host = (uint32_t*)(g->h_pin + off); off += (size_t)b.nwords * 4; }
  }
  std::vector<cudaEvent_t> ev0(L), ev1(L);
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    MCK(cudaSetDevice(a->device));
    cudaStream_t s = a->s_comp;
    MCK(cudaEventRecord(a->ev_d2h0, s));
    for (auto& p : g->plan.placements) {
      if (!p.src.len) continue;
      if (p.src.kind == BufRef::SLICED) {
        const void* ptr; uint64_t at, len;
        slice_of(g, i, (uintptr_t)p.src.ptr, &ptr, &at, &len);
        if (len) MCK(cudaMemcpyAsync(base + p.at + at, ptr, len, cudaMemcpyDeviceToHost, s));
      } else if (p.src.kind == BufRef::DEVICE && g->ranks[i] == 0) {
        MCK(cudaMemcpyAsync(base + p.at, p.src.ptr, p.src.len, cudaMemcpyDeviceToHost, s));
      }
    }
    for (auto& b : bits) if (b.member == i) MCK(cudaMemcpyAsync(b.host, a->cols[b.col].validity, (size_t)b.nwords * 4, cudaMemcpyDeviceToHost, s));
    MCK(cudaEventRecord(a->ev_d2h1, s));
  }
  if (root) g->plan.write_host_parts(base);  // metadata, host-built buffers, zero fills and padding overlap the copies
  if ((rc = msync(g))) return rc;
  // ---- validity bitmaps of the label runs: a shard's part starts at bit `runbase`; border words are completed with the
  // neighbours' border words, then every byte is written by the lowest rank that owns a bit of it
  for (auto& b : bits) {
    const uint32_t me = g->ranks[b.member];
    const MergeCol mc = g->cols_all[(size_t)me * ncols + b.col];
    const uint64_t gw0 = mc.runbase >> 5;  // global index of my word 0
    complete_valid_words(g, b.member, b.col, b.host, b.nwords);
    const uint64_t b0 = ((uint64_t)mc.runbase + 7) / 8, b1 = ((uint64_t)mc.runbase + mc.keep + 7) / 8;
    if (b1 > b0) memcpy(base + b.at + b0, (const uint8_t*)b.host + (b0 - gw0 * 4), b1 - b0);
  }
  for (size_t i = 0; i < L; i++) { float ms = 0; cudaEventElapsedTime(&ms, g->members[i]->ev_d2h0, g->members[i]->ev_d2h1); d2h = std::max(d2h, ms); }
  return merge_result(g, base, root, total, t0, d2h, res, done);
}

// v1 groups: the stacktrace record for rank 0's request, built by every member from its copy of the store (the request's Gets
// refresh every copy alike). Groups with one member per process first carry the request to every rank: its length in a small
// all-gather, then rank 0's ids in an all-gather-v.
static int merge_stacktraces(pa_merge* g, const uint8_t* ids, uint64_t n, pa_agg_result* res) {
  memset(res, 0, sizeof *res);
  const size_t L = g->members.size();
  const uint32_t W = g->world;
  if (g->members[0]->cfg.schema != PA_SCHEMA_V1) return g->fail(PA_EINVAL, "pa_merge_stacktraces needs a group of PA_SCHEMA_V1 members");
  if (g->processed || g->planned) return g->fail(PA_EINVAL, "collect the merged batch before asking for stacktraces");
  std::vector<uint8_t> req;
  const uint8_t* use = ids;
  if (L != W) {
    const bool root = g->ranks[0] == 0;
    const uint64_t kBad = ~0ull;  // rank 0's request is malformed: every rank fails, none waits for ids that never come
    const uint64_t mine = !root ? 0 : (n && !ids) || n > 0x7FFFFFFFull / 16 ? kBad : n;
    pa_agg* a = g->members[0];
    MCK(cudaSetDevice(a->device));
    MergeBufs& mb = g->mb[0];
    MCK(mb.gather_scratch.ensure(std::max<size_t>((size_t)(W + 1) * 8, 256)));
    uint8_t* slot = mb.gather_scratch.as<uint8_t>() + (size_t)W * 8;  // staged behind the gathered block
    MCK(cudaMemcpyAsync(slot, &mine, 8, cudaMemcpyHostToDevice, a->s_comp));
    MCK(cudaStreamSynchronize(a->s_comp));
    std::vector<uint8_t> hn;
    int rc = t_allgather_host(g, {slot}, 8, hn);
    if (rc) return rc;
    uint64_t n0;
    memcpy(&n0, hn.data(), 8);  // rank 0's
    if (n0 == kBad) return g->fail(PA_EINVAL, "rank 0's stacktrace request is malformed (null ids or more than int32 offsets allow)");
    n = n0;
    req.resize(n * 16);
    if (n) {
      MCK(mb.v1_ids_req.ensure(n * 16));
      if (root) MCK(cudaMemcpyAsync(mb.v1_ids_req.p, ids, n * 16, cudaMemcpyHostToDevice, a->s_comp));
      std::vector<uint64_t> count(W, 0), displ(W, 0);
      count[0] = n * 16;
      if ((rc = t_allgatherv(g, {mb.v1_ids_req.p}, {mb.v1_ids_req.p}, count, displ))) return rc;
      MCK(cudaMemcpyAsync(req.data(), mb.v1_ids_req.p, n * 16, cudaMemcpyDeviceToHost, a->s_comp));
      MCK(cudaStreamSynchronize(a->s_comp));
    }
    use = req.data();
  }
  for (size_t i = 0; i < L; i++) {
    pa_agg_result mine{};
    pa_agg* a = g->members[i];
    if (int rc = stacktraces(a, use, n, i == 0 ? res : &mine)) return g->fail(rc, a->err);
  }
  return PA_OK;
}

}  // namespace pa


// ---------------------------------------------------------------------------------------------------------------------
extern "C" {

// registered-stacks members join merge groups only with group-wide stack ids (the reason goes into the member's last error)
static bool refuse_registered(pa_agg* m) {
  if (!m->registered || m->group_stacks) return false;
  m->fail(PA_EINVAL, "merge groups do not support PA_CFG_REGISTERED_STACKS members yet");
  return true;
}

int pa_merge_create_local(pa_agg* const* members, uint32_t n, pa_merge** out) {
  if (!members || !n || !out || n > (uint32_t)kMaxWorld) return PA_EINVAL;
  uint32_t n_lz4 = 0;
  for (uint32_t i = 0; i < n; i++) {
    if (!members[i] || members[i]->device != members[0]->device) return PA_EINVAL;
    n_lz4 += lz4_gpu_member(members[i]);
  }
  bool any_registered = false;
  uint32_t n_stacks = 0;
  for (uint32_t i = 0; i < n; i++) { any_registered |= refuse_registered(members[i]); n_stacks += group_stacks_member(members[i]); }
  if (n_stacks && n_stacks != n) {  // (the reason goes into every member's last error; a plain registered member keeps its own)
    for (uint32_t i = 0; i < n; i++) if (!members[i]->registered || members[i]->group_stacks) members[i]->fail(PA_EINVAL, kStacksMixed);
    return PA_EINVAL;
  }
  if (any_registered) return PA_EINVAL;
  uint32_t n_retire = 0;
  for (uint32_t i = 0; i < n; i++) n_retire += members[i]->group_retire;
  if (n_retire && n_retire != n) {
    for (uint32_t i = 0; i < n; i++) members[i]->fail(PA_EINVAL, kRetireMixed);
    return PA_EINVAL;
  }
  if (n_lz4 && n_lz4 != n) {  // the reason goes where the caller of a PA_IPC_LZ4_FRAME_GPU member looks for it
    for (uint32_t i = 0; i < n; i++) if (lz4_gpu_member(members[i])) members[i]->fail(PA_EINVAL, kLz4Mixed);
    return PA_EINVAL;
  }
  for (uint32_t i = 1; i < n; i++) {  // (the reason goes into every member's last error)
    const pa_agg *a = members[i], *b = members[0];
    const char* why = a->cfg.schema != b->cfg.schema ? kSchemaMixed
                    : (b->cfg.schema == PA_SCHEMA_V1 && (a->store_entries != b->store_entries || a->store_frames != b->store_frames)) ? kStoreMismatch : nullptr;
    if (why) {
      for (uint32_t j = 0; j < n; j++) members[j]->fail(PA_EINVAL, why);
      return PA_EINVAL;
    }
  }
  pa_merge* g = new pa_merge();
  g->world = n;
  g->lz4 = n_lz4 == n;
  for (uint32_t i = 0; i < n; i++) { g->members.push_back(members[i]); g->ranks.push_back(i); }
  g->mb.resize(n);
  *out = g;
  return PA_OK;
}
int pa_merge_nccl_unique_id(uint8_t* id128) {
  if (!id128) return PA_EINVAL;
  NcclApi* n = nccl_api();
  if (!n) return PA_EIO;
  ncclUniqueId id;
  if (n->GetUniqueId(&id) != ncclSuccess) return PA_EIO;
  static_assert(sizeof(ncclUniqueId) == 128, "ncclUniqueId is 128 bytes");
  memcpy(id128, &id, 128);
  return PA_OK;
}
int pa_merge_create_nccl(pa_agg* member, const uint8_t* id128, uint32_t rank, uint32_t world, pa_merge** out) {
  if (member && refuse_registered(member)) return PA_EINVAL;
  if (!member || !id128 || !out || world == 0 || world > (uint32_t)kMaxWorld || rank >= world) return PA_EINVAL;
  NcclApi* n = nccl_api();
  if (!n) return PA_EIO;
  if (cudaSetDevice(member->device) != cudaSuccess) return PA_ENODEV;
  ncclUniqueId id;
  memcpy(&id, id128, 128);
  ncclComm_t comm;
  if (n->CommInitRank(&comm, (int)world, id, (int)rank) != ncclSuccess) return PA_EIO;
  pa_merge* g = new pa_merge();
  g->world = world;
  g->use_nccl = true;
  g->lz4 = lz4_gpu_member(member);
  g->members.push_back(member);
  g->ranks.push_back(rank);
  g->comms.push_back(comm);
  g->mb.resize(1);
  *out = g;
  return PA_OK;
}
int pa_merge_create_host(pa_agg* member, const pa_merge_host_transport* t, uint32_t rank, uint32_t world, pa_merge** out) {
  if (member && refuse_registered(member)) return PA_EINVAL;
  if (!member || !t || !out || world == 0 || world > (uint32_t)kMaxWorld || rank >= world || !t->allgather || !t->allgatherv || !t->alltoallv || !t->allreduce_min_u32)
    return PA_EINVAL;
  pa_merge* g = new pa_merge();
  g->world = world;
  g->use_nccl = true;  // one stream per member; ordering comes from the (synchronous) collectives
  g->host_copy = *t;
  g->host = &g->host_copy;
  g->lz4 = lz4_gpu_member(member);
  g->members.push_back(member);
  g->ranks.push_back(rank);
  g->mb.resize(1);
  *out = g;
  return PA_OK;
}
int pa_merge_create_shm(pa_agg* member, const char* name, uint32_t rank, uint32_t world, uint64_t mailbox_bytes, pa_merge** out) {
  if (member && refuse_registered(member)) return PA_EINVAL;
  if (!member || !name || name[0] != '/' || !out || world == 0 || world > (uint32_t)kMaxWorld || rank >= world) return PA_EINVAL;
  if (mailbox_bytes == 0) mailbox_bytes = 64ull << 20;
  mailbox_bytes = (mailbox_bytes + 4095) & ~4095ull;
  const size_t len = kShmHeaderBytes + (size_t)world * mailbox_bytes;
  int fd = -1;
  if (rank == 0) {
    shm_unlink(name);  // a stale segment of a previous run
    fd = shm_open(name, O_CREAT | O_EXCL | O_RDWR, 0600);
    if (fd < 0 || ftruncate(fd, (off_t)len) != 0) { if (fd >= 0) close(fd); return PA_EIO; }
  } else {
    const double t0 = now_ms();
    for (;;) {  // wait for rank 0 to create and size it
      fd = shm_open(name, O_RDWR, 0600);
      struct stat st;
      if (fd >= 0 && fstat(fd, &st) == 0 && (size_t)st.st_size >= len) break;
      if (fd >= 0) { close(fd); fd = -1; }
      if (now_ms() - t0 > 120000.0) return PA_EIO;
      sched_yield();
    }
  }
  void* base = mmap(nullptr, len, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
  close(fd);
  if (base == MAP_FAILED) return PA_ENOMEM;
  ShmHeader* h = reinterpret_cast<ShmHeader*>(base);
  if (rank == 0) {
    memset(base, 0, kShmHeaderBytes);
    h->world = world;
    h->mailbox_bytes = mailbox_bytes;
    h->ready.store(1, std::memory_order_release);
  } else {
    const double t0 = now_ms();
    while (h->ready.load(std::memory_order_acquire) != 1) { if (now_ms() - t0 > 120000.0) { munmap(base, len); return PA_EIO; } sched_yield(); }
    if (h->world != world || h->mailbox_bytes != mailbox_bytes) { munmap(base, len); return PA_EINVAL; }
  }
  pa_merge* g = new pa_merge();
  g->world = world;
  g->use_nccl = true;  // one stream per member; the (synchronous) collectives order the ranks
  g->shm = (uint8_t*)base;
  g->shm_len = len;
  g->shm_name = name;
  g->shm_owner = rank == 0;
  g->lz4 = lz4_gpu_member(member);
  cudaSetDevice(member->device);
  if (cudaHostRegister(base, len, cudaHostRegisterPortable) == cudaSuccess) g->shm_registered = true;  // DMA straight into / out of the mailboxes
  else cudaGetLastError();
  g->members.push_back(member);
  g->ranks.push_back(rank);
  g->mb.resize(1);
  *out = g;
  return PA_OK;
}
void pa_merge_destroy(pa_merge* g) {
  if (!g) return;
  for (size_t i = 0; i < g->members.size(); i++) {
    cudaSetDevice(g->members[i]->device);
    cudaStreamSynchronize(g->members[i]->s_comp);
    g->mb[i].release();
  }
  if (g->use_nccl && !g->host && !g->shm) for (auto c : g->comms) nccl_api()->CommDestroy(c);
  if (g->shm) {
    if (g->shm_registered) cudaHostUnregister(g->shm);
    g->shm_scratch.release();
    munmap(g->shm, g->shm_len);
    if (g->shm_owner) shm_unlink(g->shm_name.c_str());
  }
  if (g->h_xs) cudaFreeHost(g->h_xs);
  if (g->h_xr) cudaFreeHost(g->h_xr);
  if (g->registered) cudaHostUnregister(g->registered);
  if (g->out) cudaFreeHost(g->out);
  if (g->h_pin) cudaFreeHost(g->h_pin);
  delete g;
}
const char* pa_merge_last_error(const pa_merge* g) { return g ? g->err.c_str() : "null handle"; }

// PA_CFG_GROUP_RETIRE: pa_agg_retire_stacks for the whole group. The arguments and each member's state go round first, so that a
// refusal is taken on every rank before any other collective. Then each slot's last_use becomes the group's maximum (inverted
// around an all-reduce(min): a slot the emit marked 0xFFFFFFFF inverts to 0 and stays marked), and every member runs the single
// aggregator's selection and bookkeeping on identical inputs, so every member retires the same slots.
static const char kRetireRefused[] = "pa_merge_retire_stacks needs, on every rank, PA_CFG_GROUP_RETIRE members whose staged batch is collected, "
                                     "idle_batches >= 1, and the same idle_batches, cap, stage count and uploaded slot count";
static int merge_retire_stacks(pa_merge* g, uint32_t idle, uint64_t* handles, uint64_t cap, uint64_t* n_retired) {
  const size_t L = g->members.size();
  const uint32_t W = g->world;
  if (n_retired) *n_retired = 0;
  StreamShare share(g);
  struct RetireDims { uint64_t cap, stages, slots; uint32_t idle, ok; };
  std::vector<const void*> src(L);
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    MCK(cudaSetDevice(a->device));
    const RetireDims d{cap, a->rs_stages, a->rs_dev_slots, idle, a->group_retire && a->staged < 0 && idle > 0 && (handles || !cap) ? 1u : 0u};
    MCK(g->mb[i].gather_scratch.ensure(std::max<size_t>((size_t)(W + 1) * sizeof(RetireDims), 256)));
    uint8_t* mine = g->mb[i].gather_scratch.as<uint8_t>() + (size_t)W * sizeof(RetireDims);  // (behind the gathered block, as in merge_process)
    MCK(cudaMemcpyAsync(mine, &d, sizeof d, cudaMemcpyHostToDevice, a->s_comp));
    MCK(cudaStreamSynchronize(a->s_comp));
    src[i] = mine;
  }
  std::vector<uint8_t> hb;
  int rc = t_allgather_host(g, src, sizeof(RetireDims), hb);
  if (rc) return rc;
  const RetireDims* d = (const RetireDims*)hb.data();
  for (uint32_t r = 0; r < W; r++)
    if (!d[r].ok || d[r].idle != d[0].idle || d[r].cap != d[0].cap || d[r].stages != d[0].stages || d[r].slots != d[0].slots) {
      for (pa_agg* m : g->members) m->fail(PA_EINVAL, kRetireRefused);
      return g->fail(PA_EINVAL, kRetireRefused);
    }
  const uint64_t ns = d[0].slots;
  if (d[0].stages >= idle && ns && cap) {  // (otherwise retire_stacks selects nothing, on every rank alike)
    std::vector<uint32_t*> last(L);
    for (size_t i = 0; i < L; i++) {
      pa_agg* a = g->members[i];
      MCK(cudaSetDevice(a->device));
      last[i] = a->d_rs_last.as<uint32_t>();
      k_invert_u32<<<small_grid(a, ns), kThreads, 0, a->s_comp>>>(last[i], ns);
    }
    rc = t_allreduce_min(g, last, ns);
    // inverted back on a failed reduction too: every word then holds a batch number this member or another one recorded, so no
    // slot reads as idle longer than it is
    for (size_t i = 0; i < L; i++) {
      pa_agg* a = g->members[i];
      MCK(cudaSetDevice(a->device));
      k_invert_u32<<<small_grid(a, ns), kThreads, 0, a->s_comp>>>(last[i], ns);
    }
    if (rc) return rc;
  }
  std::vector<uint64_t> other(cap ? std::min<uint64_t>(cap, ns) : 0);
  uint64_t n0 = 0;
  for (size_t i = 0; i < L; i++) {
    pa_agg* a = g->members[i];
    uint64_t* h = i == 0 ? handles : other.data();
    uint64_t n = 0;
    if ((rc = retire_stacks(a, idle, h, cap, &n))) return g->fail(rc, a->err);
    if (i == 0) n0 = n;
    else if (n != n0 || !std::equal(h, h + n, handles)) return g->fail(PA_EIO, "the members of a PA_CFG_GROUP_RETIRE group selected different stacks to retire");
    std::lock_guard<std::mutex> lk(a->reg_mu);  // every retirement is digested too (idle_batches, then the handles), apart from registrations
    std::vector<uint64_t> wide(1 + n);
    wide[0] = idle;
    std::copy(h, h + n, wide.begin() + 1);
    a->retire_digest = pa_xxh64(wide.data(), wide.size() * 8, a->retire_digest);
  }
  if (n_retired) *n_retired = n0;
  return PA_OK;
}

namespace {
struct MergeLocks {  // the members' flush locks, taken in member order
  std::vector<std::unique_lock<std::mutex>> l;
  explicit MergeLocks(pa_merge* g) { for (pa_agg* a : g->members) l.emplace_back(a->flush_mu); }
};
}  // namespace

int pa_merge_process(pa_merge* g) {
  if (!g) return PA_EINVAL;
  MergeLocks lk(g);
  return merge_process(g);
}
int pa_merge_plan(pa_merge* g, uint64_t* ipc_len) {
  if (!g || !ipc_len) return PA_EINVAL;
  MergeLocks lk(g);
  return merge_plan(g, ipc_len);
}
int pa_merge_collect(pa_merge* g, uint8_t* base, uint64_t cap, pa_agg_result* out) {
  if (!g || !out) return PA_EINVAL;
  MergeLocks lk(g);
  return merge_collect(g, base, cap, out);
}
/* swap + H2D of every member's ring, the merged pass, plan and collect in one call (groups whose members all live in this
 * process: the output buffer is library-owned; other groups pass a shared buffer through pa_merge_collect) */
int pa_merge_flush(pa_merge* g, pa_agg_result* out) {
  if (!g || !out) return PA_EINVAL;
  MergeLocks lk(g);
  int rc;
  for (pa_agg* a : g->members) if ((rc = stage_async(a))) return g->fail(rc, a->err);
  auto drop = [&] { for (pa_agg* a : g->members) { cudaSetDevice(a->device); cudaStreamSynchronize(a->s_copy); release_staged(a); a->merged_part = false; } };
  if ((rc = merge_process(g))) { drop(); return rc; }
  uint64_t len = 0;
  if ((rc = merge_plan(g, &len))) { drop(); return rc; }
  if ((rc = merge_collect(g, nullptr, 0, out))) drop();
  return rc;
}
int pa_merge_retire_stacks(pa_merge* g, uint32_t idle_batches, uint64_t* handles, uint64_t cap, uint64_t* n_retired) {
  if (!g) return PA_EINVAL;
  MergeLocks lk(g);
  return merge_retire_stacks(g, idle_batches, handles, cap, n_retired);
}
int pa_merge_stacktraces(pa_merge* g, const uint8_t* ids, uint64_t n_ids, pa_agg_result* out) {
  if (!g || !out) return PA_EINVAL;
  MergeLocks lk(g);
  return merge_stacktraces(g, ids, n_ids, out);
}
int pa_merge_last_stats(const pa_merge* g, double* wall_ms, double* exchange_wait_ms, uint64_t* nvlink_bytes, uint64_t* n_rows_total) {
  if (!g) return PA_EINVAL;
  if (wall_ms) *wall_ms = g->ms_total;
  if (exchange_wait_ms) *exchange_wait_ms = g->ms_exchange_wait;
  if (nvlink_bytes) *nvlink_bytes = g->nvlink_bytes;
  if (n_rows_total) *n_rows_total = g->NT;
  return PA_OK;
}

}  // extern "C"
