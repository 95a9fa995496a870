// kernels.cuh — sm_90a (H100) device code for the sample → Arrow aggregation path.
//
// Every kernel here is HBM-/L2-bound integer work (no tensor cores by design). Conventions:
//   * generic passes use a fixed grid (kGrid blocks x kThreads) and take their element count
//     from device memory, so the host never synchronises between dependent passes;
//   * "first-occurrence rank" (the invariant behind every dictionary index of the reference:
//     reporter/parca_reporter.go:425, reporter/arrow_v2.go:191,:302) is computed as
//     atomicMin(first position) -> flag -> exclusive scan, never by insertion order.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace pa {

constexpr uint32_t kNull = 0xFFFFFFFFu;
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxCols = 256;  // label columns + 8 constant-ish REE columns (+2 in v1); kernel-parameter tables are sized by it
constexpr int kMaxWorld = 64;   // shards of one merged batch (mode B)

enum : uint32_t {
  ERR_TABLE_FULL = 1u, ERR_BAD_FRAME_ID = 2u, ERR_BAD_STRING_ID = 4u, ERR_BAD_LABELSET = 8u,
  ERR_BAD_KIND = 16u, ERR_INDEX_OVERFLOW = 32u, ERR_BAD_CPU = 64u, ERR_BAD_FRAME_RANGE = 128u,
  ERR_SLICE_CAP = 256u,   // mode B: this shard's slice of the location-index stream exceeds its buffer
  ERR_MERGE_LOOKUP = 512u,  // mode B: a local stack is missing from the merged dictionary (internal error)
  ERR_BAD_STACK_ID = 1024u, // registered stacks: a row names a stack id that was not registered when the batch was processed
  ERR_LABEL_PLAN = 2048u,   // a labelset the batch names carries a label name the column plan left out: the pass is redone
};

struct __align__(16) Key128 { unsigned long long hi, lo; };

// PA_CFG_REGISTERED_STACKS: one registered stack, 32 B (one L2 sector). `off` indexes the registered frame arena, which holds
// the ids at the ring's width, so every kernel that reads frames through (frames, frame_off, narrow) reads the arena unchanged.
struct __align__(32) RegStack {
  unsigned long long hash_hi, hash_lo;  // the stack id, as pa_sample_hdr carries it
  unsigned long long off;
  uint32_t depth, pad;  // PA_CFG_RETIRE_STACKS: pad = the slot's generation, with kStackFree set while the slot is free
};
constexpr uint32_t kStackFree = 0x80000000u;

// open-address stack table entry: 32 B = one L2 sector
struct __align__(32) StackSlot {
  Key128 key;          // (0,0) = empty; claimed once by a 128-bit CAS, never changes afterwards
  uint32_t first_inv;  // 0xFFFFFFFF - first row, maintained with atomicMax (memset-0 = none yet)
  uint32_t ordinal;    // first-occurrence ordinal of this stack (set by k_stack_assign)
  uint32_t offset;     // start of this stack's run in the location-index stream
  uint32_t size;       // nframes of the first occurrence (listEntryRef.listSize)
};

// device-resident counters, copied to the host once per flush
struct Counters {
  uint32_t err;
  uint32_t n_unique;
  unsigned long long n_indices64;
  uint32_t n_locations, n_lines, n_functions;
  uint32_t n_dict_type, n_dict_map, n_dict_bid, n_dict_file;
  uint32_t null_bid, null_file;
  uint32_t n_claimed;       // stack-table slots claimed so far == entries of the claimed-slot list
  uint32_t zero_claimed;    // the dedicated all-zero-id slot is on the list
  uint32_t store_overflow;  // v1: the known-stacks store ran out of entries or frame space during this flush
  uint32_t st_null_lists;   // v1 stacktrace record: known stacks with zero frames (null list entries)
  uint32_t n_runs[kMaxCols];
  uint32_t n_dict[kMaxCols];
  uint32_t n_null[kMaxCols];
  uint32_t last_nonnull_plus1[kMaxCols];
};

// ---------------------------------------------------------------------------------------------
// small helpers
// two funnel shifts (SHF) for any constant rotation; the generic (x << r) | (x >> (64 - r)) form compiled to four
// instructions for r = 31 (shift, shift-as-IMAD, shift, LOP3), which is the rotation of every XXH64 round
__device__ __forceinline__ unsigned long long rotl64(unsigned long long x, int r) {
  uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
  if (r & 32) { const uint32_t t = lo; lo = hi; hi = t; }
  const uint32_t nhi = __funnelshift_l(lo, hi, r & 31), nlo = __funnelshift_l(hi, lo, r & 31);
  return ((unsigned long long)nhi << 32) | nlo;
}
__device__ __forceinline__ unsigned long long bswap64(unsigned long long x) {
  uint32_t lo = (uint32_t)x, hi = (uint32_t)(x >> 32);
  return ((unsigned long long)__byte_perm(lo, 0, 0x0123) << 32) | __byte_perm(hi, 0, 0x0123);
}
__device__ __forceinline__ unsigned long long ldg_stream64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.global.nc.L1::no_allocate.u64 %0, [%1];" : "=l"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ Key128 ld_key(const Key128* p) {
  Key128 k;
  asm volatile("ld.volatile.global.v2.u64 {%0, %1}, [%2];" : "=l"(k.hi), "=l"(k.lo) : "l"(p));
  return k;
}
__device__ __forceinline__ Key128 cas128(Key128* addr, Key128 cmp, Key128 val) {
  Key128 old;
  asm volatile(
      "{\n .reg .b128 c, v, o;\n mov.b128 c, {%2, %3};\n mov.b128 v, {%4, %5};\n"
      " atom.global.cas.b128 o, [%6], c, v;\n mov.b128 {%0, %1}, o;\n}"
      : "=l"(old.hi), "=l"(old.lo)
      : "l"(cmp.hi), "l"(cmp.lo), "l"(val.hi), "l"(val.lo), "l"(addr)
      : "memory");
  return old;
}
__device__ __forceinline__ bool key_eq(Key128 a, Key128 b) { return a.hi == b.hi && a.lo == b.lo; }
__device__ __forceinline__ bool key_zero(Key128 a) { return (a.hi | a.lo) == 0; }
__device__ __forceinline__ uint32_t mix_slot(Key128 k) {
  unsigned long long x = k.lo ^ (k.hi * 0x9E3779B97F4A7C15ull);
  x ^= x >> 32; x *= 0xD6E8FEB86659FD93ull; x ^= x >> 32;
  return (uint32_t)x;
}
__device__ __forceinline__ uint32_t mix32(uint32_t x) {
  x ^= x >> 16; x *= 0x7FEB352Du; x ^= x >> 15; x *= 0x846CA68Bu; x ^= x >> 16;
  return x;
}

// shared-memory mbarriers and bulk (TMA) global -> shared copies: the header pass and the TMA hash kernels stage their
// inputs with them
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n .reg .pred P1;\n LAB_WAIT:\n mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n @P1 bra DONE;\n bra LAB_WAIT;\n DONE:\n}"
      ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src), "r"(bytes), "r"(bar) : "memory");
}

// contiguous per-block range of [0,n), multiple of kThreads so tiles stay aligned
__device__ __forceinline__ void block_range(uint32_t n, uint32_t* begin, uint32_t* end) {
  uint32_t per = (n + gridDim.x - 1) / gridDim.x;
  per = (per + kThreads - 1) / kThreads * kThreads;
  unsigned long long b = (unsigned long long)blockIdx.x * per;
  *begin = b < n ? (uint32_t)b : n;
  unsigned long long e = b + per;
  *end = e < n ? (uint32_t)e : n;
}

// ---------------------------------------------------------------------------------------------
// stack table: find-or-claim on the 128-bit stack id (StacktraceDictBuilderV2.index, arrow_v2.go:230)
// Every slot is appended to `claimed` by the one thread whose CAS claimed it, so the ranking passes walk the
// unique stacks (U entries) instead of scanning the whole table.
// control words of one open-address stack table (the per-batch table lives in Counters; the mode-B owner / merged
// tables carry their own)
struct TabCtl { uint32_t* n_claimed; uint32_t* zero_claimed; uint32_t* err; };
__device__ __forceinline__ TabCtl ctl_of(Counters* c) { return TabCtl{&c->n_claimed, &c->zero_claimed, &c->err}; }
__device__ __forceinline__ uint32_t stack_find_or_insert(StackSlot* tab, uint32_t mask, Key128 k, TabCtl ctr, uint32_t* claimed) {
  if (key_zero(k)) {  // the all-zero id lives in a dedicated slot past the table
    if (*(volatile uint32_t*)ctr.zero_claimed == 0u && atomicExch(ctr.zero_claimed, 1u) == 0u) claimed[atomicAdd(ctr.n_claimed, 1u)] = mask + 1;
    return mask + 1;
  }
  uint32_t idx = mix_slot(k) & mask;
  const Key128 zero{0ull, 0ull};
  for (uint32_t probe = 0; probe <= mask; probe++) {
    Key128 cur = ld_key(&tab[idx].key);
    if (cur.hi == 0 || cur.lo == 0) cur = cas128(&tab[idx].key, zero, k);  // empty / possibly torn: CAS is authoritative
    if (key_zero(cur)) { claimed[atomicAdd(ctr.n_claimed, 1u)] = idx; return idx; }
    if (key_eq(cur, k)) return idx;
    idx = (idx + 1) & mask;
  }
  atomicOr(ctr.err, ERR_TABLE_FULL);
  return kNull;
}
// read-only probe (the table is complete): slot of k, or kNull
__device__ __forceinline__ uint32_t stack_find(const StackSlot* tab, uint32_t mask, Key128 k, uint32_t zero_present) {
  if (key_zero(k)) return zero_present ? mask + 1 : kNull;
  uint32_t idx = mix_slot(k) & mask;
  for (uint32_t probe = 0; probe <= mask; probe++) {
    Key128 cur = tab[idx].key;
    if (key_eq(cur, k)) return idx;
    if (key_zero(cur)) return kNull;
    idx = (idx + 1) & mask;
  }
  return kNull;
}

// Warp-aggregated insert: lanes carrying the same id elect the lowest lane (== lowest row, rows
// ascend with the lane), which does one table walk and one atomicMax (first row)
// for the whole group. All 32 lanes must call this converged. (Occurrence counts are NOT maintained here:
// on skewed batches the per-stack atomicAdd serialised on a few hot L2 lines and cost more than the
// hashing itself; they are computed on demand by k_count_stacks.)
__device__ __forceinline__ uint32_t warp_insert(StackSlot* tab, uint32_t mask, Key128 k, uint32_t row, bool valid, Counters* ctr, uint32_t* claimed) {
  const unsigned full = 0xFFFFFFFFu;
  int lane = threadIdx.x & 31;
  unsigned long long tag = valid ? (k.lo ^ rotl64(k.hi, 29)) : (0xDEAD00000000ull + lane);
  unsigned grp = __match_any_sync(full, tag);
  int leader = __ffs(grp) - 1;
  unsigned long long lhi = __shfl_sync(full, k.hi, leader), llo = __shfl_sync(full, k.lo, leader);
  int lvalid = __shfl_sync(full, (int)valid, leader);
  bool agree = valid && lvalid && lhi == k.hi && llo == k.lo;
  bool own = valid && (lane == leader || !agree);  // tag collisions between different ids fall back to a private insert
  uint32_t idx = kNull;
  if (own) {
    idx = stack_find_or_insert(tab, mask, k, ctl_of(ctr), claimed);
    if (idx != kNull) {
      uint32_t inv = 0xFFFFFFFFu - row;
      if (*(volatile uint32_t*)&tab[idx].first_inv < inv) atomicMax(&tab[idx].first_inv, inv);
    }
  }
  uint32_t lidx = __shfl_sync(full, idx, leader);
  return own ? idx : (agree ? lidx : kNull);
}

// hashed first-position table for 32-bit keys with an unbounded universe (thread ids)
__device__ __forceinline__ uint32_t fo_hfind(const unsigned long long* hslots, uint32_t hmask, uint32_t key) {
  uint32_t idx = mix32(key) & hmask;
  for (uint32_t probe = 0; probe <= hmask; probe++) {  // bounded: a key lost to a full table must not hang the kernel
    unsigned long long sl = hslots[idx];
    if ((uint32_t)(sl >> 32) == key && sl != ~0ull) return idx;
    if (sl == ~0ull) break;  // linear probing: an empty slot ends the cluster
    idx = (idx + 1) & hmask;
  }
  return 0;  // only reachable after ERR_TABLE_FULL was raised; the batch is redone with a larger table
}
// bounded linear-probe insert of (key, pos) keeping the minimum pos; returns the slot, kNull = table full
__device__ __forceinline__ uint32_t hashed_min_insert(unsigned long long* hslots, uint32_t hmask, uint32_t key, uint32_t pos) {
  unsigned long long packed = ((unsigned long long)key << 32) | pos;
  uint32_t idx = mix32(key) & hmask;
  for (uint32_t probe = 0; probe <= hmask; probe++) {
    unsigned long long cur = hslots[idx];
    if (cur == ~0ull) {
      cur = atomicCAS(&hslots[idx], ~0ull, packed);
      if (cur == ~0ull) return idx;
    }
    if ((uint32_t)(cur >> 32) == key) { if (cur > packed) atomicMin(&hslots[idx], packed); return idx; }
    idx = (idx + 1) & hmask;
  }
  return kNull;
}

// ---------------------------------------------------------------------------------------------
// header pass: 64-byte AoS sample headers -> Arrow row columns + compact SoA side arrays.
// Replaces the per-sample appends of writeSampleV2 (reporter/parca_reporter.go:394-405).
struct HeaderArgs {
  const uint4* hdr;            // 4 x uint4 per row
  uint32_t row0, row1;         // this chunk
  uint32_t row_base;           // mode B: global row of local row 0 (dictionary memos record GLOBAL rows); 0 otherwise
  long long* timestamp;        // Arrow column
  long long* value;            // Arrow column
  uint8_t* uuid;               // Arrow column (16 B/row), written here in provided-hash mode
  uint8_t* kind;
  uint16_t* nframes;
  unsigned long long* frame_off;
  uint32_t* ls;
  uint32_t* cpu;
  uint32_t* tid;
  uint32_t* comm;              // canonical string id of meta.Comm
  const uint32_t* sid2cid;
  uint32_t n_sids, n_labelsets;
  unsigned long long n_frame_ids;  // frames staged for this batch
  int provided;                // hash arrives in the header: insert here
  StackSlot* tab;
  uint32_t mask;
  uint32_t* slot_of_row;
  Counters* ctr;
  uint32_t* claimed;           // list of claimed table slots (see stack_find_or_insert)
  // dictionary memo of the label columns: first row carrying each value. The first row of a value always
  // opens a run, so min over all rows == min over run starts; rows ascend with the grid here, which keeps the
  // atomics rare, and this DRAM-bound kernel has the issue slots to spare. nullptr = column disabled.
  uint32_t* first_ls;            // per labelset id (expanded to the labelset-derived columns by k_ls_plan)
  uint32_t* first_cpu;
  unsigned long long* tid_slots;
  uint32_t tid_mask;
  uint32_t* first_comm;
  uint32_t* first_kind;          // [8] first row of each sample kind (v1: the kind-derived columns are dictionary encoded)
  const uint4* stacks;           // k_header<true>: the registered stack records (RegStack, two uint4 each), one per slot
  uint32_t n_stacks;             // records uploaded for this batch
  uint32_t* last_use;            // k_header<true, true>: per slot, the sequence number of the last batch that named it
  uint32_t seq;                  // this batch's sequence number (batches staged so far, this one included)
};

// Each warp works through tiles of 32 consecutive rows (2 KB of contiguous headers). The next tile's headers arrive in the
// warp's shared-memory buffer by one bulk copy, issued as soon as the current tile has been read into registers, so the
// HBM reads never wait on the L2 lookups of the rows being processed (sid2cid -> first_comm, the tid probe, the first-row
// filters, the stack-table insert in provided-hash mode). Warps share no barrier: a slow insert holds up only its own warp.
// 2 KB of shared memory and at most 32 registers per thread keep all 64 warps of an SM resident, as many as these
// latency-bound lookups want. The shared-memory carveout is left to the driver: the rest of L1 caches the small lookup
// tables, and forcing the largest carveout made the pass about 30 % slower in provided-hash mode on an H100.
// kRegistered (PA_CFG_REGISTERED_STACKS): frame_off is a stack handle, generation << 32 | slot. The slot's 32-byte record must
// carry that generation and not be free; it supplies the stack id, the depth and the arena offset, and hash_hi / hash_lo /
// nframes of the row are ignored. Launched with provided = 1.
// kRetire (PA_CFG_RETIRE_STACKS): the row's batch sequence number is also stored into the slot's last_use word, only when it
// differs: every row of a batch would write the same value, and with Zipf-distributed stacks the stores to hot slots serialise
// in L2 (on an H100, each step a new batch of 4M config-3 rows: +0.026 ms of header time over plain registered stacks, +0.235 ms
// with an unconditional store; DESIGN section 7).
constexpr int kHdrBlocksPerSm = 8;

template <bool kRegistered, bool kRetire = false>
__global__ void __launch_bounds__(kThreads, kHdrBlocksPerSm) k_header(HeaderArgs a) {
  __shared__ __align__(128) uint4 tile_buf[kWarps][32 * 4];
  __shared__ __align__(8) unsigned long long tile_bar[kWarps];
  const uint32_t lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const uint32_t warp = blockIdx.x * kWarps + wib, nwarps = gridDim.x * kWarps;
  const uint32_t tiles = (a.row1 - a.row0 + 31) / 32;
  // tiles warp, warp + nwarps, ...: the trip count is uniform in the warp (warp_insert needs converged warps)
  const uint32_t my_tiles = warp < tiles ? (tiles - warp + nwarps - 1) / nwarps : 0u;
  const uint32_t bar = smem_u32(&tile_bar[wib]), buf = smem_u32(&tile_buf[wib][0]);
  auto issue = [&](uint32_t i) {  // this warp's i-th tile (64 B per row: 16-byte aligned at any row)
    const uint32_t r = a.row0 + (warp + i * nwarps) * 32;
    const uint32_t bytes = min(32u, a.row1 - r) * 64u;
    mbar_arrive_expect_tx(bar, bytes);
    bulk_g2s(buf, a.hdr + 4ull * r, bytes, bar);
  };
  if (lane == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    if (my_tiles) issue(0);
  }
  __syncwarp();
  // Row t of a tile starts at 64 * t bytes: eight lanes reading the same 16-byte word of their rows would hit two
  // 16-byte bank groups. Lane t reads word (k + t / 2) & 3 at step k, which spreads each 8-lane phase of a
  // 128-bit shared load over all 32 banks, and rotates the words back into place afterwards.
  const uint32_t swz = (lane >> 1) & 3u;
  for (uint32_t i = 0; i < my_tiles; i++) {
    const uint32_t r = a.row0 + (warp + i * nwarps) * 32 + lane;
    const bool valid = r < a.row1;
    mbar_wait(bar, i & 1u);
    uint4 q0{}, q1{}, q2{}, q3{};
    if (valid) {
      const uint4* row = &tile_buf[wib][lane * 4];
      q0 = row[swz]; q1 = row[(swz + 1) & 3u]; q2 = row[(swz + 2) & 3u]; q3 = row[(swz + 3) & 3u];
      if (swz & 1u) { const uint4 t = q3; q3 = q2; q2 = q1; q1 = q0; q0 = t; }
      if (swz & 2u) { uint4 t = q0; q0 = q2; q2 = t; t = q1; q1 = q3; q3 = t; }
    }
    __syncwarp();  // the buffer is read: refill it with the warp's next tile
    if (lane == 0 && i + 1 < my_tiles) issue(i + 1);
    Key128 k{0ull, 0ull};
    if (valid) {
      k.hi = ((unsigned long long)q0.y << 32) | q0.x;
      k.lo = ((unsigned long long)q0.w << 32) | q0.z;
      long long ts = (long long)(((unsigned long long)q1.y << 32) | q1.x);
      long long val = (long long)(((unsigned long long)q1.w << 32) | q1.z);
      uint32_t tid = q2.y, comm_sid = q2.z, ls = q2.w;
      unsigned long long foff = ((unsigned long long)q3.y << 32) | q3.x;
      uint32_t cpu = q3.z;
      uint32_t nfr = q3.w & 0xFFFFu, knd = (q3.w >> 16) & 0xFFu;
      uint32_t err = 0;
      if (knd >= 7) { err |= ERR_BAD_KIND; knd = 0; }
      if (ls >= a.n_labelsets) { err |= ERR_BAD_LABELSET; ls = 0; }
      if (comm_sid >= a.n_sids) { err |= ERR_BAD_STRING_ID; comm_sid = 0; }
      if (cpu >= 65536u) { err |= ERR_BAD_CPU; cpu = 0; }
      if (kRegistered && kRetire) {
        const uint32_t slot = (uint32_t)foff, gen = (uint32_t)(foff >> 32);
        uint4 s0{}, s1{};
        if (slot < a.n_stacks) { s0 = __ldg(a.stacks + 2ull * slot); s1 = __ldg(a.stacks + 2ull * slot + 1); }
        if (slot < a.n_stacks && s1.w == gen && !(gen & kStackFree)) {
          k.hi = ((unsigned long long)s0.y << 32) | s0.x;
          k.lo = ((unsigned long long)s0.w << 32) | s0.z;
          foff = ((unsigned long long)s1.y << 32) | s1.x;
          nfr = s1.z;
          if (a.last_use[slot] != a.seq) a.last_use[slot] = a.seq;
        } else {
          err |= ERR_BAD_STACK_ID; k = Key128{0ull, 0ull}; nfr = 0; foff = 0;
        }
      } else if (kRegistered) {
        // Without retirement every record has generation 0 and no slot is free, so the handles the check above accepts are
        // exactly those below the record count. Deciding that before the loads, not on the loaded generation, lets the
        // record's L2 latency overlap the lookups that follow (branching on it cost 0.05-0.11 ms of header time on config 3).
        if (foff < a.n_stacks) {
          const uint4 s0 = __ldg(a.stacks + 2 * foff), s1 = __ldg(a.stacks + 2 * foff + 1);
          k.hi = ((unsigned long long)s0.y << 32) | s0.x;
          k.lo = ((unsigned long long)s0.w << 32) | s0.z;
          foff = ((unsigned long long)s1.y << 32) | s1.x;
          nfr = s1.z;
        } else {
          err |= ERR_BAD_STACK_ID; k = Key128{0ull, 0ull}; nfr = 0; foff = 0;
        }
      } else if (foff + nfr > a.n_frame_ids) { err |= ERR_BAD_FRAME_RANGE; nfr = 0; foff = 0; }
      if (err) atomicOr(&a.ctr->err, err);
      a.timestamp[r] = ts;
      a.value[r] = (knd == 0) ? 1ll : val;  // TraceOriginSampling writes value 1 (:340)
      a.kind[r] = (uint8_t)knd;
      a.nframes[r] = (uint16_t)nfr;
      a.frame_off[r] = foff;
      a.ls[r] = ls;
      a.cpu[r] = cpu;
      a.tid[r] = tid;
      const uint32_t comm_cid = a.sid2cid[comm_sid];
      a.comm[r] = comm_cid;
      const uint32_t gr = a.row_base + r;
      if (a.first_ls && a.first_ls[ls] > gr) atomicMin(&a.first_ls[ls], gr);
      if (a.first_cpu && a.first_cpu[cpu] > gr) atomicMin(&a.first_cpu[cpu], gr);
      if (a.tid_slots && hashed_min_insert(a.tid_slots, a.tid_mask, tid, gr) == kNull) atomicOr(&a.ctr->err, ERR_TABLE_FULL);
      if (a.first_comm && comm_cid != 0 && a.first_comm[comm_cid] > gr) atomicMin(&a.first_comm[comm_cid], gr);
      if (a.first_kind && a.first_kind[knd] > gr) atomicMin(&a.first_kind[knd], gr);
      if (a.provided) {  // trace.Hash.Bytes(): big-endian hi||lo
        ulonglong2 id = make_ulonglong2(bswap64(k.hi), bswap64(k.lo));
        *reinterpret_cast<ulonglong2*>(a.uuid + 16ull * r) = id;
      }
    }
    if (a.provided) {
      uint32_t s = warp_insert(a.tab, a.mask, k, r, valid, a.ctr, a.claimed);
      if (valid) a.slot_of_row[r] = s;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// XXH64 x 2 seeds over each sample's frame ids + fused table insert (PA_HASH_XXH64X2).
constexpr unsigned long long XP1 = 11400714785074694791ULL, XP2 = 14029467366897019727ULL, XP3 = 1609587929392839161ULL,
                             XP4 = 9650029242287828579ULL, XP5 = 2870177450012600261ULL;
constexpr unsigned long long kSeedLo = 0x9E3779B97F4A7C15ULL;

__device__ __forceinline__ unsigned long long xxh_round_pre(unsigned long long acc, unsigned long long in_p2) {
  return rotl64(acc + in_p2, 31) * XP1;  // in_p2 = input * PRIME64_2, shared by both seeds
}
__device__ __forceinline__ unsigned long long xxh_merge(unsigned long long h, unsigned long long v) {
  v = rotl64(v * XP2, 31) * XP1;
  return (h ^ v) * XP1 + XP4;
}
__device__ __forceinline__ unsigned long long xxh_avalanche(unsigned long long h) {
  h ^= h >> 33; h *= XP2; h ^= h >> 29; h *= XP3; h ^= h >> 32;
  return h;
}
__device__ __forceinline__ unsigned long long xxh_lane_init(unsigned long long seed, int j) {
  return j == 0 ? seed + XP1 + XP2 : (j == 1 ? seed + XP2 : (j == 2 ? seed : seed - XP1));
}
struct HashArgs {
  const unsigned long long* frames;
  const uint32_t* frames32;    // non-null: the frame stream holds uint32 ids (narrow ring); `frames` is unused
  const unsigned long long* frame_off;
  const uint16_t* nframes;
  uint32_t row0, row1;
  uint8_t* uuid;
  uint32_t* slot_of_row;
  StackSlot* tab;
  uint32_t mask;
  Counters* ctr;
  uint32_t* claimed;           // list of claimed table slots (see stack_find_or_insert)
};

// Variant B ("direct"): one warp-iteration covers 32 consecutive samples. The XXH64 rounds run with 4 lanes
// per sample (one accumulator lane each, 8 samples at a time, 4 sub-iterations) and the per-sample epilogue —
// accumulator merge, avalanche, 16-byte id store, table insert — runs once with one *thread per
// sample* after a shuffle transpose, so its cost is amortised over 32 samples instead of 8 and
// the id store / slot store are fully coalesced (512 B / 128 B per warp).
__device__ __forceinline__ unsigned long long xxh_finish_own(const unsigned long long (&v)[4], unsigned long long seed, uint32_t n,
                                                             unsigned long long t0, unsigned long long t1, unsigned long long t2) {
  unsigned long long h;
  if (n >= 4) {
    h = rotl64(v[0], 1) + rotl64(v[1], 7) + rotl64(v[2], 12) + rotl64(v[3], 18);
    h = xxh_merge(h, v[0]); h = xxh_merge(h, v[1]); h = xxh_merge(h, v[2]); h = xxh_merge(h, v[3]);
  } else {
    h = seed + XP5;
  }
  h += (unsigned long long)n * 8ull;
  uint32_t t = n & 3u;
  if (t > 0) { h ^= rotl64(t0 * XP2, 31) * XP1; h = rotl64(h, 27) * XP1 + XP4; }
  if (t > 1) { h ^= rotl64(t1 * XP2, 31) * XP1; h = rotl64(h, 27) * XP1 + XP4; }
  if (t > 2) { h ^= rotl64(t2 * XP2, 31) * XP1; h = rotl64(h, 27) * XP1 + XP4; }
  return xxh_avalanche(h);
}

__global__ void __launch_bounds__(kThreads, 4) k_hash_insert(HashArgs a) {
  const unsigned full = 0xFFFFFFFFu;
  const int lane = threadIdx.x & 31, j = lane & 3, g = lane >> 2;
  const uint32_t warp = (blockIdx.x * kThreads + threadIdx.x) >> 5, nwarps = (gridDim.x * kThreads) >> 5;
  const uint32_t span = a.row1 - a.row0;
  const uint32_t iters = (span + nwarps * 32 - 1) / (nwarps * 32);
  for (uint32_t it = 0; it < iters; it++) {
    const uint32_t r = a.row0 + (it * nwarps + warp) * 32 + lane;  // the sample this lane finishes
    const bool valid = r < a.row1;
    const uint32_t n_me = valid ? a.nframes[r] : 0u;
    const unsigned long long off_me = valid ? a.frame_off[r] : 0ull;
    unsigned long long v0[4], v1[4];
#pragma unroll
    for (int sub = 0; sub < 4; sub++) {
      const int src = sub * 8 + g;  // lane that owns the sample my 4-lane group hashes now
      const uint32_t n = __shfl_sync(full, n_me, src);
      const unsigned long long off = __shfl_sync(full, off_me, src);
      const unsigned long long* q = a.frames + off + j;
      unsigned long long a0 = xxh_lane_init(0ull, j), a1 = xxh_lane_init(kSeedLo, j);
      const uint32_t ns = n >> 2;
      uint32_t s = 0;
      for (; s + 8 <= ns; s += 8) {  // 8 stripes = 8 independent 8-byte loads in flight per lane
        unsigned long long w[8];
#pragma unroll
        for (int u = 0; u < 8; u++) w[u] = ldg_stream64(q + 4 * (s + u));
#pragma unroll
        for (int u = 0; u < 8; u++) {
          unsigned long long m = w[u] * XP2;
          a0 = xxh_round_pre(a0, m);
          a1 = xxh_round_pre(a1, m);
        }
      }
      for (; s < ns; s++) {
        unsigned long long m = ldg_stream64(q + 4 * s) * XP2;
        a0 = xxh_round_pre(a0, m);
        a1 = xxh_round_pre(a1, m);
      }
      __syncwarp(full);
      // transpose: lane L (in octet `sub`) receives accumulator lane jj of sample L from lane 4*(L&7)+jj
#pragma unroll
      for (int jj = 0; jj < 4; jj++) {
        unsigned long long x0 = __shfl_sync(full, a0, 4 * (lane & 7) + jj), x1 = __shfl_sync(full, a1, 4 * (lane & 7) + jj);
        if ((lane >> 3) == sub) { v0[jj] = x0; v1[jj] = x1; }
      }
    }
    const uint32_t nt = n_me & 3u;
    const unsigned long long* tp = a.frames + off_me + (n_me & ~3u);
    unsigned long long t0 = nt > 0 ? ldg_stream64(tp) : 0ull, t1 = nt > 1 ? ldg_stream64(tp + 1) : 0ull, t2 = nt > 2 ? ldg_stream64(tp + 2) : 0ull;
    Key128 k;
    k.hi = xxh_finish_own(v0, 0ull, n_me, t0, t1, t2);
    k.lo = xxh_finish_own(v1, kSeedLo, n_me, t0, t1, t2);
    if (valid) *reinterpret_cast<ulonglong2*>(a.uuid + 16ull * r) = make_ulonglong2(bswap64(k.hi), bswap64(k.lo));
    uint32_t slot = warp_insert(a.tab, a.mask, k, r, valid, a.ctr, a.claimed);
    if (valid) a.slot_of_row[r] = slot;
  }
}

// Variant B2 ("wide", the default): two lanes per sample, each owning two of the four XXH64 accumulator lanes and loading
// 16 bytes per stripe (LDG.128): four independent multiply chains per lane (2 accumulators x 2 seeds),
// half the load / address / shuffle instructions of variant B. 16 samples per sub-step, 2 sub-steps
// per 32-sample warp batch; the epilogue is the same thread-per-sample code.
__device__ __forceinline__ uint32_t ldg_stream32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}
// two consecutive ids as uint64 values, from a uint64 stream (16 bytes) or a uint32 stream (8 bytes, widened)
__device__ __forceinline__ ulonglong2 ldg_stream128(const unsigned long long* p);
__device__ __forceinline__ ulonglong2 load_pair(const unsigned long long* p, bool aligned);
__device__ __forceinline__ ulonglong2 load_pair(const uint32_t* p, bool aligned) {
  if (aligned) { const unsigned long long w = ldg_stream64(reinterpret_cast<const unsigned long long*>(p)); return make_ulonglong2(w & 0xFFFFFFFFull, w >> 32); }
  return make_ulonglong2(ldg_stream32(p), ldg_stream32(p + 1));
}
__device__ __forceinline__ unsigned long long load_one(const unsigned long long* p) { return ldg_stream64(p); }
__device__ __forceinline__ unsigned long long load_one(const uint32_t* p) { return ldg_stream32(p); }
__device__ __forceinline__ ulonglong2 ldg_stream128(const unsigned long long* p) {
  ulonglong2 v;
  asm volatile("ld.global.nc.L1::no_allocate.v2.u64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "l"(p));
  return v;
}
#ifndef PA_WIDE_UNROLL
#define PA_WIDE_UNROLL 8
#endif
constexpr int kWideUnroll = PA_WIDE_UNROLL;
// All stripes of one sample half: tiers of kWideUnroll, 4 and up to 3 stripes, each tier with its loads in flight
// together. kAllAligned: every lane of the warp can use 16-byte loads (no predicated 8-byte fallbacks are emitted).
__device__ __forceinline__ ulonglong2 load_pair(const unsigned long long* p, bool aligned) {
  if (aligned) return ldg_stream128(p);
  return make_ulonglong2(ldg_stream64(p), ldg_stream64(p + 1));
}
template <bool kAllAligned, class IdT>
__device__ __forceinline__ void wide_stripes(const IdT* q, uint32_t ns, bool aligned, unsigned long long& a0,
                                             unsigned long long& a1, unsigned long long& b0, unsigned long long& b1) {
  auto load2 = [&](const IdT* p) -> ulonglong2 { return load_pair(p, kAllAligned || aligned); };
  auto rounds = [&](const ulonglong2& w) {
    unsigned long long mx = w.x * XP2, my = w.y * XP2;
    a0 = xxh_round_pre(a0, mx); a1 = xxh_round_pre(a1, mx);
    b0 = xxh_round_pre(b0, my); b1 = xxh_round_pre(b1, my);
  };
  uint32_t s = 0;
  for (; s + kWideUnroll <= ns; s += kWideUnroll) {
    ulonglong2 w[kWideUnroll];
#pragma unroll
    for (int u = 0; u < kWideUnroll; u++) w[u] = load2(q + 4 * (s + u));
#pragma unroll
    for (int u = 0; u < kWideUnroll; u++) rounds(w[u]);
  }
  if (s + 4 <= ns) {
    ulonglong2 w[4];
#pragma unroll
    for (int u = 0; u < 4; u++) w[u] = load2(q + 4 * (s + u));
#pragma unroll
    for (int u = 0; u < 4; u++) rounds(w[u]);
    s += 4;
  }
  if (s < ns) {  // up to three trailing stripes, still loaded together
    ulonglong2 w[3];
#pragma unroll
    for (int u = 0; u < 3; u++) w[u] = (s + u < ns) ? load2(q + 4 * (s + u)) : make_ulonglong2(0ull, 0ull);
#pragma unroll
    for (int u = 0; u < 3; u++) if (s + u < ns) rounds(w[u]);
  }
}
// one warp-tile of 32 consecutive rows (lane = row r); every lane of the warp must call it
template <class IdT>
__device__ __forceinline__ void wide_tile_t(const HashArgs& a, const IdT* frames, uint32_t r, bool valid, uint32_t n_me, unsigned long long off_me) {
  const unsigned full = 0xFFFFFFFFu;
  const int lane = threadIdx.x & 31, h = lane & 1, g = lane >> 1;  // h: which half of the stripe, g: sample within the sub-step
  {
    unsigned long long v0[4], v1[4];
#pragma unroll
    for (int sub = 0; sub < 2; sub++) {
      const int src = sub * 16 + g;
      const uint32_t n = __shfl_sync(full, n_me, src);
      const unsigned long long off = __shfl_sync(full, off_me, src);
      const IdT* q = frames + off + 2 * h;
      unsigned long long a0 = xxh_lane_init(0ull, 2 * h), b0 = xxh_lane_init(0ull, 2 * h + 1);
      unsigned long long a1 = xxh_lane_init(kSeedLo, 2 * h), b1 = xxh_lane_init(kSeedLo, 2 * h + 1);
      const bool aligned = (off & 1ull) == 0;  // paired loads (16 bytes of uint64 ids / 8 bytes of uint32 ids) need an even id offset
      if (__all_sync(full, aligned)) wide_stripes<true>(q, n >> 2, true, a0, a1, b0, b1);   // uniform batches: pure paired loads
      else wide_stripes<false>(q, n >> 2, aligned, a0, a1, b0, b1);                          // ragged: per-lane paired or 2 single loads
      __syncwarp(full);
      // transpose: lane L (in half `sub`) gets accumulators 0,1 from lane 2*(L&15) and 2,3 from lane 2*(L&15)+1
      const int s0 = 2 * (lane & 15), s1 = s0 + 1;
      unsigned long long x;
      x = __shfl_sync(full, a0, s0); if ((lane >> 4) == sub) v0[0] = x;
      x = __shfl_sync(full, b0, s0); if ((lane >> 4) == sub) v0[1] = x;
      x = __shfl_sync(full, a0, s1); if ((lane >> 4) == sub) v0[2] = x;
      x = __shfl_sync(full, b0, s1); if ((lane >> 4) == sub) v0[3] = x;
      x = __shfl_sync(full, a1, s0); if ((lane >> 4) == sub) v1[0] = x;
      x = __shfl_sync(full, b1, s0); if ((lane >> 4) == sub) v1[1] = x;
      x = __shfl_sync(full, a1, s1); if ((lane >> 4) == sub) v1[2] = x;
      x = __shfl_sync(full, b1, s1); if ((lane >> 4) == sub) v1[3] = x;
    }
    const uint32_t nt = n_me & 3u;
    const IdT* tp = frames + off_me + (n_me & ~3u);
    unsigned long long t0 = nt > 0 ? load_one(tp) : 0ull, t1 = nt > 1 ? load_one(tp + 1) : 0ull, t2 = nt > 2 ? load_one(tp + 2) : 0ull;
    Key128 k;
    k.hi = xxh_finish_own(v0, 0ull, n_me, t0, t1, t2);
    k.lo = xxh_finish_own(v1, kSeedLo, n_me, t0, t1, t2);
    if (valid) *reinterpret_cast<ulonglong2*>(a.uuid + 16ull * r) = make_ulonglong2(bswap64(k.hi), bswap64(k.lo));
    uint32_t slot = warp_insert(a.tab, a.mask, k, r, valid, a.ctr, a.claimed);
    if (valid) a.slot_of_row[r] = slot;
  }
}
__device__ __forceinline__ void wide_tile(const HashArgs& a, uint32_t r, bool valid, uint32_t n_me, unsigned long long off_me) {
  wide_tile_t<unsigned long long>(a, a.frames, r, valid, n_me, off_me);
}
// the same pass over a NARROW frame stream (uint32 ids, pa_agg_config.frame_id_bytes = 4): half the bytes per id, ids are
// widened to the uint64 values XXH64 is defined over as they are loaded
__global__ void __launch_bounds__(kThreads, 4) k_hash_insert_wide32(HashArgs a) {
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * kThreads + threadIdx.x) >> 5, nwarps = (gridDim.x * kThreads) >> 5;
  const uint32_t span = a.row1 - a.row0;
  const uint32_t iters = (span + nwarps * 32 - 1) / (nwarps * 32);
  if (iters == 0) return;
  uint32_t r = a.row0 + warp * 32 + lane;
  bool valid = r < a.row1;
  uint32_t n_me = valid ? a.nframes[r] : 0u;
  unsigned long long off_me = valid ? a.frame_off[r] : 0ull;
  for (uint32_t it = 0; it < iters; it++) {  // (the next tile's depths and offsets are fetched under the current tile, as in k_hash_insert_wide)
    const uint32_t r_nx = a.row0 + ((it + 1) * nwarps + warp) * 32 + lane;
    const bool valid_nx = it + 1 < iters && r_nx < a.row1;
    const uint32_t n_nx = valid_nx ? a.nframes[r_nx] : 0u;
    const unsigned long long off_nx = valid_nx ? a.frame_off[r_nx] : 0ull;
    wide_tile_t<uint32_t>(a, a.frames32, r, valid, n_me, off_me);
    r = r_nx; valid = valid_nx; n_me = n_nx; off_me = off_nx;
  }
}
// The NEXT tile's depths and offsets are fetched while the current tile is hashed: a tile otherwise starts with two dependent
// DRAM round trips (nframes / frame_off, then the first ids) during which the warp has nothing in flight (1.058 -> 1.045 ms)
__global__ void __launch_bounds__(kThreads, 4) k_hash_insert_wide(HashArgs a) {
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * kThreads + threadIdx.x) >> 5, nwarps = (gridDim.x * kThreads) >> 5;
  const uint32_t span = a.row1 - a.row0;
  const uint32_t iters = (span + nwarps * 32 - 1) / (nwarps * 32);
  if (iters == 0) return;
  uint32_t r = a.row0 + warp * 32 + lane;
  bool valid = r < a.row1;
  uint32_t n_me = valid ? a.nframes[r] : 0u;
  unsigned long long off_me = valid ? a.frame_off[r] : 0ull;
  for (uint32_t it = 0; it < iters; it++) {
    const uint32_t r_nx = a.row0 + ((it + 1) * nwarps + warp) * 32 + lane;
    const bool valid_nx = it + 1 < iters && r_nx < a.row1;
    const uint32_t n_nx = valid_nx ? a.nframes[r_nx] : 0u;
    const unsigned long long off_nx = valid_nx ? a.frame_off[r_nx] : 0ull;
    wide_tile(a, r, valid, n_me, off_me);
    r = r_nx; valid = valid_nx; n_me = n_nx; off_me = off_nx;
  }
}
// the same without the prefetch of the next tile's depths and offsets (PA_HASH_VARIANT=widenp)
__global__ void __launch_bounds__(kThreads, 4) k_hash_insert_wide_np(HashArgs a) {
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * kThreads + threadIdx.x) >> 5, nwarps = (gridDim.x * kThreads) >> 5;
  const uint32_t span = a.row1 - a.row0;
  const uint32_t iters = (span + nwarps * 32 - 1) / (nwarps * 32);
  for (uint32_t it = 0; it < iters; it++) {
    const uint32_t r = a.row0 + (it * nwarps + warp) * 32 + lane;
    const bool valid = r < a.row1;
    const uint32_t n_me = valid ? a.nframes[r] : 0u;
    const unsigned long long off_me = valid ? a.frame_off[r] : 0ull;
    wide_tile(a, r, valid, n_me, off_me);
  }
}

// Variant B3 ("widepf"): the lane layout of `wide` (two lanes per sample, 16-byte loads, thread-per-sample epilogue) with the
// loads software-pipelined: batches of kPfU stripes ping-pong between two register buffers, the loads of batch i+1 are
// issued before the rounds of batch i, across the two sub-steps of a tile and across tiles (the next tile's depths and
// offsets are fetched one tile ahead). A warp therefore has kPfU..2*kPfU 16-byte loads in flight ALL the time instead of
// 8 during a load phase and none during the ~340 instructions of arithmetic that follow. Ragged depths are handled by
// predication (a warp iterates to its deepest sample), so there is no separate tail code.
constexpr int kPfU = 4;
template <bool kAllAligned, class IdT>
__device__ __forceinline__ void pf_load(ulonglong2 (&w)[kPfU], const IdT* q, uint32_t ns, bool aligned, uint32_t s, bool whole) {
  if (whole) {  // warp-uniform: every lane has all kPfU stripes
#pragma unroll
    for (int u = 0; u < kPfU; u++) w[u] = load_pair(q + 4 * (s + u), kAllAligned || aligned);
  } else {
#pragma unroll
    for (int u = 0; u < kPfU; u++) w[u] = (s + u < ns) ? load_pair(q + 4 * (s + u), kAllAligned || aligned) : make_ulonglong2(0ull, 0ull);
  }
}
__device__ __forceinline__ void pf_rounds(const ulonglong2 (&w)[kPfU], uint32_t ns, uint32_t s, bool whole, unsigned long long& a0, unsigned long long& a1,
                                          unsigned long long& b0, unsigned long long& b1) {
#pragma unroll
  for (int u = 0; u < kPfU; u++) {
    if (whole || s + u < ns) {
      const unsigned long long mx = w[u].x * XP2, my = w[u].y * XP2;
      a0 = xxh_round_pre(a0, mx); a1 = xxh_round_pre(a1, mx);
      b0 = xxh_round_pre(b0, my); b1 = xxh_round_pre(b1, my);
    }
  }
}
struct PfSub {  // one sub-step (16 samples x 2 lanes) as this lane sees it
  unsigned long long off;  // first id of the lane's sample
  uint32_t ns;             // whole stripes of the lane's sample
  uint32_t nsmax, nsmin;   // over the warp
  bool aligned;
};
__device__ __forceinline__ PfSub pf_sub(uint32_t n_me, unsigned long long off_me, int src) {
  const unsigned full = 0xFFFFFFFFu;
  PfSub p;
  p.off = __shfl_sync(full, off_me, src);
  p.ns = __shfl_sync(full, n_me, src) >> 2;
  p.nsmax = __reduce_max_sync(full, p.ns);
  p.nsmin = __reduce_min_sync(full, p.ns);
  p.aligned = (p.off & 1ull) == 0;
  return p;
}
// All batches of one sub-step. On entry A holds the sub-step's first batch; on exit A holds the first batch of `nx` (if has_next).
template <bool kAllAligned, class IdT>
__device__ __forceinline__ void pf_run_sub(const IdT* frames, int h, const PfSub& cu, const PfSub& nx, bool has_next, ulonglong2 (&A)[kPfU], ulonglong2 (&B)[kPfU],
                                           unsigned long long& a0, unsigned long long& a1, unsigned long long& b0, unsigned long long& b1) {
  const IdT* q = frames + cu.off + 2 * h;
  const IdT* qn = frames + nx.off + 2 * h;
  uint32_t s = 0;
  for (;;) {
    bool more = s + kPfU < cu.nsmax;
    if (more) pf_load<kAllAligned>(B, q, cu.ns, cu.aligned, s + kPfU, s + 2 * kPfU <= cu.nsmin);
    else if (has_next) pf_load<kAllAligned>(B, qn, nx.ns, nx.aligned, 0, kPfU <= nx.nsmin);
    pf_rounds(A, cu.ns, s, s + kPfU <= cu.nsmin, a0, a1, b0, b1);
    s += kPfU;
    if (!more) {
#pragma unroll
      for (int u = 0; u < kPfU; u++) A[u] = B[u];
      break;
    }
    more = s + kPfU < cu.nsmax;
    if (more) pf_load<kAllAligned>(A, q, cu.ns, cu.aligned, s + kPfU, s + 2 * kPfU <= cu.nsmin);
    else if (has_next) pf_load<kAllAligned>(A, qn, nx.ns, nx.aligned, 0, kPfU <= nx.nsmin);
    pf_rounds(B, cu.ns, s, s + kPfU <= cu.nsmin, a0, a1, b0, b1);
    s += kPfU;
    if (!more) break;
  }
}
template <class IdT>
__device__ __forceinline__ void hash_insert_widepf(const HashArgs& a, const IdT* frames) {
  const unsigned full = 0xFFFFFFFFu;
  const int lane = threadIdx.x & 31, h = lane & 1, g = lane >> 1;
  const uint32_t warp = (blockIdx.x * kThreads + threadIdx.x) >> 5, nwarps = (gridDim.x * kThreads) >> 5;
  const uint32_t span = a.row1 - a.row0;
  const uint32_t iters = (span + nwarps * 32 - 1) / (nwarps * 32);
  if (iters == 0) return;
  auto meta = [&](uint32_t it, uint32_t& r, bool& valid, uint32_t& n_me, unsigned long long& off_me) {
    r = a.row0 + (it * nwarps + warp) * 32 + lane;
    valid = r < a.row1;
    n_me = valid ? a.nframes[r] : 0u;
    off_me = valid ? a.frame_off[r] : 0ull;
  };
  uint32_t r, n_me; bool valid; unsigned long long off_me;
  meta(0, r, valid, n_me, off_me);
  ulonglong2 A[kPfU], B[kPfU];
  PfSub s0 = pf_sub(n_me, off_me, g);
  bool all_al = __all_sync(full, (off_me & 1ull) == 0);
  if (all_al) pf_load<true>(A, frames + s0.off + 2 * h, s0.ns, true, 0, kPfU <= s0.nsmin);
  else pf_load<false>(A, frames + s0.off + 2 * h, s0.ns, s0.aligned, 0, kPfU <= s0.nsmin);
  for (uint32_t it = 0; it < iters; it++) {
    const bool has_next = it + 1 < iters;
    uint32_t r_nx = 0, n_nx = 0; bool valid_nx = false; unsigned long long off_nx = 0;
    if (has_next) meta(it + 1, r_nx, valid_nx, n_nx, off_nx);
    const PfSub s1 = pf_sub(n_me, off_me, 16 + g);
    const PfSub t0 = pf_sub(n_nx, off_nx, g);
    const bool nx_al = __all_sync(full, (off_nx & 1ull) == 0);
    unsigned long long a0 = xxh_lane_init(0ull, 2 * h), b0 = xxh_lane_init(0ull, 2 * h + 1);
    unsigned long long a1 = xxh_lane_init(kSeedLo, 2 * h), b1 = xxh_lane_init(kSeedLo, 2 * h + 1);
    if (all_al) pf_run_sub<true>(frames, h, s0, s1, true, A, B, a0, a1, b0, b1);
    else pf_run_sub<false>(frames, h, s0, s1, true, A, B, a0, a1, b0, b1);
    unsigned long long c0 = xxh_lane_init(0ull, 2 * h), d0 = xxh_lane_init(0ull, 2 * h + 1);
    unsigned long long c1 = xxh_lane_init(kSeedLo, 2 * h), d1 = xxh_lane_init(kSeedLo, 2 * h + 1);
    // the next tile's first batch is loaded with ITS alignment class: a mixed pair of tiles takes the per-lane path for that batch
    if (all_al && (nx_al || !has_next)) pf_run_sub<true>(frames, h, s1, t0, has_next, A, B, c0, c1, d0, d1);
    else pf_run_sub<false>(frames, h, s1, t0, has_next, A, B, c0, c1, d0, d1);
    // transpose: lane L gets accumulators 0,1 from lane 2*(L&15) and 2,3 from lane 2*(L&15)+1 of ITS half's sub-step
    const int l0 = 2 * (lane & 15), l1 = l0 + 1;
    const bool up = lane >= 16;
    unsigned long long v0[4], v1[4], x, y;
    x = __shfl_sync(full, a0, l0); y = __shfl_sync(full, c0, l0); v0[0] = up ? y : x;
    x = __shfl_sync(full, b0, l0); y = __shfl_sync(full, d0, l0); v0[1] = up ? y : x;
    x = __shfl_sync(full, a0, l1); y = __shfl_sync(full, c0, l1); v0[2] = up ? y : x;
    x = __shfl_sync(full, b0, l1); y = __shfl_sync(full, d0, l1); v0[3] = up ? y : x;
    x = __shfl_sync(full, a1, l0); y = __shfl_sync(full, c1, l0); v1[0] = up ? y : x;
    x = __shfl_sync(full, b1, l0); y = __shfl_sync(full, d1, l0); v1[1] = up ? y : x;
    x = __shfl_sync(full, a1, l1); y = __shfl_sync(full, c1, l1); v1[2] = up ? y : x;
    x = __shfl_sync(full, b1, l1); y = __shfl_sync(full, d1, l1); v1[3] = up ? y : x;
    const uint32_t nt = n_me & 3u;
    const IdT* tp = frames + off_me + (n_me & ~3u);
    unsigned long long t0w = nt > 0 ? load_one(tp) : 0ull, t1w = nt > 1 ? load_one(tp + 1) : 0ull, t2w = nt > 2 ? load_one(tp + 2) : 0ull;
    Key128 k;
    k.hi = xxh_finish_own(v0, 0ull, n_me, t0w, t1w, t2w);
    k.lo = xxh_finish_own(v1, kSeedLo, n_me, t0w, t1w, t2w);
    if (valid) *reinterpret_cast<ulonglong2*>(a.uuid + 16ull * r) = make_ulonglong2(bswap64(k.hi), bswap64(k.lo));
    uint32_t slot = warp_insert(a.tab, a.mask, k, r, valid, a.ctr, a.claimed);
    if (valid) a.slot_of_row[r] = slot;
    r = r_nx; valid = valid_nx; n_me = n_nx; off_me = off_nx; s0 = t0; all_al = nx_al;
  }
}
__global__ void __launch_bounds__(kThreads, 4) k_hash_insert_widepf(HashArgs a) { hash_insert_widepf<unsigned long long>(a, a.frames); }
__global__ void __launch_bounds__(kThreads, 3) k_hash_insert_widepf3(HashArgs a) { hash_insert_widepf<unsigned long long>(a, a.frames); }  // 85 registers: no spills, 24 warps per SM
__global__ void __launch_bounds__(kThreads, 4) k_hash_insert_widepf32(HashArgs a) { hash_insert_widepf<uint32_t>(a, a.frames32); }

// Variant D ("bulk"): the north-star mechanism. Every lane issues ONE cp.async.bulk (TMA 1-D bulk copy, SASS UBLKCP) that
// brings its own sample's frame ids — one contiguous run of <= 64 ids — into a padded shared-memory slot; the copies of a
// warp's 32 samples complete on one mbarrier (32 arrivals + their byte counts). STAGES tiles per warp are in flight, so
// global loads are outstanding ALL the time without holding a single register, and no per-stripe address arithmetic is
// left in the instruction stream. Hashing is thread-per-sample straight out of shared memory: eight independent multiply
// chains per thread (4 XXH64 accumulators x 2 seeds), no shuffles, no transpose; slots are 528 B apart, so the 32 lanes'
// 8-byte reads fall into banks 4*lane + c (4 wavefronts per LDS.64, bank-conflict bound but far from the issue limit).
// A tile with a stack deeper than one slot falls back to the direct-load tile code above.
__device__ __forceinline__ unsigned long long lds64(uint32_t addr) {
  unsigned long long v;
  asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(addr));
  return v;
}
constexpr int kBulkSlotBytes = 64 * 8 + 16;              // 64 ids + 8 B alignment skew + 8 B round-up to a 16-byte multiple
constexpr int kBulkStageBytes = 32 * kBulkSlotBytes;     // one warp-tile
template <int WARPS, int STAGES>
struct BulkSmem {
  alignas(128) uint8_t data[WARPS][STAGES][kBulkStageBytes];
  alignas(8) unsigned long long bar[WARPS][STAGES];
  uint32_t meta[WARPS][STAGES][32];  // per sample: nframes | skew << 16 | in-slot flag << 31
};
template <int WARPS, int STAGES>
__global__ void __launch_bounds__(WARPS * 32, 1) k_hash_insert_bulk(HashArgs a) {
  extern __shared__ __align__(128) uint8_t bulk_smem_raw[];
  BulkSmem<WARPS, STAGES>& sm = *reinterpret_cast<BulkSmem<WARPS, STAGES>*>(bulk_smem_raw);
  const unsigned full = 0xFFFFFFFFu;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const uint32_t warp = blockIdx.x * WARPS + wib, nwarps = gridDim.x * WARPS;
  const uint32_t span = a.row1 - a.row0;
  const uint32_t tiles = (span + 31) / 32;
  if (lane == 0)
    for (int st = 0; st < STAGES; st++) mbar_init(smem_u32(&sm.bar[wib][st]), 32);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();
  // issue the copies of tile `t` (if any) into stage `st`
  auto issue = [&](uint32_t t, int st) {
    if (t >= tiles) return;  // warp-uniform
    const uint32_t r = a.row0 + t * 32 + lane;
    const bool valid = r < a.row1;
    const uint32_t n = valid ? a.nframes[r] : 0u;
    const unsigned long long off = valid ? a.frame_off[r] : 0ull;
    const bool fits = __all_sync(full, n <= 64u);
    const uint32_t bar = smem_u32(&sm.bar[wib][st]);
    const uint32_t skew = (uint32_t)(off & 1ull);
    sm.meta[wib][st][lane] = n | (skew << 16) | (fits ? 0x80000000u : 0u);
    if (fits && n) {
      const uint32_t bytes = ((skew + n + 1u) & ~1u) * 8u;  // [off - skew, off + n) rounded up to a multiple of 16 bytes
      mbar_arrive_expect_tx(bar, bytes);
      bulk_g2s(smem_u32(&sm.data[wib][st][lane * kBulkSlotBytes]), a.frames + (off - skew), bytes, bar);
    } else {
      mbar_arrive(bar);
    }
  };
  uint32_t my_tiles = tiles > warp ? (tiles - warp + nwarps - 1) / nwarps : 0u;
#pragma unroll
  for (int st = 0; st < STAGES - 1; st++) issue(warp + (uint32_t)st * nwarps, st);
  uint32_t phase_bits = 0;  // parity of each stage's barrier
  for (uint32_t k = 0; k < my_tiles; k++) {
    const int st = (int)(k % STAGES);
    // keep STAGES-1 tiles in flight: refill the stage consumed in the previous iteration
    issue(warp + (k + STAGES - 1) * nwarps, (int)((k + STAGES - 1) % STAGES));
    const uint32_t t = warp + k * nwarps;
    const uint32_t r = a.row0 + t * 32 + lane;
    const bool valid = r < a.row1;
    mbar_wait(smem_u32(&sm.bar[wib][st]), (phase_bits >> st) & 1u);
    phase_bits ^= 1u << st;
    const uint32_t m = sm.meta[wib][st][lane];
    const uint32_t n_me = m & 0xFFFFu;
    if (!(m & 0x80000000u)) {  // warp-uniform: a stack deeper than one slot somewhere in the tile
      wide_tile(a, r, valid, n_me, valid ? a.frame_off[r] : 0ull);
      __syncwarp(full);
      continue;
    }
    const uint32_t base = smem_u32(&sm.data[wib][st][lane * kBulkSlotBytes]) + ((m >> 16) & 1u) * 8u;
    unsigned long long v0[4], v1[4];
#pragma unroll
    for (int j = 0; j < 4; j++) { v0[j] = xxh_lane_init(0ull, j); v1[j] = xxh_lane_init(kSeedLo, j); }
    const uint32_t ns = n_me >> 2;
    uint32_t sx = 0;
    for (; sx + 2 <= ns; sx += 2) {  // two stripes per step: 8 loads issued before their 24 multiplies
      unsigned long long w[8];
#pragma unroll
      for (int u = 0; u < 8; u++) w[u] = lds64(base + 32u * sx + 8u * u);
#pragma unroll
      for (int u = 0; u < 8; u++) {
        const unsigned long long mm = w[u] * XP2;
        v0[u & 3] = xxh_round_pre(v0[u & 3], mm);
        v1[u & 3] = xxh_round_pre(v1[u & 3], mm);
      }
    }
    if (sx < ns) {
#pragma unroll
      for (int u = 0; u < 4; u++) {
        const unsigned long long mm = lds64(base + 32u * sx + 8u * u) * XP2;
        v0[u] = xxh_round_pre(v0[u], mm);
        v1[u] = xxh_round_pre(v1[u], mm);
      }
    }
    const uint32_t nt = n_me & 3u, tb = base + 8u * (n_me & ~3u);
    const unsigned long long t0 = nt > 0 ? lds64(tb) : 0ull, t1 = nt > 1 ? lds64(tb + 8) : 0ull, t2 = nt > 2 ? lds64(tb + 16) : 0ull;
    __syncwarp(full);  // every lane is done with this stage before the next iteration's refill
    Key128 key;
    key.hi = xxh_finish_own(v0, 0ull, n_me, t0, t1, t2);
    key.lo = xxh_finish_own(v1, kSeedLo, n_me, t0, t1, t2);
    if (valid) *reinterpret_cast<ulonglong2*>(a.uuid + 16ull * r) = make_ulonglong2(bswap64(key.hi), bswap64(key.lo));
    const uint32_t slot = warp_insert(a.tab, a.mask, key, r, valid, a.ctr, a.claimed);
    if (valid) a.slot_of_row[r] = slot;
  }
}

// Variant E ("tma"): the lane layout and arithmetic of `wide` (two lanes per sample, four multiply chains per lane,
// thread-per-sample epilogue), but the ids reach the lanes through shared memory, brought there by cp.async.bulk (SASS UBLKCP)
// in SMALL stages: one stage = one batch of 8 stripes (256 B) of the 16 samples of a sub-step = 16 bulk copies of <= 272 B
// into 288-B slots (4.5 KB), STAGES of them per warp, WARPS warps per SM (16 x 3: 216 KB). Why this shape: `wide`'s 16-byte
// loads touch one 32-byte sector of 16 different lines per instruction — 16 L1 wavefronts and 16 L2 tag look-ups per 512 B
// (ncu: LSU data pipe 66 %, L2 tags 62 %, DRAM 65 %: everything moderately busy, nothing saturated). A bulk copy fetches whole
// lines without passing the LSU pipe, and the LDS.128 reads of the staged batch are conflict free (slot stride 288 B: four
// consecutive samples fall into four different 32-byte bank groups), 4 wavefronts per 512 B. The first bulk kernel (variant D)
// had whole-stack slots and thread-per-sample hashing and could keep only 6 warps per SM resident; this one keeps 16.
// Odd id offsets are copied from one id earlier (16-byte alignment) and read back with 8-byte loads; any depth works (a
// sub-step simply takes more batches); the < 4 trailing ids of a stack are read directly.
__device__ __forceinline__ ulonglong2 lds128(uint32_t addr) {
  ulonglong2 v;
  asm volatile("ld.shared.v2.u64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "r"(addr));
  return v;
}
// BATCH = stripes per sample per stage (8 or 16): the copy engine handles one bulk copy per ~16-19 cycles per SM whatever its size,
// so 256-byte copies (BATCH 8) cap the kernel near 4 TB/s; 512-byte copies (BATCH 16 = whole 64-frame stacks) do not.
template <int BATCH> constexpr int kTmaSlotBytes = BATCH * 32 + 32;   // BATCH stripes + 8 B alignment skew + 8 B round-up, padded (stride = 32 mod 128)
template <int WARPS, int STAGES, int BATCH>
struct TmaSmem {
  alignas(128) uint8_t data[WARPS][STAGES][16 * kTmaSlotBytes<BATCH>];  // one stage = one batch of the 16 samples of a sub-step
  alignas(8) unsigned long long bar[WARPS][STAGES];
};
template <int WARPS, int STAGES, int BATCH>
__global__ void __launch_bounds__(WARPS * 32, 1) k_hash_insert_tma(HashArgs a) {
  extern __shared__ __align__(128) uint8_t tma_smem_raw[];
  TmaSmem<WARPS, STAGES, BATCH>& sm = *reinterpret_cast<TmaSmem<WARPS, STAGES, BATCH>*>(tma_smem_raw);
  constexpr uint32_t kSlot = kTmaSlotBytes<BATCH>, kStage = 16u * kSlot;
  const unsigned full = 0xFFFFFFFFu;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, h = lane & 1, g = lane >> 1;
  const uint32_t warp = blockIdx.x * WARPS + wib, nwarps = gridDim.x * WARPS;
  const uint32_t span = a.row1 - a.row0;
  const uint32_t tiles = (span + 31) / 32;
  if (lane == 0)
    for (int st = 0; st < STAGES; st++) mbar_init(smem_u32(&sm.bar[wib][st]), 32);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();
  const uint32_t my_tiles = tiles > warp ? (tiles - warp + nwarps - 1) / nwarps : 0u;
  if (my_tiles == 0) return;
  // rows of this warp's k-th tile, as every lane sees its own row; nb = batches per sub-step (warp-uniform)
  auto load_meta = [&](uint32_t k, uint32_t& r, bool& valid, uint32_t& n, unsigned long long& off, uint32_t& nb) {
    r = a.row0 + (warp + k * nwarps) * 32 + lane;
    valid = r < a.row1;
    n = valid ? a.nframes[r] : 0u;
    off = valid ? a.frame_off[r] : 0ull;
    nb = (__reduce_max_sync(full, n >> 2) + (uint32_t)BATCH - 1u) / (uint32_t)BATCH;
  };
  const uint32_t data0 = smem_u32(&sm.data[wib][0][0]), bar0 = smem_u32(&sm.bar[wib][0]);
  // ---- producer: items are (tile, sub-step, batch) in consumption order
  uint32_t pk = 0, p_sub = 0, p_b = 0, p_stage = 0, p_r, p_n, p_nb; bool p_valid; unsigned long long p_off;
  load_meta(0, p_r, p_valid, p_n, p_off, p_nb);
  auto produce = [&]() {
    while (pk < my_tiles && p_nb == 0) {  // tiles without a whole stripe have no items
      if (++pk < my_tiles) load_meta(pk, p_r, p_valid, p_n, p_off, p_nb);
    }
    if (pk >= my_tiles) return;  // warp-uniform
    const int src_lane = (int)p_sub * 16 + (lane & 15);
    const uint32_t n_s = __shfl_sync(full, p_n, src_lane);
    const unsigned long long off_s = __shfl_sync(full, p_off, src_lane);
    const uint32_t bar = bar0 + 8u * p_stage;
    const uint32_t ns = n_s >> 2, first = (uint32_t)BATCH * p_b;
    const uint32_t cnt = ns > first ? min((uint32_t)BATCH, ns - first) : 0u;
    if (lane < 16 && cnt) {
      const uint32_t skew = (uint32_t)(off_s & 1ull);
      const uint32_t bytes = ((skew + 4u * cnt + 1u) & ~1u) * 8u;  // [first id - skew, last id] rounded up to a multiple of 16 bytes
      mbar_arrive_expect_tx(bar, bytes);
      bulk_g2s(data0 + p_stage * kStage + (uint32_t)lane * kSlot, a.frames + (off_s + 4ull * first - skew), bytes, bar);
    } else {
      mbar_arrive(bar);
    }
    p_stage = p_stage + 1 == STAGES ? 0 : p_stage + 1;
    if (++p_b == p_nb) {
      p_b = 0;
      if (++p_sub == 2) {
        p_sub = 0;
        p_nb = 0;
        if (++pk < my_tiles) load_meta(pk, p_r, p_valid, p_n, p_off, p_nb);
      }
    }
  };
#pragma unroll
  for (int i = 0; i < STAGES - 1; i++) produce();
  // ---- consumer
  uint32_t c_stage = 0, phase_bits = 0;
  for (uint32_t k = 0; k < my_tiles; k++) {
    uint32_t r, n_me, nb; bool valid; unsigned long long off_me;
    load_meta(k, r, valid, n_me, off_me, nb);
    unsigned long long acc[2][4];  // [sub][a0, a1, b0, b1]
#pragma unroll
    for (int sub = 0; sub < 2; sub++) {
      const uint32_t ns_s = __shfl_sync(full, n_me, sub * 16 + g) >> 2;
      const uint32_t skew_s = (uint32_t)(__shfl_sync(full, off_me, sub * 16 + g) & 1ull);
      const bool any_skew = __any_sync(full, skew_s != 0);
      unsigned long long a0 = xxh_lane_init(0ull, 2 * h), b0 = xxh_lane_init(0ull, 2 * h + 1);
      unsigned long long a1 = xxh_lane_init(kSeedLo, 2 * h), b1 = xxh_lane_init(kSeedLo, 2 * h + 1);
      for (uint32_t b = 0; b < nb; b++) {
        produce();  // refills the stage consumed in the previous iteration
        mbar_wait(bar0 + 8u * c_stage, (phase_bits >> c_stage) & 1u);
        phase_bits ^= 1u << c_stage;
        const uint32_t first = (uint32_t)BATCH * b;
        const uint32_t cnt = ns_s > first ? min((uint32_t)BATCH, ns_s - first) : 0u;
        const uint32_t base = data0 + c_stage * kStage + (uint32_t)g * kSlot + skew_s * 8u + (uint32_t)h * 16u;
        if (!any_skew && __all_sync(full, cnt == (uint32_t)BATCH)) {
#pragma unroll
          for (int blk = 0; blk < BATCH / 8; blk++) {
            ulonglong2 w[8];
#pragma unroll
            for (int u = 0; u < 8; u++) w[u] = lds128(base + 32u * (8 * blk + u));
#pragma unroll
            for (int u = 0; u < 8; u++) {
              const unsigned long long mx = w[u].x * XP2, my = w[u].y * XP2;
              a0 = xxh_round_pre(a0, mx); a1 = xxh_round_pre(a1, mx);
              b0 = xxh_round_pre(b0, my); b1 = xxh_round_pre(b1, my);
            }
          }
        } else {
          for (uint32_t u = 0; u < cnt; u++) {
            const unsigned long long mx = lds64(base + 32u * u) * XP2, my = lds64(base + 32u * u + 8u) * XP2;
            a0 = xxh_round_pre(a0, mx); a1 = xxh_round_pre(a1, mx);
            b0 = xxh_round_pre(b0, my); b1 = xxh_round_pre(b1, my);
          }
        }
        __syncwarp(full);  // every lane has read this stage before the next produce() refills it
        c_stage = c_stage + 1 == STAGES ? 0 : c_stage + 1;
      }
      acc[sub][0] = a0; acc[sub][1] = a1; acc[sub][2] = b0; acc[sub][3] = b1;
    }
    // transpose: lane L gets accumulators 0,1 from lane 2*(L&15) and 2,3 from lane 2*(L&15)+1 of ITS half's sub-step
    const int l0 = 2 * (lane & 15), l1 = l0 + 1;
    const bool up = lane >= 16;
    unsigned long long v0[4], v1[4], x, y;
    x = __shfl_sync(full, acc[0][0], l0); y = __shfl_sync(full, acc[1][0], l0); v0[0] = up ? y : x;
    x = __shfl_sync(full, acc[0][2], l0); y = __shfl_sync(full, acc[1][2], l0); v0[1] = up ? y : x;
    x = __shfl_sync(full, acc[0][0], l1); y = __shfl_sync(full, acc[1][0], l1); v0[2] = up ? y : x;
    x = __shfl_sync(full, acc[0][2], l1); y = __shfl_sync(full, acc[1][2], l1); v0[3] = up ? y : x;
    x = __shfl_sync(full, acc[0][1], l0); y = __shfl_sync(full, acc[1][1], l0); v1[0] = up ? y : x;
    x = __shfl_sync(full, acc[0][3], l0); y = __shfl_sync(full, acc[1][3], l0); v1[1] = up ? y : x;
    x = __shfl_sync(full, acc[0][1], l1); y = __shfl_sync(full, acc[1][1], l1); v1[2] = up ? y : x;
    x = __shfl_sync(full, acc[0][3], l1); y = __shfl_sync(full, acc[1][3], l1); v1[3] = up ? y : x;
    const uint32_t nt = n_me & 3u;
    const unsigned long long* tp = a.frames + off_me + (n_me & ~3u);
    const unsigned long long t0w = nt > 0 ? load_one(tp) : 0ull, t1w = nt > 1 ? load_one(tp + 1) : 0ull, t2w = nt > 2 ? load_one(tp + 2) : 0ull;
    Key128 key;
    key.hi = xxh_finish_own(v0, 0ull, n_me, t0w, t1w, t2w);
    key.lo = xxh_finish_own(v1, kSeedLo, n_me, t0w, t1w, t2w);
    if (valid) *reinterpret_cast<ulonglong2*>(a.uuid + 16ull * r) = make_ulonglong2(bswap64(key.hi), bswap64(key.lo));
    const uint32_t slot = warp_insert(a.tab, a.mask, key, r, valid, a.ctr, a.claimed);
    if (valid) a.slot_of_row[r] = slot;
  }
}

// Variant F ("tmag"): variant E with FOUR bulk copies per stage instead of sixteen. ptxas turns a per-lane cp.async.bulk into a
// loop over the active lanes (ELECT / R2UR x5 / UBLKCP / BRA.U.ANY: its operands live in uniform registers), so sixteen copies
// cost ~160 issue slots and ~600 cycles of one warp per stage. Rows are contiguous in the ring, so one copy can bring the whole
// stacks of four consecutive samples (<= 2 KiB); the four groups of a sub-step sit 2080 B apart (= 32 mod 128) and lane pair g
// hashes sample (g & 3) * 4 + (g >> 2), so the four pairs of every 128-bit shared-memory phase read from four different groups:
// conflict free for uniform depths. One stage = one sub-step (16 whole stacks, 8.3 KB). A tile whose groups are not contiguous
// or exceed 256 ids goes through the direct-load tile code.
constexpr int kTmagGroupBytes = 2048 + 32;
constexpr int kTmagStageBytes = 4 * kTmagGroupBytes;
template <int WARPS, int STAGES>
struct TmagSmem {
  alignas(128) uint8_t data[WARPS][STAGES][kTmagStageBytes];
  alignas(8) unsigned long long bar[WARPS][STAGES];
};
template <int WARPS, int STAGES>
__global__ void __launch_bounds__(WARPS * 32, 1) k_hash_insert_tmag(HashArgs a) {
  extern __shared__ __align__(128) uint8_t tmag_smem_raw[];
  TmagSmem<WARPS, STAGES>& sm = *reinterpret_cast<TmagSmem<WARPS, STAGES>*>(tmag_smem_raw);
  const unsigned full = 0xFFFFFFFFu;
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5, h = lane & 1, g = lane >> 1;
  const uint32_t warp = blockIdx.x * WARPS + wib, nwarps = gridDim.x * WARPS;
  const uint32_t span = a.row1 - a.row0;
  const uint32_t tiles = (span + 31) / 32;
  if (lane == 0)
    for (int st = 0; st < STAGES; st++) mbar_init(smem_u32(&sm.bar[wib][st]), 32);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncthreads();
  const uint32_t my_tiles = tiles > warp ? (tiles - warp + nwarps - 1) / nwarps : 0u;
  if (my_tiles == 0) return;
  // Per tile, as lane L sees its own row: depth, offset, ids of the earlier rows of its group of four (pre), ids of the whole
  // group (tot), and whether the whole tile can be staged (every group contiguous and <= 256 ids).
  struct Meta { uint32_t r, n, pre, tot; unsigned long long off; bool valid, staged; };
  auto load_meta = [&](uint32_t k) {
    Meta m;
    m.r = a.row0 + (warp + k * nwarps) * 32 + lane;
    m.valid = m.r < a.row1;
    m.n = m.valid ? a.nframes[m.r] : 0u;
    m.off = m.valid ? a.frame_off[m.r] : 0ull;
    const uint32_t up1 = __shfl_up_sync(full, m.n, 1), up2 = __shfl_up_sync(full, m.n, 2), up3 = __shfl_up_sync(full, m.n, 3);
    const int q = lane & 3;
    m.pre = (q > 0 ? up1 : 0u) + (q > 1 ? up2 : 0u) + (q > 2 ? up3 : 0u);
    m.tot = __shfl_sync(full, m.pre + m.n, lane | 3);
    const unsigned long long off0 = __shfl_sync(full, m.off, lane & ~3);
    m.staged = __all_sync(full, (m.n == 0 || m.off == off0 + m.pre) && m.tot <= 256u);
    return m;
  };
  const uint32_t data0 = smem_u32(&sm.data[wib][0][0]), bar0 = smem_u32(&sm.bar[wib][0]);
  // ---- producer: two items per tile (its two sub-steps), in consumption order
  uint32_t pk = 0, p_sub = 0, p_stage = 0;
  Meta pm = load_meta(0);
  auto produce = [&]() {
    if (pk >= my_tiles) return;  // warp-uniform
    const uint32_t bar = bar0 + 8u * p_stage;
    const int src_lane = (int)p_sub * 16 + (lane & 15);
    const uint32_t tot_s = __shfl_sync(full, pm.tot, src_lane);
    const unsigned long long off_s = __shfl_sync(full, pm.off, src_lane);
    if (pm.staged && lane < 16 && (lane & 3) == 0 && tot_s) {
      const uint32_t skew = (uint32_t)(off_s & 1ull);
      const uint32_t bytes = ((skew + tot_s + 1u) & ~1u) * 8u;
      mbar_arrive_expect_tx(bar, bytes);
      bulk_g2s(data0 + p_stage * kTmagStageBytes + (uint32_t)(lane >> 2) * kTmagGroupBytes, a.frames + (off_s - skew), bytes, bar);
    } else {
      mbar_arrive(bar);
    }
    p_stage = p_stage + 1 == STAGES ? 0 : p_stage + 1;
    if (++p_sub == 2) {
      p_sub = 0;
      if (++pk < my_tiles) pm = load_meta(pk);
    }
  };
#pragma unroll
  for (int i = 0; i < STAGES - 1; i++) produce();
  // ---- consumer
  uint32_t c_stage = 0, phase_bits = 0;
  const int sg = (g & 3) * 4 + (g >> 2);  // the sample (within a sub-step) this lane pair hashes
  for (uint32_t k = 0; k < my_tiles; k++) {
    const Meta cm = load_meta(k);
    if (!cm.staged) {  // warp-uniform: both (empty) items of the tile are consumed, the tile goes through the direct-load code
      for (int sub = 0; sub < 2; sub++) {
        produce();
        mbar_wait(bar0 + 8u * c_stage, (phase_bits >> c_stage) & 1u);
        phase_bits ^= 1u << c_stage;
        c_stage = c_stage + 1 == STAGES ? 0 : c_stage + 1;
      }
      wide_tile(a, cm.r, cm.valid, cm.n, cm.off);
      __syncwarp(full);
      continue;
    }
    unsigned long long acc[2][4];  // [sub][a0, a1, b0, b1]
#pragma unroll
    for (int sub = 0; sub < 2; sub++) {
      const int ml = sub * 16 + sg;  // the lane that holds this pair's sample
      const uint32_t ns = __shfl_sync(full, cm.n, ml) >> 2;
      const uint32_t pre = __shfl_sync(full, cm.pre, ml);
      const uint32_t skew = (uint32_t)(__shfl_sync(full, cm.off, ml & ~3) & 1ull);  // of the group's first id
      unsigned long long a0 = xxh_lane_init(0ull, 2 * h), b0 = xxh_lane_init(0ull, 2 * h + 1);
      unsigned long long a1 = xxh_lane_init(kSeedLo, 2 * h), b1 = xxh_lane_init(kSeedLo, 2 * h + 1);
      produce();  // refills the stage consumed before this one
      mbar_wait(bar0 + 8u * c_stage, (phase_bits >> c_stage) & 1u);
      phase_bits ^= 1u << c_stage;
      const uint32_t base = data0 + c_stage * kTmagStageBytes + (uint32_t)(g & 3) * kTmagGroupBytes + (skew + pre) * 8u + (uint32_t)h * 16u;
      const bool al16 = ((skew + pre) & 1u) == 0;
      const uint32_t nsmin = __reduce_min_sync(full, ns), nsmax = __reduce_max_sync(full, ns);
      uint32_t s = 0;
      if (__all_sync(full, al16)) {
        for (; s + 8 <= nsmin; s += 8) {  // warp-uniform: every pair has 8 more stripes
          ulonglong2 w[8];
#pragma unroll
          for (int u = 0; u < 8; u++) w[u] = lds128(base + 32u * (s + u));
#pragma unroll
          for (int u = 0; u < 8; u++) {
            const unsigned long long mx = w[u].x * XP2, my = w[u].y * XP2;
            a0 = xxh_round_pre(a0, mx); a1 = xxh_round_pre(a1, mx);
            b0 = xxh_round_pre(b0, my); b1 = xxh_round_pre(b1, my);
          }
        }
      }
      for (; s < nsmax; s++) {  // ragged rest (and everything, when an odd id offset forces 8-byte reads)
        if (s < ns) {
          const unsigned long long mx = lds64(base + 32u * s) * XP2, my = lds64(base + 32u * s + 8u) * XP2;
          a0 = xxh_round_pre(a0, mx); a1 = xxh_round_pre(a1, mx);
          b0 = xxh_round_pre(b0, my); b1 = xxh_round_pre(b1, my);
        }
      }
      __syncwarp(full);  // every lane has read this stage before the next produce() refills it
      c_stage = c_stage + 1 == STAGES ? 0 : c_stage + 1;
      acc[sub][0] = a0; acc[sub][1] = a1; acc[sub][2] = b0; acc[sub][3] = b1;
    }
    // transpose: lane L (sample s = L & 15 of its half's sub-step) takes accumulators 0,1 / 2,3 from the two lanes of the pair that hashed s
    const int sp = ((lane & 3) * 4 + ((lane & 15) >> 2));
    const int l0 = 2 * sp, l1 = l0 + 1;
    const bool up = lane >= 16;
    unsigned long long v0[4], v1[4], x, y;
    x = __shfl_sync(full, acc[0][0], l0); y = __shfl_sync(full, acc[1][0], l0); v0[0] = up ? y : x;
    x = __shfl_sync(full, acc[0][2], l0); y = __shfl_sync(full, acc[1][2], l0); v0[1] = up ? y : x;
    x = __shfl_sync(full, acc[0][0], l1); y = __shfl_sync(full, acc[1][0], l1); v0[2] = up ? y : x;
    x = __shfl_sync(full, acc[0][2], l1); y = __shfl_sync(full, acc[1][2], l1); v0[3] = up ? y : x;
    x = __shfl_sync(full, acc[0][1], l0); y = __shfl_sync(full, acc[1][1], l0); v1[0] = up ? y : x;
    x = __shfl_sync(full, acc[0][3], l0); y = __shfl_sync(full, acc[1][3], l0); v1[1] = up ? y : x;
    x = __shfl_sync(full, acc[0][1], l1); y = __shfl_sync(full, acc[1][1], l1); v1[2] = up ? y : x;
    x = __shfl_sync(full, acc[0][3], l1); y = __shfl_sync(full, acc[1][3], l1); v1[3] = up ? y : x;
    const uint32_t nt = cm.n & 3u;
    const unsigned long long* tp = a.frames + cm.off + (cm.n & ~3u);
    const unsigned long long t0w = nt > 0 ? load_one(tp) : 0ull, t1w = nt > 1 ? load_one(tp + 1) : 0ull, t2w = nt > 2 ? load_one(tp + 2) : 0ull;
    Key128 key;
    key.hi = xxh_finish_own(v0, 0ull, cm.n, t0w, t1w, t2w);
    key.lo = xxh_finish_own(v1, kSeedLo, cm.n, t0w, t1w, t2w);
    if (cm.valid) *reinterpret_cast<ulonglong2*>(a.uuid + 16ull * cm.r) = make_ulonglong2(bswap64(key.hi), bswap64(key.lo));
    const uint32_t slot = warp_insert(a.tab, a.mask, key, cm.r, cm.valid, a.ctr, a.claimed);
    if (cm.valid) a.slot_of_row[cm.r] = slot;
  }
}

// Variant C: same arithmetic and epilogue as k_hash_insert, but the frame ids reach the XXH64 lanes
// through shared memory: every warp owns a two-stage ring (8 samples x 544 B per stage) that it fills
// with cp.async (LDGSTS, 16 B per lane = one coalesced 512-B sample per instruction, no registers
// held) one sub-step ahead of the one it is hashing. Loads are therefore in flight *all the time*
// instead of only between compute bursts, and the 8-byte LDS reads are bank-conflict free thanks to
// the 32-byte pad per sample slot (half-warp = 4 samples x 4 lanes -> 32 distinct banks).
constexpr int kSlotBytes = 64 * 8 + 32;          // one sample of up to 64 frames + pad
constexpr int kStageBytes = 8 * kSlotBytes;      // 8 samples
constexpr int kHashStagedSmem = kWarps * 2 * kStageBytes;

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async8(uint32_t dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
// stage the 8 samples owned by lanes sub*8 .. sub*8+7 (n <= 64 frames each) into `stage`
__device__ __forceinline__ void stage_samples(const unsigned long long* frames, uint32_t n_me, unsigned long long off_me, int sub, uint32_t stage,
                                              int lane) {
  const unsigned full = 0xFFFFFFFFu;
#pragma unroll
  for (int i = 0; i < 8; i++) {
    const uint32_t n = __shfl_sync(full, n_me, sub * 8 + i);
    const unsigned long long off = __shfl_sync(full, off_me, sub * 8 + i);
    const unsigned long long* src = frames + off;
    const uint32_t dst = stage + i * kSlotBytes;
    if ((off & 1ull) == 0) {  // 16-byte aligned source: one 16-byte copy per lane covers words 2l, 2l+1
      const uint32_t w = 2u * lane;
      if (w + 1 < n) cp_async16(dst + 8 * w, src + w);
      else if (w < n) cp_async8(dst + 8 * w, src + w);
    } else {                  // odd word offset: 8-byte copies
      if ((uint32_t)lane < n) cp_async8(dst + 8 * lane, src + lane);
      if ((uint32_t)lane + 32 < n) cp_async8(dst + 8 * (lane + 32), src + lane + 32);
    }
  }
}

__global__ void __launch_bounds__(kThreads, 3) k_hash_insert_staged(HashArgs a) {
  extern __shared__ __align__(16) uint8_t hsmem[];
  const unsigned full = 0xFFFFFFFFu;
  const int lane = threadIdx.x & 31, j = lane & 3, g = lane >> 2, wib = threadIdx.x >> 5;
  const uint32_t warp = (blockIdx.x * kThreads + threadIdx.x) >> 5, nwarps = (gridDim.x * kThreads) >> 5;
  const uint32_t span = a.row1 - a.row0;
  const uint32_t iters = (span + nwarps * 32 - 1) / (nwarps * 32);
  const uint32_t ring = (uint32_t)__cvta_generic_to_shared(hsmem) + wib * 2 * kStageBytes;

  auto batch_row = [&](uint32_t it) { return a.row0 + (it * nwarps + warp) * 32 + lane; };
  uint32_t r = batch_row(0);
  bool valid = r < a.row1;
  uint32_t n_me = valid ? a.nframes[r] : 0u;
  unsigned long long off_me = valid ? a.frame_off[r] : 0ull;
  bool staged = __all_sync(full, n_me <= 64u);
  if (iters && staged) stage_samples(a.frames, n_me, off_me, 0, ring, lane);
  cp_async_commit();

  for (uint32_t it = 0; it < iters; it++) {
    // the next batch's sizes/offsets (its first sub-step is staged during this batch's last one)
    uint32_t r_nx = batch_row(it + 1);
    bool valid_nx = (it + 1 < iters) && r_nx < a.row1;
    uint32_t n_nx = valid_nx ? a.nframes[r_nx] : 0u;
    unsigned long long off_nx = valid_nx ? a.frame_off[r_nx] : 0ull;
    bool staged_nx = __all_sync(full, n_nx <= 64u);

    unsigned long long v0[4], v1[4];
#pragma unroll
    for (int sub = 0; sub < 4; sub++) {
      const uint32_t cur = ring + (sub & 1) * kStageBytes, nxt = ring + ((sub + 1) & 1) * kStageBytes;
      if (sub < 3) { if (staged) stage_samples(a.frames, n_me, off_me, sub + 1, nxt, lane); }
      else if (it + 1 < iters && staged_nx) stage_samples(a.frames, n_nx, off_nx, 0, nxt, lane);
      cp_async_commit();
      cp_async_wait<1>();  // everything but the group just committed has landed
      __syncwarp(full);
      const int src = sub * 8 + g;
      const uint32_t n = __shfl_sync(full, n_me, src);
      const unsigned long long off = __shfl_sync(full, off_me, src);
      unsigned long long a0 = xxh_lane_init(0ull, j), a1 = xxh_lane_init(kSeedLo, j);
      const uint32_t ns = n >> 2;
      if (staged) {
        const uint32_t q = cur + g * kSlotBytes + 8 * j;
        uint32_t s = 0;
        for (; s + 8 <= ns; s += 8) {
          unsigned long long w[8];
#pragma unroll
          for (int u = 0; u < 8; u++) w[u] = lds64(q + 32 * (s + u));
#pragma unroll
          for (int u = 0; u < 8; u++) { unsigned long long m = w[u] * XP2; a0 = xxh_round_pre(a0, m); a1 = xxh_round_pre(a1, m); }
        }
        for (; s < ns; s++) { unsigned long long m = lds64(q + 32 * s) * XP2; a0 = xxh_round_pre(a0, m); a1 = xxh_round_pre(a1, m); }
      } else {  // a stack deeper than one slot in this batch: stream it from global memory
        const unsigned long long* q = a.frames + off + j;
        for (uint32_t s = 0; s < ns; s++) { unsigned long long m = ldg_stream64(q + 4 * s) * XP2; a0 = xxh_round_pre(a0, m); a1 = xxh_round_pre(a1, m); }
      }
      __syncwarp(full);  // all lanes are done with `cur` before the next sub-step refills it
#pragma unroll
      for (int jj = 0; jj < 4; jj++) {
        unsigned long long x0 = __shfl_sync(full, a0, 4 * (lane & 7) + jj), x1 = __shfl_sync(full, a1, 4 * (lane & 7) + jj);
        if ((lane >> 3) == sub) { v0[jj] = x0; v1[jj] = x1; }
      }
    }
    const uint32_t nt = n_me & 3u;
    const unsigned long long* tp = a.frames + off_me + (n_me & ~3u);
    unsigned long long t0 = nt > 0 ? ldg_stream64(tp) : 0ull, t1 = nt > 1 ? ldg_stream64(tp + 1) : 0ull, t2 = nt > 2 ? ldg_stream64(tp + 2) : 0ull;
    Key128 k;
    k.hi = xxh_finish_own(v0, 0ull, n_me, t0, t1, t2);
    k.lo = xxh_finish_own(v1, kSeedLo, n_me, t0, t1, t2);
    if (valid) *reinterpret_cast<ulonglong2*>(a.uuid + 16ull * r) = make_ulonglong2(bswap64(k.hi), bswap64(k.lo));
    uint32_t slot = warp_insert(a.tab, a.mask, k, r, valid, a.ctr, a.claimed);
    if (valid) a.slot_of_row[r] = slot;
    r = r_nx; valid = valid_nx; n_me = n_nx; off_me = off_nx; staged = staged_nx;
  }
  cp_async_wait<0>();
}

// ---------------------------------------------------------------------------------------------
// block-wide exclusive scan (kThreads threads). T needs operator+ and a zero-initialised T().
struct Pair { uint32_t cnt; unsigned long long fr; };
__device__ __forceinline__ Pair operator+(Pair a, Pair b) { return Pair{a.cnt + b.cnt, a.fr + b.fr}; }
__device__ __forceinline__ uint32_t shfl_up_t(uint32_t v, int d) { return __shfl_up_sync(0xFFFFFFFFu, v, d); }
__device__ __forceinline__ Pair shfl_up_t(Pair v, int d) {
  return Pair{__shfl_up_sync(0xFFFFFFFFu, v.cnt, d), __shfl_up_sync(0xFFFFFFFFu, v.fr, d)};
}
__device__ __forceinline__ unsigned long long shfl_up_t(unsigned long long v, int d) { return __shfl_up_sync(0xFFFFFFFFu, v, d); }
__device__ __forceinline__ unsigned long long shfl_idx_t(unsigned long long v, int l) { return __shfl_sync(0xFFFFFFFFu, v, l); }
__device__ __forceinline__ unsigned long long zero_of(unsigned long long) { return 0ull; }
__device__ __forceinline__ uint32_t shfl_idx_t(uint32_t v, int l) { return __shfl_sync(0xFFFFFFFFu, v, l); }
__device__ __forceinline__ Pair shfl_idx_t(Pair v, int l) { return Pair{__shfl_sync(0xFFFFFFFFu, v.cnt, l), __shfl_sync(0xFFFFFFFFu, v.fr, l)}; }
__device__ __forceinline__ uint32_t zero_of(uint32_t) { return 0u; }
__device__ __forceinline__ Pair zero_of(Pair) { return Pair{0u, 0ull}; }

template <class T>
__device__ __forceinline__ T block_exclusive_scan(T v, T* total) {
  __shared__ T s_w[kWarps];
  __shared__ T s_tot;
  int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  T inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    T o = shfl_up_t(inc, d);
    if (lane >= d) inc = o + inc;
  }
  if (lane == 31) s_w[w] = inc;
  __syncthreads();
  if (threadIdx.x == 0) {
    T run = zero_of(v);
    for (int i = 0; i < kWarps; i++) { T t = s_w[i]; s_w[i] = run; run = run + t; }
    s_tot = run;
  }
  __syncthreads();
  T excl_in_warp = shfl_up_t(inc, 1);
  if (lane == 0) excl_in_warp = zero_of(v);
  T res = s_w[w] + excl_in_warp;
  *total = s_tot;
  __syncthreads();  // s_w / s_tot are reused by the next tile
  return res;
}

// Generic fixed-grid reduce-then-scan. F provides:
//   typedef T; uint32_t n(); T value(uint32_t i); void emit(uint32_t i, T exclusive, T v); void total(int job, T t);
// blockIdx.y selects an independent job; two launches per scan (reduce, emit). (A cooperative single-launch variant with grid-wide barriers
// between the phases was measured and was slower than these pipelined launches: DESIGN.md section 7.)
template <class F>
__global__ void __launch_bounds__(kThreads) k_scan_reduce(F f, typename F::T* partial) {
  typedef typename F::T T;
  T* partial_of_job = partial + (size_t)blockIdx.y * gridDim.x;
  uint32_t n = f.n(), begin, end;
  block_range(n, &begin, &end);
  T acc = zero_of(T());
  for (uint32_t i = begin + threadIdx.x; i < end; i += kThreads) acc = acc + f.value(i);
  T tot;
  block_exclusive_scan(acc, &tot);
  if (threadIdx.x == 0) partial_of_job[blockIdx.x] = tot;
}
// Emit phase. `partial` holds the per-block TOTALS written by k_scan_reduce; every block sums the
// totals of its predecessors itself (at most a few hundred values), which removes the separate
// "scan the partials" launch; the last block also publishes the grand total.
template <class F>
__global__ void __launch_bounds__(kThreads) k_scan_emit(F f, const typename F::T* partial) {
  typedef typename F::T T;
  const T* partial_of_job = partial + (size_t)blockIdx.y * gridDim.x;
  uint32_t n = f.n(), begin, end;
  block_range(n, &begin, &end);
  T mine = zero_of(T());
  for (uint32_t b = threadIdx.x; b < blockIdx.x; b += kThreads) mine = mine + partial_of_job[b];
  T run;
  block_exclusive_scan(mine, &run);  // run = sum of all preceding blocks' totals
  if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) f.total((int)blockIdx.y, run + partial_of_job[blockIdx.x]);
  for (uint32_t tile = begin; tile < end; tile += kThreads) {
    uint32_t i = tile + threadIdx.x;
    bool in = i < end;
    T v = in ? f.value(i) : zero_of(T());
    T tot;
    T ex = block_exclusive_scan(v, &tot);
    if (in) f.emit(i, run + ex, v);
    run = run + tot;
  }
}

// ---------------------------------------------------------------------------------------------
// (1) unique stacks in first-occurrence order. The table holds each stack's first row; ordinals
// come from a bitmap over rows (one bit per first occurrence) + a popcount prefix over its words,
// so only table-sized and N/32-sized passes are needed (no scan over all rows).
__global__ void __launch_bounds__(kThreads) k_stack_bits(const StackSlot* tab, const uint32_t* claimed, const uint32_t* n_claimed, uint32_t* rowbits) {
  const uint32_t n = *n_claimed;
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
    uint32_t f = 0xFFFFFFFFu - tab[claimed[i]].first_inv;
    atomicOr(&rowbits[f >> 5], 1u << (f & 31));
  }
}
struct WordsF {  // exclusive popcount prefix over bitmap words
  typedef uint32_t T;
  const uint32_t* bits;
  uint32_t* wprefix;
  uint32_t n_words;
  uint32_t* total_out;
  __device__ uint32_t n() const { return n_words; }
  __device__ uint32_t value(uint32_t i) const { return (uint32_t)__popc(bits[i]); }
  __device__ void emit(uint32_t i, uint32_t ex, uint32_t) const { wprefix[i] = ex; }
  __device__ void total(int, uint32_t t) const { *total_out = t; }
};
// nframes == nullptr (mode B, merged table): the slot already carries the size of the stack's first occurrence
__global__ void __launch_bounds__(kThreads) k_stack_assign(StackSlot* tab, const uint32_t* claimed, const uint32_t* n_claimed, const uint32_t* rowbits,
                                                           const uint32_t* wprefix, const uint16_t* nframes, uint32_t* uniq_row, uint32_t* uniq_slot,
                                                           uint32_t* uniq_size) {
  const uint32_t n = *n_claimed;
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
    uint32_t sidx = claimed[i];
    uint32_t f = 0xFFFFFFFFu - tab[sidx].first_inv;
    uint32_t ord = wprefix[f >> 5] + (uint32_t)__popc(rowbits[f >> 5] & ((1u << (f & 31)) - 1u));
    uniq_row[ord] = f;
    tab[sidx].ordinal = ord;
    uniq_slot[ord] = sidx;
    uniq_size[ord] = nframes ? (uint32_t)nframes[f] : tab[sidx].size;
  }
}
struct UniqOffsetF {  // startOffset := indices.Len() at each first occurrence (arrow_v2.go:302)
  typedef unsigned long long T;
  const Counters* ctr;
  Counters* ctr_w;
  const uint32_t* uniq_size;
  const uint32_t* uniq_slot;
  StackSlot* tab;
  __device__ uint32_t n() const { return ctr->n_unique; }
  __device__ unsigned long long value(uint32_t u) const { return uniq_size[u]; }
  __device__ void emit(uint32_t u, unsigned long long ex, unsigned long long v) const {
    StackSlot* e = &tab[uniq_slot[u]];
    e->offset = (uint32_t)ex;
    e->size = (uint32_t)v;
  }
  __device__ void total(int, unsigned long long t) const {
    ctr_w->n_indices64 = t;
    if (t > 0x7FFFFFFFull) atomicOr(&ctr_w->err, ERR_INDEX_OVERFLOW);  // ListView offsets are int32 (arrow_v2.go:233)
  }
};

// (2) per-row ListView offset/size: hit => reuse the first occurrence's (offset,size) (arrow_v2.go:293-299)
// v2: the ListView (offset, size) of each row; v1 (ord_out != nullptr): the row's stack ordinal, which is
// both the run key and the dictionary index of the stacktrace_id column.
__global__ void __launch_bounds__(kThreads) k_rows_materialize(uint32_t n_rows, const uint32_t* slot_of_row, const StackSlot* tab,
                                                               int* st_offsets, int* st_sizes, uint32_t* ord_out) {
  const uint32_t stride = gridDim.x * kThreads * 4;
  for (uint32_t base = blockIdx.x * kThreads * 4; base < n_rows; base += stride) {
    uint32_t sl[4];
    uint2 os[4];
    uint32_t od[4];
#pragma unroll
    for (int u = 0; u < 4; u++) { uint32_t r = base + u * kThreads + threadIdx.x; sl[u] = r < n_rows ? slot_of_row[r] : kNull; }
#pragma unroll
    for (int u = 0; u < 4; u++) {
      if (ord_out) od[u] = sl[u] != kNull ? tab[sl[u]].ordinal : 0u;
      else os[u] = sl[u] != kNull ? *reinterpret_cast<const uint2*>(&tab[sl[u]].offset) : make_uint2(0u, 0u);
    }
#pragma unroll
    for (int u = 0; u < 4; u++) {
      uint32_t r = base + u * kThreads + threadIdx.x;
      if (r >= n_rows) continue;
      if (ord_out) ord_out[r] = od[u];
      else { st_offsets[r] = (int)os[u].x; st_sizes[r] = (int)os[u].y; }
    }
  }
}
// v1: dictionary values of the stacktrace_id column = the 16-byte ids of the unique stacks in ordinal order
__global__ void __launch_bounds__(kThreads) k_gather_ids(const Counters* ctr, const uint32_t* uniq_row, const uint8_t* uuid, uint8_t* out, int* offsets) {
  uint32_t nu = ctr->n_unique;
  for (uint32_t u = blockIdx.x * kThreads + threadIdx.x; u <= nu; u += gridDim.x * kThreads) {
    offsets[u] = (int)(16u * u);
    if (u < nu) *reinterpret_cast<ulonglong2*>(out + 16ull * u) = *reinterpret_cast<const ulonglong2*>(uuid + 16ull * uniq_row[u]);
  }
}
// v1: dictionary order of the kind-derived string columns. A class enters a column's dictionary at the first
// row whose kind maps to it; with at most 7 kinds this is a one-warp job.
__global__ void k_kind_ranks(const uint32_t* first_kind, const uint32_t* kindtab, uint32_t* kindrank, uint32_t* kind_order, uint32_t* n_kind_dict) {
  int t = threadIdx.x;  // one thread per kind-derived column (6 string columns)
  if (t >= 6) return;
  uint32_t first_class[8];
  for (int c = 0; c < 8; c++) { first_class[c] = kNull; kind_order[t * 8 + c] = kNull; }
  if (t < 2) {  // rows 6,7 (period, duration) are not dictionary encoded: keep them defined
    for (int c = 0; c < 8; c++) { kindrank[(6 + t) * 8 + c] = kNull; kind_order[(6 + t) * 8 + c] = kNull; }
    n_kind_dict[6 + t] = 0;
  }
  for (int k = 0; k < 7; k++) {
    uint32_t c = kindtab[t * 8 + k];
    if (c != kNull && first_kind[k] < first_class[c]) first_class[c] = first_kind[k];
  }
  uint32_t n = 0;
  for (int c = 0; c < 8; c++) {
    kindrank[t * 8 + c] = kNull;
    if (first_class[c] == kNull) continue;
    uint32_t r = 0;
    for (int o = 0; o < 8; o++) r += (first_class[o] < first_class[c]) ? 1u : 0u;
    kindrank[t * 8 + c] = r;
    kind_order[t * 8 + r] = (uint32_t)c;
    n++;
  }
  n_kind_dict[t] = n;
}

// On-demand side table: occurrences per unique stack, in first-occurrence order (the reference emits one
// row per sample and never counts — SURVEY section 0.2 — so this stays off the flush path). Lanes of a
// warp that hit the same stack are aggregated before the atomicAdd.
__global__ void __launch_bounds__(kThreads) k_count_stacks(uint32_t n_rows, const uint32_t* slot_of_row, const StackSlot* tab, uint32_t* counts) {
  const unsigned full = 0xFFFFFFFFu;
  uint32_t stride = gridDim.x * kThreads, iters = (n_rows + stride - 1) / stride;
  int lane = threadIdx.x & 31;
  for (uint32_t it = 0; it < iters; it++) {
    uint32_t r = it * stride + blockIdx.x * kThreads + threadIdx.x;
    uint32_t sl = r < n_rows ? slot_of_row[r] : kNull;
    unsigned grp = __match_any_sync(full, sl);
    if (sl != kNull && lane == __ffs(grp) - 1) atomicAdd(&counts[tab[sl].ordinal], (uint32_t)__popc(grp));
  }
}

// (3) gather the frames of the unique stacks, in first-occurrence order, into the location-index
// stream and record each frame's first position (appendLocationV2 dedup key = the frame, :421)
// `frames` holds uint64 ids, or uint32 ids when the top bit of n_frames_registered's companion flag is set (narrow ring)
__device__ __forceinline__ unsigned long long frame_at(const unsigned long long* frames, unsigned long long i, uint32_t narrow) {
  return narrow ? (unsigned long long)reinterpret_cast<const uint32_t*>(frames)[i] : frames[i];
}
__global__ void __launch_bounds__(kThreads) k_gather_unique(const Counters* ctr, const uint32_t* uniq_row, const uint32_t* slot_of_row,
                                                            const StackSlot* tab, const unsigned long long* frames,
                                                            const unsigned long long* frame_off, uint32_t n_frames_registered,
                                                            uint32_t* ustream, uint32_t* loc_first, Counters* ctr_w, uint32_t narrow) {
  uint32_t nu = ctr->n_unique;
  int lane = threadIdx.x & 31;
  uint32_t warp = (blockIdx.x * kThreads + threadIdx.x) >> 5, nwarps = (gridDim.x * kThreads) >> 5;
  for (uint32_t u = warp; u < nu; u += nwarps) {
    uint32_t r = uniq_row[u];
    StackSlot e = tab[slot_of_row[r]];
    const unsigned long long base = frame_off[r];
    for (uint32_t jx = lane; jx < e.size; jx += 32) {
      unsigned long long fid = frame_at(frames, base + jx, narrow);
      uint32_t pos = e.offset + jx;
      if (fid >= n_frames_registered) { atomicOr(&ctr_w->err, ERR_BAD_FRAME_ID); fid = 0; }
      ustream[pos] = (uint32_t)fid;
      if (loc_first[(uint32_t)fid] > pos) atomicMin(&loc_first[(uint32_t)fid], pos);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// first-occurrence ranking of 32-bit keys (dictionary index assignment). Batched: blockIdx.y = job.
//   min    : first[key] = min position            (element-sized; fused into the producer where possible)
//   bits   : bitmap[first[key]] = 1 for every present key         (table-sized)
//   words  : exclusive popcount prefix over the bitmap words      (n/32-sized)
//   assign : rank[key] = prefix + popc(below), order[rank] = key  (table-sized)
//   map    : out[i] = rank[keys[i]] (+ validity bitmap)           (element-sized)
struct FoJob {
  const uint32_t* keys;
  const uint32_t* n_ptr;   // element count lives on the device (nullptr: use n_imm)
  const uint32_t* n_map_ptr;  // mode B: elements THIS shard maps (its slice of the stream); nullptr = the same count
  uint32_t n_imm;
  uint32_t* first;         // direct: [universe] first position (memset 0xFF)
  unsigned long long* hslots;  // hashed: (key<<32 | first position), memset 0xFF
  uint32_t hmask;
  uint32_t hashed;
  uint32_t universe;       // direct table entries
  uint32_t nullable;       // keys == kNull are nulls (skipped, mapped to index 0 + validity 0)
  uint32_t skip_min;       // first[] already filled by a producer kernel
  uint32_t* rank;          // direct: [universe], hashed: [hmask+1]
  uint32_t* order;         // [n_unique] key by rank
  uint32_t* out;           // [n] rank per element (may alias keys); nullptr = skip
  uint32_t* validity;      // [ceil(n/32)] bitmap words; nullptr = skip
  uint32_t* bitmap;        // [ceil(n_max/32)+1] zeroed
  uint32_t* wprefix;       // [ceil(n_max/32)+1]
  uint32_t* n_unique;      // -> Counters
  uint32_t* n_null;        // -> Counters (may be nullptr)
  Counters* ctr;
};
__device__ __forceinline__ uint32_t gtid() { return blockIdx.x * kThreads + threadIdx.x; }
__device__ __forceinline__ uint32_t gstride() { return gridDim.x * kThreads; }

__global__ void __launch_bounds__(kThreads) k_fo_min(const FoJob* jobs) {
  const FoJob& j = jobs[blockIdx.y];
  if (j.skip_min) return;
  uint32_t n = j.n_ptr ? *j.n_ptr : j.n_imm;
  for (uint32_t i = gtid(); i < n; i += gstride()) {
    uint32_t key = j.keys[i];
    if (j.nullable && key == kNull) continue;
    if (j.first[key] > i) atomicMin(&j.first[key], i);  // hashed jobs (thread ids) record first rows in k_header
  }
}
__global__ void __launch_bounds__(kThreads) k_fo_zero(const FoJob* jobs) {  // clear only the bitmap words this batch will use
  const FoJob& j = jobs[blockIdx.y];
  uint32_t nw = (j.n_ptr ? *j.n_ptr : j.n_imm) / 32 + 1;
  for (uint32_t i = gtid(); i < nw; i += gstride()) j.bitmap[i] = 0u;
}
__global__ void __launch_bounds__(kThreads) k_fo_bits(const FoJob* jobs) {
  const FoJob& j = jobs[blockIdx.y];
  uint32_t entries = j.hashed ? j.hmask + 1 : j.universe;
  for (uint32_t e = gtid(); e < entries; e += gstride()) {
    uint32_t f;
    if (j.hashed) { unsigned long long sl = j.hslots[e]; if (sl == ~0ull) continue; f = (uint32_t)sl; }
    else { f = j.first[e]; if (f == kNull) continue; }
    atomicOr(&j.bitmap[f >> 5], 1u << (f & 31));
  }
}
struct FoWordsF {
  typedef uint32_t T;
  const FoJob* jobs;
  int sel;  // >= 0: that job; < 0: blockIdx.y (stand-alone batched kernels)
  __device__ const FoJob& J() const { return jobs[sel >= 0 ? sel : (int)blockIdx.y]; }
  __device__ uint32_t n() const { const FoJob& j = J(); return ((j.n_ptr ? *j.n_ptr : j.n_imm) + 31) / 32; }
  __device__ uint32_t value(uint32_t i) const { return (uint32_t)__popc(J().bitmap[i]); }
  __device__ void emit(uint32_t i, uint32_t ex, uint32_t) const { J().wprefix[i] = ex; }
  __device__ void total(int job, uint32_t t) const { *jobs[sel >= 0 ? sel : job].n_unique = t; }
};
__global__ void __launch_bounds__(kThreads) k_fo_assign(const FoJob* jobs) {
  const FoJob& j = jobs[blockIdx.y];
  uint32_t entries = j.hashed ? j.hmask + 1 : j.universe;
  for (uint32_t e = gtid(); e < entries; e += gstride()) {
    uint32_t f, key;
    if (j.hashed) { unsigned long long sl = j.hslots[e]; if (sl == ~0ull) continue; f = (uint32_t)sl; key = (uint32_t)(sl >> 32); }
    else { f = j.first[e]; if (f == kNull) continue; key = e; }
    uint32_t r = j.wprefix[f >> 5] + (uint32_t)__popc(j.bitmap[f >> 5] & ((1u << (f & 31)) - 1u));
    j.rank[e] = r;
    j.order[r] = key;
  }
}
// element -> dictionary index (+ validity bitmap, null count). Four independent elements per thread
// keep enough loads in flight.
__global__ void __launch_bounds__(kThreads) k_fo_map(const FoJob* jobs) {
  const FoJob& j = jobs[blockIdx.y];
  if (!j.out) return;
  uint32_t n = j.n_map_ptr ? *j.n_map_ptr : (j.n_ptr ? *j.n_ptr : j.n_imm), begin, end;
  block_range(n, &begin, &end);
  uint32_t nulls = 0;
  for (uint32_t tile = begin; tile < end; tile += 4 * kThreads) {
    uint32_t key[4], val[4];
    bool valid[4];
#pragma unroll
    for (int u = 0; u < 4; u++) {
      uint32_t i = tile + u * kThreads + threadIdx.x;
      key[u] = i < end ? j.keys[i] : kNull;
      valid[u] = i < end && !(j.nullable && key[u] == kNull);
    }
#pragma unroll
    for (int u = 0; u < 4; u++) val[u] = valid[u] ? j.rank[j.hashed ? fo_hfind(j.hslots, j.hmask, key[u]) : key[u]] : 0u;
#pragma unroll
    for (int u = 0; u < 4; u++) {
      uint32_t i = tile + u * kThreads + threadIdx.x;
      if (i < end) { j.out[i] = val[u]; nulls += valid[u] ? 0u : 1u; }
      unsigned bits = __ballot_sync(0xFFFFFFFFu, valid[u]);
      if (j.validity && (threadIdx.x & 31) == 0 && (i & ~31u) < end) j.validity[i >> 5] = bits;
    }
  }
  if (j.n_null) {
    for (int d = 16; d > 0; d >>= 1) nulls += __shfl_down_sync(0xFFFFFFFFu, nulls, d);
    if ((threadIdx.x & 31) == 0 && nulls) atomicAdd(j.n_null, nulls);
  }
}

// ---------------------------------------------------------------------------------------------
// location dictionary: resolved per-frame attributes gathered in location order
struct FrameTable {  // device copy of the registered, pre-resolved frames (see agg.cu resolve_frame)
  const unsigned long long* addr;
  const uint32_t* type_cid;
  const uint32_t* map_cid;
  const uint32_t* bid_cid;   // kNull = null
  const unsigned long long* line;
  const uint32_t* func;      // kNull = no line (native / oomprof)
};
struct LocOut {
  unsigned long long* address;  // Arrow: location.address
  uint32_t* type_key;
  uint32_t* map_key;
  uint32_t* bid_key;
  int* line_off;                // Arrow: lines ListView offsets
  int* line_size;               // Arrow: lines ListView sizes
  uint32_t* line_valid;         // Arrow: lines validity words
  unsigned long long* line_no;  // Arrow: line.line
  uint32_t* func_key;
};
struct LocLinesF {  // scan of has_line over locations (lineListOffsets, parca_reporter.go:428)
  typedef uint32_t T;
  const Counters* ctr;
  Counters* ctr_w;
  const uint32_t* loc_order;
  FrameTable ft;
  LocOut o;
  __device__ uint32_t n() const { return ctr->n_locations; }
  __device__ uint32_t value(uint32_t i) const { return ft.func[loc_order[i]] != kNull; }
  __device__ void emit(uint32_t i, uint32_t ex, uint32_t v) const {
    uint32_t fid = loc_order[i];
    o.address[i] = ft.addr[fid];
    o.type_key[i] = ft.type_cid[fid];
    o.map_key[i] = ft.map_cid[fid];
    o.bid_key[i] = ft.bid_cid[fid];
    o.line_off[i] = (int)ex;
    o.line_size[i] = (int)v;
    if (v) { o.line_no[ex] = ft.line[fid]; o.func_key[ex] = ft.func[fid]; }
  }
  __device__ void total(int, uint32_t t) const { ctr_w->n_lines = t; }
};
// validity words of the lines ListView (null where the location has no line, arrow_v2.go:403-418)
__global__ void __launch_bounds__(kThreads) k_line_validity(const Counters* ctr, const int* line_size, uint32_t* words) {
  uint32_t n = ctr->n_locations;
  uint32_t nw = (n + 31) / 32;
  int lane = threadIdx.x & 31;
  uint32_t warp = (blockIdx.x * kThreads + threadIdx.x) >> 5, nwarps = (gridDim.x * kThreads) >> 5;
  for (uint32_t w = warp; w < nw; w += nwarps) {
    uint32_t i = w * 32 + lane;
    unsigned bits = __ballot_sync(0xFFFFFFFFu, i < n && line_size[i] > 0);
    if (lane == 0) words[w] = bits;
  }
}
// function table in function-dictionary order: filename keys for the nested dictionary
__global__ void __launch_bounds__(kThreads) k_func_keys(const Counters* ctr, const uint32_t* func_order, const uint32_t* fn_file_cid, uint32_t* file_key) {
  uint32_t n = ctr->n_functions;
  for (uint32_t k = blockIdx.x * kThreads + threadIdx.x; k < n; k += gridDim.x * kThreads) file_key[k] = fn_file_cid[func_order[k]];
}


// The label column plan of the batch, checked and applied at the head of the label chain. For every labelset the batch names
// (first_ls != kNull, recorded by k_header; in a merged batch all-reduced over the shards) a warp gives it a row of the key
// matrix [used labelsets][planned columns], which KeyLs reaches through rank[], and walks its (name ordinal, value id) pairs:
// each name sets its bit in the used-name bitmap; a planned one writes its value id into the row and lowers the first row of
// its value (min over the labelsets carrying it of the labelset's first row); an unplanned one raises ERR_LABEL_PLAN, and the
// host redoes the pass with exactly the used names planned. Rows are handed out by an atomic counter: the matrix is only an
// indirection, so their order does not reach the output. Planned columns ascend by ordinal (binary search in shared memory).
struct LsPlanArgs {
  const uint32_t* first_ls; uint32_t n_labelsets;
  const uint32_t* off; const uint2* pairs;  // the registered labelsets: pairs [off[ls], off[ls + 1]) of (name ordinal, value id)
  uint32_t n_cols;                          // planned labelset-derived columns (the key matrix's row length)
  uint32_t* rank;                           // [labelset] -> row of the key matrix (used labelsets only)
  uint32_t* keys;                           // [row][n_cols] -> value id or kNull
  uint32_t* n_used;                         // rows handed out (zeroed)
  uint32_t* used_names;                     // bitmap over the name ordinals (zeroed)
  Counters* ctr;
  uint32_t plan_ord[kMaxCols];              // name ordinal of each planned column, ascending
  uint32_t* col_first[kMaxCols];            // first-row table of each planned column, by value id
};
__global__ void __launch_bounds__(kThreads) k_ls_plan(LsPlanArgs a) {
  __shared__ uint32_t s_ord[kMaxCols];
  for (uint32_t i = threadIdx.x; i < a.n_cols; i += kThreads) s_ord[i] = a.plan_ord[i];
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31;
  bool miss = false;
  // 32 consecutive labelsets per warp and step: the trip count is uniform in the warp (the ballot needs all of it)
  for (uint32_t base = blockIdx.x * kThreads + (threadIdx.x & ~31u); base < a.n_labelsets; base += gridDim.x * kThreads) {
    const uint32_t ls = base + lane;
    const uint32_t f = ls < a.n_labelsets ? a.first_ls[ls] : kNull;
    const uint32_t used = __ballot_sync(0xFFFFFFFFu, f != kNull);
    if (!used) continue;
    uint32_t row0 = 0;
    if (lane == 0) row0 = atomicAdd(a.n_used, (uint32_t)__popc(used));
    row0 = __shfl_sync(0xFFFFFFFFu, row0, 0);
    if (a.n_cols) {  // the warp's rows start all null (consecutive rows: coalesced stores)
      uint32_t* rows = a.keys + (size_t)row0 * a.n_cols;
      const uint32_t cells = (uint32_t)__popc(used) * a.n_cols;
      for (uint32_t i = lane; i < cells; i += 32) rows[i] = kNull;
    }
    __syncwarp();
    if (f != kNull) {
      const uint32_t row = row0 + (uint32_t)__popc(used & ((1u << lane) - 1u));
      a.rank[ls] = row;
      uint32_t* keys = a.keys + (size_t)row * a.n_cols;
      for (uint32_t p = a.off[ls], e = a.off[ls + 1]; p < e; p++) {
        const uint2 kv = a.pairs[p];
        uint32_t* w = &a.used_names[kv.x >> 5];
        const uint32_t bit = 1u << (kv.x & 31);
        if (!(*w & bit)) atomicOr(w, bit);
        uint32_t lo = 0, hi = a.n_cols;
        while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (s_ord[mid] < kv.x) lo = mid + 1; else hi = mid; }
        if (lo < a.n_cols && s_ord[lo] == kv.x) {
          keys[lo] = kv.y;
          uint32_t* fp = a.col_first[lo] + kv.y;
          if (*fp > f) atomicMin(fp, f);
        } else {
          miss = true;
        }
      }
    }
  }
  if (miss) atomicOr(&a.ctr->err, ERR_LABEL_PLAN);
}

// ---------------------------------------------------------------------------------------------
// run-end encoding of every REE column in two fused passes over the rows
// (label columns: reporter/arrow.go:97-131; constant-ish columns: arrow.go:50-59,:166-207).
// Rows are partitioned into one contiguous range per WARP, so neither pass needs a block barrier:
// the previous row's inputs come from the neighbouring lane (shuffle) or are carried across steps.
// Column order is fixed by the host: [labelset-derived LS columns][cpu][thread_id][thread_name][8 kind columns].
enum : uint32_t { COL_LS = 0, COL_CPU = 1, COL_TID = 2, COL_COMM = 3, COL_KIND = 4, COL_ORD = 5, COL_TS = 6 };
struct ReeCol {
  uint32_t type, param;
  int* run_ends;       // Arrow: run_ends child
  uint32_t* run_keys;  // key of each run (kNull = null run)
  uint32_t* first;     // dictionary first-ROW table (direct), filled by k_header / k_ls_plan
  unsigned long long* hslots;  // hashed variant (thread_id): (key << 32 | first row)
  uint32_t hmask;
  uint32_t nullable;
  const uint32_t* rank;  // dictionary index per key (direct) / per slot (hashed), ready before the emit pass
  uint32_t* validity;    // Arrow validity words of the run values (zeroed; only for nullable columns)
};
struct ReeArgs {
  uint32_t n_rows, ncols;
  uint32_t n_ls;                 // LS columns are 0..n_ls-1
  int c_cpu, c_tid, c_comm;      // column index or -1
  uint32_t c_kind;               // first of the 8 kind columns
  const ReeCol* cols;
  const uint32_t* ls; const uint32_t* cpu; const uint32_t* tid; const uint32_t* comm; const uint8_t* kind;
  const uint32_t* ls_rank;                    // [labelset] -> row of ls_keys (k_ls_plan)
  const uint32_t* ls_keys; uint32_t n_lscols; // [row][LS column] -> value id or kNull
  const uint32_t* kindtab;                    // [8][8] -> class id or kNull
  uint32_t* partial;                          // [ncols][total warps]
  Counters* ctr;
  // v1 schema only (nullptr / -1 otherwise)
  const uint32_t* ord;       // stack ordinal per row -> stacktrace_id column (run key == dictionary index)
  const long long* ts;       // timestamp per row -> run-end encoded int64 column
  long long* ts_vals;        // value of every timestamp run
  int c_ord, c_ts;
  const uint32_t* kindrank;  // [6][8] class -> dictionary index of the kind-derived string columns
  uint32_t kind_dict_mask;   // bit t: kind column t is dictionary encoded
  // mode B (one merged batch over several shards): this shard's rows are the global rows row_base .. row_base+n_rows-1
  uint32_t row_base;         // added to every run end
  unsigned long long* edge_keys;  // [ncols][4] = first key, first null, last key, last null of this shard (count pass); nullptr = off
  const struct MergeCol* mc; // per column: how many local runs stay in this shard's part + validity bit shift (emit pass); nullptr = off
};
struct EdgeCol {   // what one shard contributes to the cross-shard run merge of one REE column
  uint32_t n_runs, n_null, lastnn, n_rows;
  unsigned long long first_key, last_key;  // 64 bits: the v1 timestamp column's keys are int64
  uint32_t first_null, last_null;
};
struct MergeCol {
  uint32_t keep;       // local runs that stay in this shard's part: n_runs, or n_runs-1 when its last run continues in the next shard
  uint32_t vshift;     // (global index of this shard's first run) mod 32: validity bits are written at their global bit position
  uint32_t runbase;    // global index of this shard's first run
  uint32_t pad;
};
__device__ __forceinline__ void warp_range(uint32_t n, uint32_t* begin, uint32_t* end, uint32_t* wg) {
  uint32_t nw = gridDim.x * kWarps;
  uint32_t w = blockIdx.x * kWarps + (threadIdx.x >> 5);
  uint32_t per = (n + nw - 1) / nw;
  per = (per + 31) / 32 * 32;
  unsigned long long b = (unsigned long long)w * per, e = b + per;
  *begin = b < n ? (uint32_t)b : n;
  *end = e < n ? (uint32_t)e : n;
  *wg = w;
}
// EMIT = false: count boundaries per (column, warp) and track the last row carrying each label.
// EMIT = true : write run ends / final dictionary indices / validity bits at their final positions.
// Column-parallel: blockIdx.y selects a column group, so a warp encodes ONE
// column (or the 8 kind-derived columns, which share their skip test) over its row range with all of its
// state in registers, and different columns progress concurrently on different warps instead of being
// walked one after the other inside every row step.
struct ReeGroup { uint32_t type, col, param; };
struct ReeGroups { uint32_t n; ReeGroup g[kMaxCols]; };

constexpr int kReeUnroll = 4;  // 32-row sub-steps per iteration: their key loads / rank lookups are in flight together
constexpr int kReeBlocksPerSm = 8;  // grid of the two run-end passes: they are latency-bound, so they fill every warp slot

template <bool EMIT, bool MERGED, class KeyT, class K>
__device__ __forceinline__ void ree_single(const ReeArgs& a, uint32_t c, bool has_dict, K kf) {
  const unsigned full = 0xFFFFFFFFu;
  const int lane = threadIdx.x & 31;
  uint32_t begin, end, wg;
  warp_range(a.n_rows, &begin, &end, &wg);
  const uint32_t nwarps = gridDim.x * kWarps;
  const ReeCol col = a.cols[c];
  uint32_t acc = EMIT ? a.partial[c * nwarps + wg] : 0u, last = 0, nulls = 0;
  const uint32_t keep = (EMIT && MERGED) ? a.mc[c].keep : 0xFFFFFFFFu, vshift = (EMIT && MERGED) ? a.mc[c].vshift : 0u;  // single aggregator: folded away
  KeyT ckey = 0; bool cnull = true;                 // previous row of lane 0
  if (begin < end && begin > 0) kf.get(begin - 1, ckey, cnull);
  const unsigned lt = (1u << lane) - 1u;
  for (uint32_t base = begin; base < end; base += 32 * kReeUnroll) {
    KeyT key[kReeUnroll]; bool null[kReeUnroll], in[kReeUnroll], bnd[kReeUnroll];
    unsigned m[kReeUnroll];
#pragma unroll
    for (int u = 0; u < kReeUnroll; u++) {
      const uint32_t r = base + u * 32 + lane;
      in[u] = r < end; key[u] = 0; null[u] = true;
      if (in[u]) kf.get(r, key[u], null[u]);
      if (!EMIT && MERGED && in[u]) {
        if (r == 0) { a.edge_keys[c * 4 + 0] = (unsigned long long)key[u]; a.edge_keys[c * 4 + 1] = null[u] ? 1u : 0u; }
        if (r + 1 == a.n_rows) { a.edge_keys[c * 4 + 2] = (unsigned long long)key[u]; a.edge_keys[c * 4 + 3] = null[u] ? 1u : 0u; }
      }
    }
#pragma unroll
    for (int u = 0; u < kReeUnroll; u++) {
      const uint32_t r = base + u * 32 + lane;
      KeyT pk = __shfl_up_sync(full, key[u], 1); int pn = __shfl_up_sync(full, (int)null[u], 1);
      if (lane == 0) { pk = ckey; pn = cnull; }
      bnd[u] = in[u] && (r == 0 || null[u] || pn || pk != key[u]);
      m[u] = __ballot_sync(full, bnd[u]);
      ckey = __shfl_sync(full, key[u], 31); cnull = __shfl_sync(full, (int)null[u], 31);
    }
    if (!EMIT) {
#pragma unroll
      for (int u = 0; u < kReeUnroll; u++) {
        acc += (uint32_t)__popc(m[u]);
        unsigned nn = __ballot_sync(full, in[u] && !null[u]);
        if (nn) last = base + u * 32 + (32 - __clz(nn));
        nulls += (uint32_t)__popc(__ballot_sync(full, bnd[u] && null[u]));
      }
    } else {
      uint32_t k[kReeUnroll], stored[kReeUnroll];
      uint32_t run = acc;
#pragma unroll
      for (int u = 0; u < kReeUnroll; u++) { k[u] = run + (uint32_t)__popc(m[u] & lt); run += (uint32_t)__popc(m[u]); }
#pragma unroll
      for (int u = 0; u < kReeUnroll; u++) {  // all dictionary lookups of the iteration are issued before any is consumed
        stored[u] = (uint32_t)key[u];
        if (has_dict && bnd[u]) stored[u] = null[u] ? 0u : col.rank[col.hslots ? fo_hfind(col.hslots, col.hmask, (uint32_t)key[u]) : (uint32_t)key[u]];
      }
#pragma unroll
      for (int u = 0; u < kReeUnroll; u++) {
        if (bnd[u]) {
          if (k[u] > 0) col.run_ends[k[u] - 1] = (int)((MERGED ? a.row_base : 0u) + base + u * 32 + lane);  // run k starts here => run k-1 ends here
          if (!MERGED || k[u] < keep) { if (sizeof(KeyT) == 8) a.ts_vals[k[u]] = (long long)key[u]; else col.run_keys[k[u]] = stored[u]; }
        }
      }
      if (col.validity && col.nullable) {  // validity bits of the runs emitted by one sub-step span at most two words
        uint32_t pos = acc + vshift;
#pragma unroll
        for (int u = 0; u < kReeUnroll; u++) {
          if (m[u]) {
            const uint32_t w0 = pos >> 5, kb = k[u] + vshift;
            const bool v = bnd[u] && !null[u] && (!MERGED || k[u] < keep);
            unsigned m0 = __reduce_or_sync(full, (v && (kb >> 5) == w0) ? (1u << (kb & 31)) : 0u);
            unsigned m1 = __reduce_or_sync(full, (v && (kb >> 5) != w0) ? (1u << (kb & 31)) : 0u);
            if (lane == 0) { if (m0) atomicOr(&col.validity[w0], m0); if (m1) atomicOr(&col.validity[w0 + 1], m1); }
          }
          pos += (uint32_t)__popc(m[u]);
        }
      }
      acc = run;
    }
  }
  if (!EMIT && lane == 0) {
    a.partial[c * nwarps + wg] = acc;
    if (last) atomicMax(&a.ctr->last_nonnull_plus1[c], last);
    if (nulls) atomicAdd(&a.ctr->n_null[c], nulls);
  }
}
struct KeyLs { const uint32_t* ls; const uint32_t* rank; const uint32_t* keys; uint32_t stride, c;
  __device__ __forceinline__ void get(uint32_t r, uint32_t& k, bool& n) const { k = __ldg(&keys[(size_t)__ldg(&rank[ls[r]]) * stride + c]); n = k == kNull; } };
struct KeyU32 { const uint32_t* v;
  __device__ __forceinline__ void get(uint32_t r, uint32_t& k, bool& n) const { k = v[r]; n = false; } };
struct KeyComm { const uint32_t* v;  // labels.Builder.Set(name, "") deletes the label: "" => null
  __device__ __forceinline__ void get(uint32_t r, uint32_t& k, bool& n) const { k = v[r]; n = k == 0; } };
struct KeyTs { const long long* v;
  __device__ __forceinline__ void get(uint32_t r, long long& k, bool& n) const { k = v[r]; n = false; } };

// the 8 kind-derived columns: one warp, eight running positions in registers, one skip test per step
template <bool EMIT, bool MERGED>
__device__ __forceinline__ void ree_kinds(const ReeArgs& a, const uint32_t* s_kind, const uint32_t* s_krank) {
  const unsigned full = 0xFFFFFFFFu;
  const int lane = threadIdx.x & 31;
  uint32_t begin, end, wg;
  warp_range(a.n_rows, &begin, &end, &wg);
  const uint32_t nwarps = gridDim.x * kWarps;
  uint32_t acc[8], nulls[8];
#pragma unroll
  for (int t = 0; t < 8; t++) { acc[t] = EMIT ? a.partial[(a.c_kind + t) * nwarps + wg] : 0u; nulls[t] = 0; }
  uint32_t ckind = 0;
  if (begin < end && begin > 0) ckind = a.kind[begin - 1];
  uint32_t nk = (begin + lane < end) ? a.kind[begin + lane] : 0u;
  const unsigned lt = (1u << lane) - 1u;
  for (uint32_t base = begin; base < end; base += 32) {
    const uint32_t r = base + lane;
    const bool in = r < end;
    const uint32_t kind = nk;
    if (r + 32 < end) nk = a.kind[r + 32];
    uint32_t pkind = __shfl_up_sync(full, kind, 1);
    if (lane == 0) pkind = ckind;
    const bool first_row = r == 0;
    if (!EMIT && MERGED && in && (first_row || r + 1 == a.n_rows)) {
#pragma unroll
      for (int t = 0; t < 8; t++) {
        const uint32_t v = s_kind[t * 8 + kind];
        if (first_row) { a.edge_keys[(a.c_kind + t) * 4 + 0] = v; a.edge_keys[(a.c_kind + t) * 4 + 1] = v == kNull ? 1u : 0u; }
        if (r + 1 == a.n_rows) { a.edge_keys[(a.c_kind + t) * 4 + 2] = v; a.edge_keys[(a.c_kind + t) * 4 + 3] = v == kNull ? 1u : 0u; }
      }
    }
    const bool kchange = in && (first_row || kind != pkind || kind >= 3u);  // kinds >= 3 carry a null temporality
    if (__ballot_sync(full, kchange)) {
#pragma unroll
      for (int t = 0; t < 8; t++) {
        uint32_t v = s_kind[t * 8 + kind], pv = s_kind[t * 8 + pkind];
        const bool null = v == kNull;
        const bool boundary = in && (first_row || null || pv == kNull || pv != v);
        const unsigned m = __ballot_sync(full, boundary);
        if (!EMIT) {
          acc[t] += (uint32_t)__popc(m);
          nulls[t] += (uint32_t)__popc(__ballot_sync(full, boundary && null));
        } else if (m) {
          const ReeCol& col = a.cols[a.c_kind + t];
          const uint32_t k = acc[t] + (uint32_t)__popc(m & lt);
          const uint32_t keep = MERGED ? a.mc[a.c_kind + t].keep : 0xFFFFFFFFu, vshift = MERGED ? a.mc[a.c_kind + t].vshift : 0u;
          if ((a.kind_dict_mask >> t) & 1u) v = null ? 0u : s_krank[t * 8 + v];  // v1: dictionary index of the class
          if (boundary) {
            if (k > 0) col.run_ends[k - 1] = (int)((MERGED ? a.row_base : 0u) + r);
            if (!MERGED || k < keep) col.run_keys[k] = v;
          }
          if (col.validity && col.nullable) {
            const uint32_t w0 = (acc[t] + vshift) >> 5, kb = k + vshift;
            const bool ok = boundary && !null && (!MERGED || k < keep);
            unsigned m0 = __reduce_or_sync(full, (ok && (kb >> 5) == w0) ? (1u << (kb & 31)) : 0u);
            unsigned m1 = __reduce_or_sync(full, (ok && (kb >> 5) != w0) ? (1u << (kb & 31)) : 0u);
            if (lane == 0) { if (m0) atomicOr(&col.validity[w0], m0); if (m1) atomicOr(&col.validity[w0 + 1], m1); }
          }
          acc[t] += (uint32_t)__popc(m);
        }
      }
    }
    ckind = __shfl_sync(full, kind, 31);
  }
  if (!EMIT && lane == 0) {
#pragma unroll
    for (int t = 0; t < 8; t++) {
      a.partial[(a.c_kind + t) * nwarps + wg] = acc[t];
      if (nulls[t]) atomicAdd(&a.ctr->n_null[a.c_kind + t], nulls[t]);
    }
  }
}

template <bool EMIT, bool MERGED>
__global__ void __launch_bounds__(kThreads) k_ree_col(ReeArgs a, ReeGroups groups) {
  __shared__ uint32_t s_kind[64], s_krank[64];
  const ReeGroup g = groups.g[blockIdx.y];
  if (g.type == COL_KIND) {
    if (threadIdx.x < 64) { s_kind[threadIdx.x] = a.kindtab[threadIdx.x]; s_krank[threadIdx.x] = (EMIT && a.kindrank && threadIdx.x < 48) ? a.kindrank[threadIdx.x] : 0u; }
    __syncthreads();
    ree_kinds<EMIT, MERGED>(a, s_kind, s_krank);
    return;
  }
  switch (g.type) {
    case COL_LS: ree_single<EMIT, MERGED, uint32_t>(a, g.col, true, KeyLs{a.ls, a.ls_rank, a.ls_keys, a.n_lscols, g.param}); break;
    case COL_CPU: ree_single<EMIT, MERGED, uint32_t>(a, g.col, true, KeyU32{a.cpu}); break;
    case COL_TID: ree_single<EMIT, MERGED, uint32_t>(a, g.col, true, KeyU32{a.tid}); break;
    case COL_COMM: ree_single<EMIT, MERGED, uint32_t>(a, g.col, true, KeyComm{a.comm}); break;
    case COL_ORD: ree_single<EMIT, MERGED, uint32_t>(a, g.col, false, KeyU32{a.ord}); break;  // bytes.Equal on the 16-byte id
    default: ree_single<EMIT, MERGED, long long>(a, g.col, false, KeyTs{a.ts}); break;           // COL_TS: Int64RunEndBuilder.Append
  }
}
__global__ void __launch_bounds__(kThreads) k_ree_scan_partials(ReeArgs a, int g, uint32_t col0) {  // grid = columns col0 .., kThreads threads
  const uint32_t c = col0 + blockIdx.x;
  uint32_t* p = a.partial + (size_t)c * g;
  uint32_t run = 0;
  for (int base = 0; base < g; base += kThreads) {  // block-wide exclusive scan, kThreads partials per round
    int i = base + threadIdx.x;
    uint32_t v = i < g ? p[i] : 0u, tot;
    uint32_t ex = block_exclusive_scan(v, &tot);
    if (i < g) p[i] = run + ex;
    run += tot;
  }
  if (threadIdx.x == 0) {
    a.ctr->n_runs[c] = run;
    if (run) a.cols[c].run_ends[run - 1] = (int)(a.row_base + a.n_rows);  // the last run ends at the (shard's last global) row count
  }
}

// ---------------------------------------------------------------------------------------------
// v1 schema: device-resident store of known stacks — the `stacks` LRU of the reference
// (reporter/parca_reporter.go:105; `Get` then `Add` per sample at :224-227, `Get` per requested id in buildStacktraceRecord :1555).
// An LRU's content after any access sequence is the `capacity` distinct keys accessed most recently, so the store keeps, per
// entry, the time of its last access —
//     stamp = epoch << 32 | position      epoch: one per ingested batch and per stacktrace request
//                                         position: LAST row of the stack in the batch / index of the id in the request
// — and after every batch drops all but the `capacity` largest stamps (radix select + k_store_kill). stamp 0 = evicted: the slot
// and its frames stay until the next compaction (k_store_rebuild) or until the stack is seen again (it is then revived in place).
// What is NOT reference behaviour: the frame arena is finite (pa_agg_config.stack_cache_frames); running out of it clears the
// store as a whole (an evicted stack and a never-seen one both produce the reference's "missing stacktrace" row).
struct __align__(32) StoreSlot {
  Key128 key;              // (0,0) = empty; claimed by a 128-bit CAS
  unsigned long long off;  // first frame in the store's frame arena
  uint32_t size;           // frames; kNull = claimed but dropped (no room)
  uint32_t claimed;        // only used by the dedicated all-zero-id slot (index mask+1)
};
struct StoreCtl { unsigned long long used_frames; uint32_t entries; uint32_t live; };  // entries: claimed slots (live + evicted)

__device__ __forceinline__ uint32_t store_find(const StoreSlot* st, uint32_t mask, Key128 k) {
  if (key_zero(k)) return st[mask + 1].claimed ? mask + 1 : kNull;
  uint32_t idx = mix_slot(k) & mask;
  for (uint32_t probe = 0; probe <= mask; probe++) {
    Key128 cur = st[idx].key;
    if (key_eq(cur, k)) return idx;
    if (key_zero(cur)) return kNull;  // never deleted from: an empty slot ends the cluster
    idx = (idx + 1) & mask;
  }
  return kNull;
}

struct StoreInsertArgs {
  const Counters* ctr;
  const uint32_t* uniq_row;
  const uint32_t* slot_of_row;
  const StackSlot* tab;
  const uint16_t* nframes;
  const unsigned long long* frame_off;
  const unsigned long long* frames;  // device copy, or the mapped pinned ring in provided-hash mode
  uint32_t narrow;                   // the frame stream holds uint32 ids
  uint32_t n_frames_registered;
  StoreSlot* st;
  uint32_t mask;
  uint32_t* arena;
  unsigned long long cap_frames;
  uint32_t cap_entries;              // physical: claimed slots the table may hold
  StoreCtl* ctl;
  Counters* ctr_w;
  unsigned long long* stamp;         // [mask + 2] last access per slot, 0 = evicted
  const uint32_t* last_row;          // [batch table slots] last row of every stack of the batch
  unsigned long long epoch_hi;       // epoch << 32
  uint32_t min_last_p1;              // only stacks with last_row + 1 >= this are stored (a batch with more unique stacks than the cache holds)
  // merged batch (k_store_insert<true>): the merged dictionary instead of this shard's rows, indexed by merged ordinal
  const StackSlot* gtab;             // merged table: key and depth of the global first occurrence
  const uint32_t* g_slot;            // [U] merged table slot of every ordinal
  const uint32_t* g_last_inv;        // [U] 0xFFFFFFFF - global last row
  const uint32_t* g_frames;          // frames of the stacks the store lacks, gathered from the shards that hold their first occurrence
  const unsigned long long* g_foff;  // [U + 1] where each ordinal's frames start in g_frames (an ordinal without frames there: equal neighbours)
  // k_store_insert<true, true> (PA_CFG_GROUP_STACKS): g_foff indexes g_refs instead, one entry per stack. Each is a handle, resolved
  // through this member's own records (g_recs) into its own registered arena (`frames`): the handles are the same on every member,
  // but the arenas may be laid out differently (PA_CFG_GROUP_RETIRE: compactions at different points of the registrations)
  const unsigned long long* g_refs;  // handle of each needed stack, from its global first occurrence
  const uint4* g_recs;               // RegStack records, two uint4 each
  uint32_t n_recs;
};
// last occurrence of every stack of the batch (the LRU's access time of its entry)
__global__ void __launch_bounds__(kThreads) k_last_rows(uint32_t n_rows, const uint32_t* slot_of_row, uint32_t* last_row) {
  // from the last row down: the first visit of a stack is (nearly always) its last row, every earlier row then fails the plain
  // comparison and issues no atomic
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n_rows; i += gridDim.x * kThreads) {
    const uint32_t r = n_rows - 1u - i;
    const uint32_t s = slot_of_row[r];
    if (s != kNull && last_row[s] < r) atomicMax(&last_row[s], r);
  }
}
// stamps of the batch's unique stacks as select keys (last row + 1, so that 0 stays "nothing")
__global__ void __launch_bounds__(kThreads) k_batch_stamps(const Counters* ctr, const uint32_t* uniq_row, const uint32_t* slot_of_row, const uint32_t* last_row,
                                                           unsigned long long* out) {
  const uint32_t nu = ctr->n_unique;
  for (uint32_t u = blockIdx.x * kThreads + threadIdx.x; u < nu; u += gridDim.x * kThreads) out[u] = (unsigned long long)last_row[slot_of_row[uniq_row[u]]] + 1ull;
}
// one radix-select pass: histogram of byte `shift / 8` over the non-zero keys whose higher bytes equal `prefix`
__global__ void __launch_bounds__(kThreads) k_select_hist(const unsigned long long* keys, uint64_t n, unsigned long long prefix, int shift, uint32_t* hist) {
  __shared__ uint32_t h[256];
  if (threadIdx.x < 256) h[threadIdx.x] = 0;
  __syncthreads();
  const unsigned long long hi_mask = shift >= 56 ? 0ull : (~0ull << (shift + 8));
  for (uint64_t i = (uint64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (uint64_t)gridDim.x * kThreads) {
    const unsigned long long k = keys[i];
    if (k != 0 && (k & hi_mask) == prefix) atomicAdd(&h[(k >> shift) & 0xFFu], 1u);
  }
  __syncthreads();
  if (threadIdx.x < 256 && h[threadIdx.x]) atomicAdd(&hist[threadIdx.x], h[threadIdx.x]);
}
// evict: every entry accessed before `threshold`
__global__ void __launch_bounds__(kThreads) k_store_kill(unsigned long long* stamp, uint64_t n, unsigned long long threshold, StoreCtl* ctl) {
  uint32_t killed = 0;
  for (uint64_t i = (uint64_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (uint64_t)gridDim.x * kThreads) {
    const unsigned long long k = stamp[i];
    if (k != 0 && k < threshold) { stamp[i] = 0; killed++; }
  }
  for (int o = 16; o > 0; o >>= 1) killed += __shfl_xor_sync(0xFFFFFFFFu, killed, o);
  if ((threadIdx.x & 31) == 0 && killed) atomicSub(&ctl->live, killed);
}
// one warp per unique stack of the batch (unique within the launch, so a key is claimed by at most one warp).
// MERGED: one replica of a merge group's store; u is the merged ordinal, frames come from the gathered buffer.
// REFS (with MERGED): frames come from the member's registered arena; the gathered handle (g_refs) names the member's own record
// (g_recs), which gives the offset.
template <bool MERGED, bool REFS = false>
__global__ void __launch_bounds__(kThreads) k_store_insert(StoreInsertArgs a) {
  const unsigned full = 0xFFFFFFFFu;
  uint32_t nu = a.ctr->n_unique;
  int lane = threadIdx.x & 31;
  uint32_t warp = (blockIdx.x * kThreads + threadIdx.x) >> 5, nwarps = (gridDim.x * kThreads) >> 5;
  const Key128 zero{0ull, 0ull};
  for (uint32_t u = warp; u < nu; u += nwarps) {
    uint32_t r = 0, size, lr;
    if constexpr (MERGED) {
      size = a.gtab[a.g_slot[u]].size;
      lr = 0xFFFFFFFFu - a.g_last_inv[u];
    } else {
      r = a.uniq_row[u];
      size = a.nframes[r];
      lr = a.last_row[a.slot_of_row[r]];
    }
    unsigned long long off = 0;
    int fresh = 0;
    if (lr + 1u < a.min_last_p1) continue;  // warp-uniform: older than everything the cache will hold after this batch
    if (lane == 0) {
      Key128 k = MERGED ? a.gtab[a.g_slot[u]].key : a.tab[a.slot_of_row[r]].key;
      uint32_t idx = kNull;
      if (key_zero(k)) {
        idx = a.mask + 1;
        fresh = atomicCAS(&a.st[idx].claimed, 0u, 1u) == 0u;
      } else {
        uint32_t p = mix_slot(k) & a.mask;
        for (uint32_t probe = 0; probe <= a.mask; probe++) {
          Key128 cur = ld_key(&a.st[p].key);
          if (cur.hi == 0 || cur.lo == 0) cur = cas128(&a.st[p].key, zero, k);
          if (key_zero(cur)) { idx = p; fresh = 1; break; }
          if (key_eq(cur, k)) { idx = p; break; }
          p = (p + 1) & a.mask;
        }
      }
      if (idx == kNull) {  // the table itself is full
        atomicOr(&a.ctr_w->store_overflow, 1u);
      } else if (fresh || a.st[idx].size == kNull || a.stamp[idx] == 0) {
        // new key; or one that was claimed when there was no room for its frames; or an evicted one, which the reference would Add
        // again with the frames of THIS interval's first sample carrying the id (they differ from the old ones only when two
        // stacks share a provided id) — its old frames are garbage until the next compaction
        const bool was_claimed = !fresh;
        uint32_t e = was_claimed ? 0u : atomicAdd(&a.ctl->entries, 1u);
        off = atomicAdd(&a.ctl->used_frames, (unsigned long long)size);
        if (e >= a.cap_entries || off + size > a.cap_frames) {
          a.st[idx].size = kNull;
          atomicOr(&a.ctr_w->store_overflow, 1u);
          fresh = 0;
        } else {
          a.st[idx].off = off;
          a.st[idx].size = size;
          a.stamp[idx] = a.epoch_hi | lr;
          atomicAdd(&a.ctl->live, 1u);
          fresh = 1;
        }
      } else {  // known and alive: refresh the access time
        a.stamp[idx] = a.epoch_hi | lr;
      }
    }
    fresh = __shfl_sync(full, fresh, 0);
    if (!fresh) continue;
    off = __shfl_sync(full, off, 0);
    if constexpr (MERGED && REFS) {
      const unsigned long long k = a.g_foff[u];
      if (a.g_foff[u + 1] - k != (size ? 1u : 0u)) {  // not in the gathered set: a logic error, reported instead of storing garbage
        if (lane == 0) atomicOr(&a.ctr_w->err, ERR_MERGE_LOOKUP);
        continue;
      }
      unsigned long long base = size ? a.g_refs[k] : 0ull;
      if (size) {  // the sender's k_header accepted this handle in this batch, so a mismatch here is a logic error
        const uint32_t slot = (uint32_t)base, gen = (uint32_t)(base >> 32);
        const uint4 s1 = slot < a.n_recs ? __ldg(a.g_recs + 2ull * slot + 1) : make_uint4(0u, 0u, 0u, kStackFree);
        if (s1.w != gen || (gen & kStackFree) || s1.z != size) {
          if (lane == 0) atomicOr(&a.ctr_w->err, ERR_MERGE_LOOKUP);
          continue;
        }
        base = ((unsigned long long)s1.y << 32) | s1.x;
      }
      for (uint32_t j = lane; j < size; j += 32) {
        unsigned long long fid = frame_at(a.frames, base + j, a.narrow);
        if (fid >= a.n_frames_registered) { atomicOr(&a.ctr_w->err, ERR_BAD_FRAME_ID); fid = 0; }
        a.arena[off + j] = (uint32_t)fid;
      }
    } else if constexpr (MERGED) {  // the frames were checked where they were packed (k_store_pack)
      const unsigned long long base = a.g_foff[u];
      if (a.g_foff[u + 1] - base != size) {  // not in the gathered set: a logic error, reported instead of storing garbage
        if (lane == 0) atomicOr(&a.ctr_w->err, ERR_MERGE_LOOKUP);
        continue;
      }
      for (uint32_t j = lane; j < size; j += 32) a.arena[off + j] = a.g_frames[base + j];
    } else {
      const unsigned long long base = a.frame_off[r];
      for (uint32_t j = lane; j < size; j += 32) {
        unsigned long long fid = frame_at(a.frames, base + j, a.narrow);
        if (fid >= a.n_frames_registered) { atomicOr(&a.ctr_w->err, ERR_BAD_FRAME_ID); fid = 0; }
        a.arena[off + j] = (uint32_t)fid;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// v1 stacktrace record (buildStacktraceRecord, parca_reporter.go:1545-1739): requested ids -> flattened
// locations -> lines, every column of LocationsWriter (arrow.go:209-254) built by scans and gathers.
// compaction: the live entries of one store into an empty one (one warp per old slot)
struct StoreRebuildArgs {
  const StoreSlot* old_st; const unsigned long long* old_stamp; const uint32_t* old_arena; uint32_t old_mask;
  StoreSlot* st; unsigned long long* stamp; uint32_t* arena; uint32_t mask; StoreCtl* ctl;
};
__global__ void __launch_bounds__(kThreads) k_store_rebuild(StoreRebuildArgs a) {
  const unsigned full = 0xFFFFFFFFu;
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * kThreads + threadIdx.x) >> 5, nwarps = (gridDim.x * kThreads) >> 5;
  const Key128 zero{0ull, 0ull};
  for (uint32_t i = warp; i <= a.old_mask + 1; i += nwarps) {
    const unsigned long long stp = a.old_stamp[i];
    const uint32_t size = a.old_st[i].size;
    if (stp == 0 || size == kNull) continue;  // warp-uniform
    if (i <= a.old_mask && key_zero(a.old_st[i].key)) continue;
    unsigned long long off = 0;
    if (lane == 0) {
      uint32_t idx;
      if (i == a.old_mask + 1) { idx = a.mask + 1; a.st[idx].claimed = 1u; }
      else {
        const Key128 k = a.old_st[i].key;
        uint32_t p = mix_slot(k) & a.mask;
        for (;;) {  // the new table has room for every live entry
          Key128 cur = cas128(&a.st[p].key, zero, k);
          if (key_zero(cur)) break;
          p = (p + 1) & a.mask;
        }
        idx = p;
      }
      atomicAdd(&a.ctl->entries, 1u);
      atomicAdd(&a.ctl->live, 1u);
      off = atomicAdd(&a.ctl->used_frames, (unsigned long long)size);
      a.st[idx].off = off;
      a.st[idx].size = size;
      a.stamp[idx] = stp;
    }
    off = __shfl_sync(full, off, 0);
    const unsigned long long src = a.old_st[i].off;
    for (uint32_t j = lane; j < size; j += 32) a.arena[off + j] = a.old_arena[src + j];
  }
}
__global__ void __launch_bounds__(kThreads) k_st_lookup(const uint8_t* ids, uint32_t n, const StoreSlot* st, uint32_t mask, uint32_t* q_slot,
                                                        uint32_t* q_nloc, unsigned long long* stamp, unsigned long long epoch_hi) {
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
    ulonglong2 raw = *reinterpret_cast<const ulonglong2*>(ids + 16ull * i);  // libpf.TraceHashFromBytes: big-endian hi||lo
    Key128 k{bswap64(raw.x), bswap64(raw.y)};
    uint32_t sl = store_find(st, mask, k);
    if (sl != kNull && (st[sl].size == kNull || stamp[sl] == 0)) sl = kNull;  // dropped for lack of room / evicted
    if (sl != kNull) atomicMax(&stamp[sl], epoch_hi | i);                     // r.stacks.Get moves the entry to the front (:1555)
    q_slot[i] = sl;
    q_nloc[i] = sl == kNull ? 1u : st[sl].size;  // a missing stack still yields one placeholder location (:1556-1573)
  }
}
struct StLocF {  // LocationsList offsets: exclusive scan of the per-stack location counts
  typedef unsigned long long T;
  const uint32_t* q_nloc;
  uint32_t n_ids;
  int* loc_off;
  Counters* ctr_w;
  __device__ uint32_t n() const { return n_ids; }
  __device__ unsigned long long value(uint32_t i) const { return q_nloc[i]; }
  __device__ void emit(uint32_t i, unsigned long long ex, unsigned long long) const { loc_off[i] = (int)ex; }
  __device__ void total(int, unsigned long long t) const {
    loc_off[n_ids] = (int)t;
    ctr_w->n_indices64 = t;
    ctr_w->n_locations = (uint32_t)t;
    if (t > 0x7FFFFFFFull) atomicOr(&ctr_w->err, ERR_INDEX_OVERFLOW);  // List offsets are int32
  }
};
struct FrameTableV1 {  // device mirror of FrameTableHost's v1 columns
  const unsigned long long* addr;
  const uint32_t* type_cid;
  const uint32_t* map_cid;
  const uint32_t* bid_cid;
  const uint32_t* fn_cid;    // kNull = no line
  const uint32_t* file_cid;
  const unsigned long long* line;
  const unsigned long long* col;
  const uint8_t* complete;
};
// one warp per requested stack: its frames' ids in location order, is_complete, list validity
__global__ void __launch_bounds__(kThreads) k_st_expand(uint32_t n_ids, const uint32_t* q_slot, const int* loc_off, const StoreSlot* st,
                                                        const uint32_t* arena, const uint8_t* frame_complete, uint32_t* loc_fid,
                                                        uint8_t* complete, uint8_t* list_valid, Counters* ctr_w) {
  const unsigned full = 0xFFFFFFFFu;
  int lane = threadIdx.x & 31;
  uint32_t warp = (blockIdx.x * kThreads + threadIdx.x) >> 5, nwarps = (gridDim.x * kThreads) >> 5;
  for (uint32_t i = warp; i < n_ids; i += nwarps) {
    uint32_t sl = q_slot[i];
    uint32_t base = (uint32_t)loc_off[i];
    if (sl == kNull) {
      if (lane == 0) { loc_fid[base] = kNull; complete[i] = 0; list_valid[i] = 1; }
      continue;
    }
    unsigned long long off = st[sl].off;
    uint32_t size = st[sl].size;
    int ok = 1;
    for (uint32_t j = lane; j < size; j += 32) {
      uint32_t fid = arena[off + j];
      loc_fid[base + j] = fid;
      ok &= (int)frame_complete[fid];
    }
    ok = __all_sync(full, ok);
    if (lane == 0) {
      complete[i] = (uint8_t)ok;
      list_valid[i] = size != 0;  // LocationsList.Append(false) for an empty trace (:1576-1580)
      if (size == 0) atomicAdd(&ctr_w->st_null_lists, 1u);
    }
  }
}
// bytes (0/1) -> Arrow bitmap words; n may live on the device
__global__ void __launch_bounds__(kThreads) k_pack_bits(const uint8_t* src, const uint32_t* n_ptr, uint32_t n_imm, uint32_t* words) {
  uint32_t n = n_ptr ? *n_ptr : n_imm;
  uint32_t nw = (n + 31) / 32;
  int lane = threadIdx.x & 31;
  uint32_t warp = (blockIdx.x * kThreads + threadIdx.x) >> 5, nwarps = (gridDim.x * kThreads) >> 5;
  for (uint32_t w = warp; w < nw; w += nwarps) {
    uint32_t i = w * 32 + lane;
    unsigned bits = __ballot_sync(0xFFFFFFFFu, i < n && src[i] != 0);
    if (lane == 0) words[w] = bits;
  }
}
struct StLocOut {
  unsigned long long* address;
  uint32_t* type_key;
  uint32_t* map_key;   // kNull = null
  uint32_t* bid_key;   // kNull = null
  int* line_off;       // [L+1]
  uint8_t* has_line;   // lines validity source
  long long* line_no;
  unsigned long long* column;
  uint32_t* fn_key;
  uint32_t* file_key;  // kNull = null
};
struct StLinesF {  // per-location gather fused into the scan that assigns the Lines offsets
  typedef uint32_t T;
  const Counters* ctr;
  Counters* ctr_w;
  const uint32_t* loc_fid;
  FrameTableV1 ft;
  StLocOut o;
  uint32_t unknown_type_cid, missing_fn_cid;
  __device__ uint32_t n() const { return ctr->n_locations; }
  __device__ uint32_t value(uint32_t i) const { uint32_t fid = loc_fid[i]; return fid == kNull ? 1u : (ft.fn_cid[fid] != kNull ? 1u : 0u); }
  __device__ void emit(uint32_t i, uint32_t ex, uint32_t v) const {
    uint32_t fid = loc_fid[i];
    o.line_off[i] = (int)ex;
    o.has_line[i] = (uint8_t)v;
    if (fid == kNull) {  // the "missing stacktrace" placeholder (:1557-1571)
      o.address[i] = 0ull; o.type_key[i] = unknown_type_cid; o.map_key[i] = kNull; o.bid_key[i] = kNull;
      o.line_no[ex] = 0ll; o.column[ex] = 0ull; o.fn_key[ex] = missing_fn_cid; o.file_key[ex] = kNull;
      return;
    }
    o.address[i] = ft.addr[fid]; o.type_key[i] = ft.type_cid[fid]; o.map_key[i] = ft.map_cid[fid]; o.bid_key[i] = ft.bid_cid[fid];
    if (v) { o.line_no[ex] = (long long)ft.line[fid]; o.column[ex] = ft.col[fid]; o.fn_key[ex] = ft.fn_cid[fid]; o.file_key[ex] = ft.file_cid[fid]; }
  }
  __device__ void total(int, uint32_t t) const { ctr_w->n_lines = t; o.line_off[n()] = (int)t; }
};
// run-end encoding of a materialised key column (BinaryDictionaryRunEndBuilder, arrow.go:97-131): a run starts
// at row 0, at every null (AppendNull always opens a run) and wherever the key changes. blockIdx.y = column.
struct StRunCol { const uint32_t* keys; const uint32_t* n_ptr; uint32_t* run_key; int* run_end; };
struct StRunF {
  typedef uint32_t T;
  StRunCol c[4];
  Counters* ctr_w;
  __device__ uint32_t n() const { return *c[blockIdx.y].n_ptr; }
  __device__ uint32_t value(uint32_t i) const {
    const uint32_t* k = c[blockIdx.y].keys;
    uint32_t cur = k[i];
    return (i == 0 || cur == kNull || cur != k[i - 1]) ? 1u : 0u;
  }
  __device__ void emit(uint32_t i, uint32_t ex, uint32_t v) const {
    if (!v) return;
    const StRunCol& col = c[blockIdx.y];
    col.run_key[ex] = col.keys[i];
    if (ex) col.run_end[ex - 1] = (int)i;
  }
  __device__ void total(int job, uint32_t t) const {
    ctr_w->n_runs[job] = t;
    if (t) c[job].run_end[t - 1] = (int)*c[job].n_ptr;
  }
};


// ---------------------------------------------------------------------------------------------
// On-demand side table: occurrences per (labelset, stack) pair, in first-occurrence order. Like k_count_stacks this
// is NOT part of the reference's record (one row per sample, nothing is counted: SURVEY section 0.2); it is the
// "hash-and-count" view of the same batch for callers that want pprof-style aggregated samples. Open addressing on the
// 64-bit pair, warp-aggregated: lanes carrying the same pair elect their lowest lane (== lowest row), which does one
// table walk, one atomicMax (first row) and one atomicAdd (group size) for the whole group.
struct __align__(16) PairSlot {
  unsigned long long key;  // ((labelset << 32) | stack ordinal) + 1; 0 = empty
  uint32_t first_inv;      // 0xFFFFFFFF - first row
  uint32_t count;
};
__global__ void __launch_bounds__(kThreads) k_pair_count(uint32_t n_rows, const uint32_t* ls, const uint32_t* slot_of_row, const StackSlot* tab,
                                                         PairSlot* pt, uint32_t pmask, uint32_t* overflow) {
  const unsigned full = 0xFFFFFFFFu;
  uint32_t stride = gridDim.x * kThreads, iters = (n_rows + stride - 1) / stride;
  int lane = threadIdx.x & 31;
  for (uint32_t it = 0; it < iters; it++) {
    uint32_t r = it * stride + blockIdx.x * kThreads + threadIdx.x;
    bool valid = r < n_rows;
    unsigned long long key = 0ull;
    if (valid) {
      uint32_t sl = slot_of_row[r];
      key = (((unsigned long long)ls[r] << 32) | (sl != kNull ? tab[sl].ordinal : 0u)) + 1ull;
    }
    unsigned grp = __match_any_sync(full, key);
    if (!valid || lane != __ffs(grp) - 1) continue;
    uint32_t idx = mix_slot(Key128{key, key >> 32}) & pmask;
    bool placed = false;
    for (uint32_t probe = 0; probe <= pmask; probe++) {
      unsigned long long cur = pt[idx].key;
      if (cur == 0ull) cur = atomicCAS(&pt[idx].key, 0ull, key);
      if (cur == 0ull || cur == key) { placed = true; break; }
      idx = (idx + 1) & pmask;
    }
    if (!placed) { atomicOr(overflow, 1u); continue; }
    atomicMax(&pt[idx].first_inv, 0xFFFFFFFFu - r);
    atomicAdd(&pt[idx].count, (uint32_t)__popc(grp));
  }
}
__global__ void __launch_bounds__(kThreads) k_pair_bits(const PairSlot* pt, uint32_t nslots, uint32_t* rowbits) {
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < nslots; i += gridDim.x * kThreads) {
    if (pt[i].key == 0ull) continue;
    uint32_t f = 0xFFFFFFFFu - pt[i].first_inv;
    atomicOr(&rowbits[f >> 5], 1u << (f & 31));
  }
}
__global__ void __launch_bounds__(kThreads) k_pair_emit(const PairSlot* pt, uint32_t nslots, const uint32_t* rowbits, const uint32_t* wprefix,
                                                        uint32_t cap, uint32_t* out_ls, uint32_t* out_stack, uint32_t* out_count) {
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < nslots; i += gridDim.x * kThreads) {
    PairSlot e = pt[i];
    if (e.key == 0ull) continue;
    uint32_t f = 0xFFFFFFFFu - e.first_inv;
    uint32_t ord = wprefix[f >> 5] + (uint32_t)__popc(rowbits[f >> 5] & ((1u << (f & 31)) - 1u));
    if (ord >= cap) continue;
    unsigned long long pair = e.key - 1ull;
    out_ls[ord] = (uint32_t)(pair >> 32);
    out_stack[ord] = (uint32_t)pair;
    out_count[ord] = e.count;
  }
}


// ---------------------------------------------------------------------------------------------
// Multi-GPU mode B (one merged batch, SURVEY section 8e): every shard hashes and deduplicates its own rows, then
// exports (1) its rows as 64-byte headers that carry the computed stack id and point at (2) the frames of its
// UNIQUE stacks only. The merging GPU receives 64 B per row plus U*F*8 B per shard over NVLink and runs the
// provided-id pipeline on the union in global row order, so every dictionary comes out in the order the
// reference would produce on the unsharded stream.
__global__ void __launch_bounds__(kThreads) k_shard_export_rows(uint32_t n_rows, const uint4* hdr_in, const uint8_t* uuid, const uint32_t* slot_of_row,
                                                                const StackSlot* tab, unsigned long long frame_base, uint4* hdr_out) {
  for (uint32_t r = blockIdx.x * kThreads + threadIdx.x; r < n_rows; r += gridDim.x * kThreads) {
    const uint4* h = hdr_in + 4ull * r;
    uint4 q1 = __ldg(h + 1), q2 = __ldg(h + 2), q3 = __ldg(h + 3);
    ulonglong2 id = *reinterpret_cast<const ulonglong2*>(uuid + 16ull * r);  // big-endian hi||lo
    unsigned long long hi = bswap64(id.x), lo = bswap64(id.y);
    uint32_t sl = slot_of_row[r];
    StackSlot e = tab[sl];
    unsigned long long foff = frame_base + e.offset;  // every row of a stack points at the shard's single copy of its frames
    uint4 q0 = make_uint4((uint32_t)hi, (uint32_t)(hi >> 32), (uint32_t)lo, (uint32_t)(lo >> 32));
    q3.x = (uint32_t)foff;
    q3.y = (uint32_t)(foff >> 32);
    q3.w = (q3.w & 0xFFFF0000u) | (e.size & 0xFFFFu);  // nframes of the stack's first occurrence (what the record keeps)
    uint4* o = hdr_out + 4ull * r;
    o[0] = q0; o[1] = q1; o[2] = q2; o[3] = q3;
  }
}
// frames of the unique stacks, first-occurrence order, as frame ids again (the location ranking rewrote the
// gathered stream in place with location indices; loc_order maps an index back to its frame id)
__global__ void __launch_bounds__(kThreads) k_shard_export_frames(const Counters* ctr, const uint32_t* ustream, const uint32_t* loc_order,
                                                                  unsigned long long* out) {
  const uint32_t n = (uint32_t)ctr->n_indices64;
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) out[i] = loc_order[ustream[i]];
}

// merging GPU: rows of one shard -> their positions in the global order, written straight into the staging buffer
// (four threads per 64-byte row: coalesced reads, one full row per scattered write)
__global__ void __launch_bounds__(kThreads) k_scatter_rows(const uint4* src, const unsigned long long* global_row, unsigned long long n_rows,
                                                           unsigned long long n_total, uint4* dst, uint32_t* bad) {
  const unsigned long long n4 = n_rows * 4ull;
  for (unsigned long long t = (unsigned long long)blockIdx.x * kThreads + threadIdx.x; t < n4; t += (unsigned long long)gridDim.x * kThreads) {
    unsigned long long g = global_row[t >> 2];
    if (g >= n_total) { *bad = 1u; continue; }
    dst[g * 4ull + (t & 3ull)] = __ldg(src + t);
  }
}


// ---------------------------------------------------------------------------------------------
// Multi-GPU mode B, dictionary merge (SURVEY section 8e; the "slices" form): the merged batch is the reference's record for
// the stream [shard 0's rows, shard 1's rows, ...], i.e. shard m's local row r is global row row_base_m + r. Rows never
// leave their shard. What is exchanged is O(unique keys):
//   stacks    : every shard sends (id, global first row, depth) of its unique stacks to the id's owner shard
//               (hash of the id mod G: one all-to-all), owners keep the minimum row, the owners' lists are all-gathered
//               and every shard ranks the merged list the usual way (first-row bitmap -> popcount prefix);
//   locations : first positions in the merged unique-stack frame stream, one all-reduce(min) over the frame-indexed table;
//   labels    : all-reduce(min) over the direct first-row tables, all-gather of the thread-id lists;
//   run ends  : per column (run count, first/last key) of every shard, all-gathered; neighbouring runs merge at shard edges.
// Because global rows ascend with the shard index, the stacks whose first occurrence is in shard m occupy one contiguous
// range of ordinals, hence one contiguous range of the location-index stream: shard m gathers exactly that range.
struct __align__(8) StackEntry { unsigned long long hi, lo; uint32_t row, size; };  // 24 B on the wire

__device__ __forceinline__ uint32_t owner_of(Key128 k, uint32_t world) {
  unsigned long long x = k.hi ^ rotl64(k.lo, 23);
  x ^= x >> 29; x *= 0xBF58476D1CE4E5B9ull; x ^= x >> 32;
  return (uint32_t)(x % world);
}
struct OwnerOffsets { uint32_t off[kMaxWorld + 1]; };
// pass 1: entries per owner
__global__ void __launch_bounds__(kThreads) k_owner_count(const StackSlot* tab, const uint32_t* claimed, const uint32_t* n_claimed, uint32_t world, uint32_t* cnt) {
  __shared__ uint32_t s_cnt[kMaxWorld];
  if (threadIdx.x < kMaxWorld) s_cnt[threadIdx.x] = 0;
  __syncthreads();
  const uint32_t n = *n_claimed;
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) atomicAdd(&s_cnt[owner_of(tab[claimed[i]].key, world)], 1u);
  __syncthreads();
  if (threadIdx.x < world && s_cnt[threadIdx.x]) atomicAdd(&cnt[threadIdx.x], s_cnt[threadIdx.x]);
}
// pass 2: (id, global first row, depth of that first occurrence), bucketed by owner (order inside a bucket is irrelevant)
__global__ void __launch_bounds__(kThreads) k_owner_pack(const StackSlot* tab, const uint32_t* claimed, const uint32_t* n_claimed, uint32_t world,
                                                         OwnerOffsets offs, uint32_t* cursor, uint32_t row_base, const uint16_t* nframes, StackEntry* out) {
  const uint32_t n = *n_claimed;
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
    const StackSlot e = tab[claimed[i]];
    const uint32_t f = 0xFFFFFFFFu - e.first_inv, o = owner_of(e.key, world);
    out[offs.off[o] + atomicAdd(&cursor[o], 1u)] = StackEntry{e.key.hi, e.key.lo, row_base + f, (uint32_t)nframes[f]};
  }
}
// owner / merged table insert: keeps, per id, the entry with the smallest global row (its depth rides along: both live in
// one 64-bit word, inverted row in the high half, so a single atomicMax decides)
__device__ __forceinline__ unsigned long long* slot_minpack(StackSlot* e) { return reinterpret_cast<unsigned long long*>(&e->first_inv); }
__global__ void __launch_bounds__(kThreads) k_entries_insert(const StackEntry* in, uint32_t n, StackSlot* tab, uint32_t mask, uint32_t* ctl /*n_claimed, zero_claimed, err*/,
                                                             uint32_t* claimed) {
  const TabCtl tc{ctl, ctl + 1, ctl + 2};
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
    const StackEntry en = in[i];
    const uint32_t idx = stack_find_or_insert(tab, mask, Key128{en.hi, en.lo}, tc, claimed);
    if (idx == kNull) continue;
    const unsigned long long pack = ((unsigned long long)(0xFFFFFFFFu - en.row) << 32) | en.size;
    unsigned long long* mp = slot_minpack(&tab[idx]);
    if (*(volatile unsigned long long*)mp < pack) atomicMax(mp, pack);
  }
}
// owner table -> list of its (deduplicated) entries
__global__ void __launch_bounds__(kThreads) k_entries_compact(const StackSlot* tab, const uint32_t* claimed, const uint32_t* n_claimed, StackEntry* out) {
  const uint32_t n = *n_claimed;
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
    StackSlot e = tab[claimed[i]];
    const unsigned long long pack = *slot_minpack(&e);
    out[i] = StackEntry{e.key.hi, e.key.lo, 0xFFFFFFFFu - (uint32_t)(pack >> 32), (uint32_t)pack};
  }
}
// merged table: minpack -> the regular slot fields (first_inv = inverted global first row, size) so that the ranking kernels
// (k_stack_bits / k_stack_assign / UniqOffsetF) run on it unchanged
__global__ void __launch_bounds__(kThreads) k_merged_unpack(StackSlot* tab, const uint32_t* claimed, const uint32_t* n_claimed) {
  const uint32_t n = *n_claimed;
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
    StackSlot* e = &tab[claimed[i]];
    const unsigned long long pack = *slot_minpack(e);
    e->first_inv = (uint32_t)(pack >> 32);
    e->ordinal = 0;
    e->size = (uint32_t)pack;
  }
}
// every local unique stack takes (ordinal, offset, size) of the merged dictionary
__global__ void __launch_bounds__(kThreads) k_local_adopt(StackSlot* ltab, const uint32_t* lclaimed, const uint32_t* n_lclaimed, const StackSlot* gtab, uint32_t gmask,
                                                          const uint32_t* gctl, uint32_t* err) {
  const uint32_t n = *n_lclaimed, zero_present = gctl[1];
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
    StackSlot* e = &ltab[lclaimed[i]];
    const uint32_t g = stack_find(gtab, gmask, e->key, zero_present);
    if (g == kNull) { atomicOr(err, ERR_MERGE_LOOKUP); continue; }
    e->ordinal = gtab[g].ordinal; e->offset = gtab[g].offset; e->size = gtab[g].size;
  }
}
// which ordinals (a contiguous range, see above) have their first occurrence in this shard, and the stream range they cover
struct MergeCtl { uint32_t ord0, ord1, off0, slice_len; uint32_t n_tids, pad[3]; };
__global__ void k_won_range(const uint32_t* uniq_row, const uint32_t* uniq_slot, const StackSlot* gtab, const Counters* ctr, uint32_t row_base, uint32_t n_rows,
                            uint32_t ustream_cap, MergeCtl* mc, Counters* ctr_w) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const uint32_t nu = ctr->n_unique;
  auto lower = [&](unsigned long long row) { uint32_t lo = 0, hi = nu; while (lo < hi) { uint32_t mid = (lo + hi) >> 1; if (uniq_row[mid] < row) lo = mid + 1; else hi = mid; } return lo; };
  const uint32_t o0 = lower(row_base), o1 = lower((unsigned long long)row_base + n_rows);
  const unsigned long long total = ctr->n_indices64;
  const unsigned long long f0 = o0 < nu ? gtab[uniq_slot[o0]].offset : total, f1 = o1 < nu ? gtab[uniq_slot[o1]].offset : total;
  mc->ord0 = o0; mc->ord1 = o1; mc->off0 = (uint32_t)f0; mc->slice_len = (uint32_t)(f1 - f0);
  if (f1 - f0 > ustream_cap) { atomicOr(&ctr_w->err, ERR_SLICE_CAP); mc->slice_len = 0; mc->ord1 = o0; }
}
// this shard's range of the merged unique-stack frame stream (frame ids; mapped to location indices in place later) and the
// first GLOBAL position of every frame it contains
__global__ void __launch_bounds__(kThreads) k_gather_won(const MergeCtl* mc, const uint32_t* uniq_row, const uint32_t* uniq_slot, const StackSlot* gtab, uint32_t row_base,
                                                         const unsigned long long* frames, const unsigned long long* frame_off, uint32_t n_frames_registered,
                                                         uint32_t* ustream, uint32_t* loc_first, Counters* ctr_w, uint32_t narrow) {
  const uint32_t o0 = mc->ord0, o1 = mc->ord1, off0 = mc->off0;
  int lane = threadIdx.x & 31;
  uint32_t warp = (blockIdx.x * kThreads + threadIdx.x) >> 5, nwarps = (gridDim.x * kThreads) >> 5;
  for (uint32_t u = o0 + warp; u < o1; u += nwarps) {
    const uint32_t r = uniq_row[u] - row_base;
    const StackSlot e = gtab[uniq_slot[u]];
    const unsigned long long base = frame_off[r];
    for (uint32_t jx = lane; jx < e.size; jx += 32) {
      unsigned long long fid = frame_at(frames, base + jx, narrow);
      const uint32_t pos = e.offset + jx;
      if (fid >= n_frames_registered) { atomicOr(&ctr_w->err, ERR_BAD_FRAME_ID); fid = 0; }
      ustream[pos - off0] = (uint32_t)fid;
      if (loc_first[(uint32_t)fid] > pos) atomicMin(&loc_first[(uint32_t)fid], pos);
    }
  }
}
// thread-id dictionary: list of this shard's (tid, global first row) pairs, and the insert of the other shards' lists
__global__ void __launch_bounds__(kThreads) k_tid_pack(const unsigned long long* hslots, uint32_t hmask, uint32_t* n_out, unsigned long long* out) {
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i <= hmask; i += gridDim.x * kThreads) {
    const unsigned long long sl = hslots[i];
    if (sl != ~0ull) out[atomicAdd(n_out, 1u)] = sl;
  }
}
__global__ void __launch_bounds__(kThreads) k_tid_insert(const unsigned long long* in, uint32_t n, unsigned long long* hslots, uint32_t hmask, Counters* ctr_w) {
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
    const unsigned long long sl = in[i];
    if (hashed_min_insert(hslots, hmask, (uint32_t)(sl >> 32), (uint32_t)sl) == kNull) atomicOr(&ctr_w->err, ERR_TABLE_FULL);
  }
}
// element-wise minimum (the in-process stand-in for ncclAllReduce(min) when every shard of the group lives on one device)
__global__ void __launch_bounds__(kThreads) k_min_u32(uint32_t* dst, const uint32_t* src, size_t n) {
  for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (size_t)gridDim.x * kThreads) { uint32_t v = src[i]; if (v < dst[i]) dst[i] = v; }
}
// x -> ~x in place: around an all-reduce(min), it makes a max-reduction (PA_CFG_GROUP_RETIRE: the group's last_use of each slot)
__global__ void __launch_bounds__(kThreads) k_invert_u32(uint32_t* p, size_t n) {
  for (size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x; i < n; i += (size_t)gridDim.x * kThreads) p[i] = ~p[i];
}
// run-end columns across shards. edges[m][c] come from every shard (all-gather); a shard's last run continues in the next
// non-empty shard when both border rows are non-null and carry the same key (BinaryDictionaryRunEndBuilder.Append,
// reporter/arrow.go:97-131: a row extends the current run iff the previous value is non-null and byte-equal). The
// continued run is written by the shard where it ENDS; the shard where it starts drops its last run.
__global__ void __launch_bounds__(kThreads) k_edges_pack(const Counters* ctr, const unsigned long long* edge_keys, uint32_t ncols, uint32_t row_base, uint32_t n_rows, EdgeCol* out) {
  for (uint32_t c = threadIdx.x; c < ncols; c += blockDim.x) {
    const uint32_t lnn = ctr->last_nonnull_plus1[c];
    out[c] = EdgeCol{ctr->n_runs[c], ctr->n_null[c], lnn ? row_base + lnn : 0u, n_rows, edge_keys[c * 4 + 0], edge_keys[c * 4 + 2],
                     (uint32_t)edge_keys[c * 4 + 1], (uint32_t)edge_keys[c * 4 + 3]};
  }
}
__global__ void __launch_bounds__(kThreads) k_merge_cols(const EdgeCol* edges /*[world][ncols]*/, uint32_t world, uint32_t me, uint32_t ncols,
                                                         MergeCol* mine /*[ncols]*/, MergeCol* all /*[world][ncols]*/, Counters* ctr_w) {
  for (uint32_t c = threadIdx.x; c < ncols; c += blockDim.x) {
    uint32_t base = 0, nulls = 0, lastnn = 0;
    for (uint32_t m = 0; m < world; m++) {
      const EdgeCol e = edges[(size_t)m * ncols + c];
      uint32_t keep = e.n_runs;
      if (e.n_rows) {
        uint32_t nx = m + 1;
        while (nx < world && edges[(size_t)nx * ncols + c].n_rows == 0) nx++;
        if (nx < world) {
          const EdgeCol f = edges[(size_t)nx * ncols + c];
          if (!e.last_null && !f.first_null && e.last_key == f.first_key) keep = e.n_runs - 1;
        }
      }
      const MergeCol mcv{keep, base & 31u, base, 0u};
      all[(size_t)m * ncols + c] = mcv;
      if (m == me) mine[c] = mcv;
      base += keep; nulls += e.n_null; lastnn = max(lastnn, e.lastnn);
    }
    // the counters now describe the MERGED column (identical on every shard)
    ctr_w->n_runs[c] = base; ctr_w->n_null[c] = nulls; ctr_w->last_nonnull_plus1[c] = lastnn;
  }
}

// ---- v1 merged batch: the stacktrace_id dictionary and the known-stacks store, both replicated on every shard. Every shard
// applies the same merged accesses to its copy of the store, so the copies stay identical; only the frames of the stacks the
// store lacks cross between the shards, each sent by the shard that holds the stack's global first occurrence.
// dictionary values of the stacktrace_id column: the merged ids in ordinal order, as the hash kernels write them per row
__global__ void __launch_bounds__(kThreads) k_merged_ids(const Counters* ctr, const StackSlot* gtab, const uint32_t* g_slot, uint8_t* out, int* offsets) {
  const uint32_t nu = ctr->n_unique;
  for (uint32_t u = blockIdx.x * kThreads + threadIdx.x; u <= nu; u += gridDim.x * kThreads) {
    offsets[u] = (int)(16u * u);
    if (u < nu) { const Key128 k = gtab[g_slot[u]].key; *reinterpret_cast<ulonglong2*>(out + 16ull * u) = make_ulonglong2(bswap64(k.hi), bswap64(k.lo)); }
  }
}
// last global row of every merged stack this shard holds, inverted: one all-reduce(min) over the shards gives the global last row
__global__ void __launch_bounds__(kThreads) k_merged_last_rows(uint32_t n_rows, const uint32_t* slot_of_row, const StackSlot* ltab, uint32_t row_base, uint32_t* last_inv) {
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n_rows; i += gridDim.x * kThreads) {  // from the last row down, as k_last_rows
    const uint32_t r = n_rows - 1u - i, s = slot_of_row[r];
    if (s == kNull) continue;
    const uint32_t o = ltab[s].ordinal, v = 0xFFFFFFFFu - (row_base + r);
    if (last_inv[o] > v) atomicMin(&last_inv[o], v);
  }
}
// select keys of the U >= capacity case (k_batch_stamps over merged ordinals)
__global__ void __launch_bounds__(kThreads) k_merged_stamps(const Counters* ctr, const uint32_t* last_inv, unsigned long long* out) {
  const uint32_t nu = ctr->n_unique;
  for (uint32_t u = blockIdx.x * kThreads + threadIdx.x; u < nu; u += gridDim.x * kThreads) out[u] = (unsigned long long)(0xFFFFFFFFu - last_inv[u]) + 1ull;
}
// frames (depth) each merged stack contributes to the exchange: those the insert may write — stacks it stores (last row + 1 >=
// min_last_p1) that the store does not hold live (after a clear: all of them). Every replica computes the same.
__global__ void __launch_bounds__(kThreads) k_store_need(const Counters* ctr, const StackSlot* gtab, const uint32_t* g_slot, const uint32_t* last_inv,
                                                         uint32_t min_last_p1, const StoreSlot* st, uint32_t mask, const unsigned long long* stamp,
                                                         uint32_t* need) {
  const uint32_t nu = ctr->n_unique;
  for (uint32_t u = blockIdx.x * kThreads + threadIdx.x; u < nu; u += gridDim.x * kThreads) {
    const StackSlot e = gtab[g_slot[u]];
    bool n = (0xFFFFFFFFu - last_inv[u]) + 1u >= min_last_p1;
    if (n) {
      const uint32_t sl = store_find(st, mask, e.key);
      n = sl == kNull || st[sl].size == kNull || stamp[sl] == 0;
    }
    need[u] = n ? e.size : 0u;
  }
}
struct StoreFramesF {  // where each merged stack's frames start in the gathered buffer: exclusive scan of k_store_need
  typedef unsigned long long T;
  const Counters* ctr;
  const uint32_t* need;
  unsigned long long* foff;
  __device__ uint32_t n() const { return ctr->n_unique; }
  __device__ unsigned long long value(uint32_t u) const { return need[u]; }
  __device__ void emit(uint32_t u, unsigned long long ex, unsigned long long) const { foff[u] = ex; }
  __device__ void total(int, unsigned long long t) const { foff[ctr->n_unique] = t; }
};
// every rank's share of the gathered buffer: rank r sends the stacks whose global first row lies in its rows (a contiguous
// range of ordinals, see k_won_range), so its block starts at foff[first ordinal at or after row_base[r]]
struct RankRows { uint32_t base[kMaxWorld + 1]; };
__global__ void k_rank_bounds(const Counters* ctr, const uint32_t* g_row, const unsigned long long* foff, RankRows rr, uint32_t world, unsigned long long* out) {
  const uint32_t r = threadIdx.x, nu = ctr->n_unique;
  if (r > world) return;
  uint32_t lo = 0, hi = nu;
  while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (g_row[mid] < rr.base[r]) lo = mid + 1; else hi = mid; }
  out[r] = foff[lo];
}
// this shard's block: the frames of its won stacks that k_store_need selected, from their (local) first occurrence
__global__ void __launch_bounds__(kThreads) k_store_pack(const MergeCtl* mc, const uint32_t* g_row, uint32_t row_base, const uint32_t* need,
                                                         const unsigned long long* foff, const unsigned long long* frames, const unsigned long long* frame_off,
                                                         uint32_t n_frames_registered, uint32_t narrow, uint32_t* out, Counters* ctr_w) {
  const uint32_t o0 = mc->ord0, o1 = mc->ord1;
  const unsigned long long base0 = foff[o0];
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * kThreads + threadIdx.x) >> 5, nwarps = (gridDim.x * kThreads) >> 5;
  for (uint32_t u = o0 + warp; u < o1; u += nwarps) {
    const uint32_t size = need[u];
    if (!size) continue;
    const unsigned long long src = frame_off[g_row[u] - row_base], dst = foff[u] - base0;
    for (uint32_t j = lane; j < size; j += 32) {
      unsigned long long fid = frame_at(frames, src + j, narrow);
      if (fid >= n_frames_registered) { atomicOr(&ctr_w->err, ERR_BAD_FRAME_ID); fid = 0; }
      out[dst + j] = (uint32_t)fid;
    }
  }
}
// PA_CFG_GROUP_STACKS groups: every member holds the same registered stacks, so a stack the store lacks crosses as one reference
// instead of its frames — the handle of its global first occurrence, which keeps that occurrence's frames when two registered
// stacks share a provided id
struct StoreRefsF {  // where each merged stack's reference goes in the gathered buffer: exclusive scan of (k_store_need != 0)
  typedef unsigned long long T;
  const Counters* ctr;
  const uint32_t* need;
  unsigned long long* ridx;
  __device__ uint32_t n() const { return ctr->n_unique; }
  __device__ unsigned long long value(uint32_t u) const { return need[u] ? 1ull : 0ull; }
  __device__ void emit(uint32_t u, unsigned long long ex, unsigned long long) const { ridx[u] = ex; }
  __device__ void total(int, unsigned long long t) const { ridx[ctr->n_unique] = t; }
};
// this shard's block: the references of its won stacks that k_store_need selected. A row's reference is the handle its header
// still carries: hdr_foff points at row 0's frame_off word, and the 64-byte headers are 8 words apart
__global__ void __launch_bounds__(kThreads) k_store_pack_refs(const MergeCtl* mc, const uint32_t* g_row, uint32_t row_base, const uint32_t* need,
                                                              const unsigned long long* ridx, const unsigned long long* hdr_foff, unsigned long long* out) {
  const uint32_t o0 = mc->ord0, o1 = mc->ord1;
  const unsigned long long base0 = ridx[o0];
  for (uint32_t u = o0 + blockIdx.x * kThreads + threadIdx.x; u < o1; u += gridDim.x * kThreads)
    if (need[u]) out[ridx[u] - base0] = hdr_foff[(size_t)(g_row[u] - row_base) * 8];
}

// ---------------------------------------------------------------------------------------------
// LZ4_FRAME body compression on the device (PA_IPC_LZ4_FRAME_GPU). Every non-empty Arrow buffer of the stream becomes one
// LZ4 frame of independent blocks of at most 64 KiB of input; one warp encodes one block. The encoding is a function of the
// block's bytes alone (no atomics, no dependence on grid size or timing), and keeps every LZ4 block rule: matches of 4 or
// more bytes, offsets 1..65535 inside the block, the last match starting 13 or more bytes before the block's end and ending
// 5 or more bytes before it.
constexpr uint32_t kLz4Block = 65536;
constexpr int kLz4HashLog = 12;
constexpr int kLz4Warps = 4;       // warps per thread block: 4 x 8 KiB hash tables
constexpr uint16_t kLz4Empty = 0xFFFF;  // no position: a match never starts at 65535 (the last start is len - 13)

struct Lz4Blk { const uint8_t* src; uint32_t len; uint32_t buf; };    // src == nullptr: zeros
struct Lz4Buf { uint64_t len; uint32_t first, nblk; };                // blocks first .. first+nblk-1 of one Arrow buffer

__device__ __forceinline__ uint32_t lz4_byte(const uint8_t* s, uint32_t i) { return s ? (uint32_t)__ldg(s + i) : 0u; }
__device__ __forceinline__ uint32_t lz4_word(const uint8_t* s, uint32_t i) {
  return s ? (uint32_t)__ldg(s + i) | (uint32_t)__ldg(s + i + 1) << 8 | (uint32_t)__ldg(s + i + 2) << 16 | (uint32_t)__ldg(s + i + 3) << 24 : 0u;
}
__device__ __forceinline__ uint32_t lz4_hash(uint32_t v) { return (v * 2654435761u) >> (32 - kLz4HashLog); }

// One sequence (nlit literals from src[lit0..], then a match of mlen bytes at distance off; mlen == 0: the closing literals),
// written by the whole warp at out[*op]. False when it would not fit in `cap` bytes (the block is then stored raw).
__device__ __forceinline__ bool lz4_sequence(uint8_t* out, uint32_t* op, uint32_t cap, const uint8_t* src, uint32_t lit0, uint32_t nlit,
                                             uint32_t off, uint32_t mlen, uint32_t lane) {
  const uint32_t ml = mlen ? mlen - 4 : 0;
  const uint32_t litx = nlit >= 15 ? (nlit - 15) / 255 + 1 : 0, mlx = ml >= 15 ? (ml - 15) / 255 + 1 : 0;
  const uint32_t total = 1 + litx + nlit + (mlen ? 2 + mlx : 0);
  if (*op + total > cap) return false;
  uint8_t* o = out + *op;
  if (lane == 0) o[0] = (uint8_t)(min(nlit, 15u) << 4 | min(ml, 15u));
  for (uint32_t j = lane; j < litx; j += 32) o[1 + j] = j + 1 < litx ? 255 : (uint8_t)((nlit - 15) % 255);
  for (uint32_t j = lane; j < nlit; j += 32) o[1 + litx + j] = (uint8_t)lz4_byte(src, lit0 + j);
  if (mlen) {
    uint8_t* q = o + 1 + litx + nlit;
    if (lane == 0) { q[0] = (uint8_t)(off & 0xFF); q[1] = (uint8_t)(off >> 8); }
    for (uint32_t j = lane; j < mlx; j += 32) q[2 + j] = j + 1 < mlx ? 255 : (uint8_t)((ml - 15) % 255);
  }
  *op += total;
  return true;
}

// Greedy LZ4 of one block per warp. Each step looks up the 32 positions p..p+31 at once in a hash table of block-relative
// positions; the lowest position whose candidate matches starts the next match, which is extended 32 bytes per ballot. Lanes
// that share a hash slot insert their positions with a fixed rule (the highest position wins). blk_size[b] = compressed
// bytes, or 0x80000000 | len when the encoding would not be smaller than the block (stored raw).
__global__ void __launch_bounds__(kLz4Warps * 32) k_lz4_compress(const Lz4Blk* __restrict__ blks, uint32_t nblk, uint8_t* __restrict__ slots,
                                                                uint32_t* __restrict__ blk_size) {
  __shared__ uint16_t tab_all[kLz4Warps][1 << kLz4HashLog];
  const uint32_t lane = threadIdx.x & 31, b = blockIdx.x * kLz4Warps + (threadIdx.x >> 5);
  if (b >= nblk) return;  // whole warps only
  uint16_t* tab = tab_all[threadIdx.x >> 5];
  const Lz4Blk k = blks[b];
  const uint8_t* src = k.src;
  const uint32_t n = k.len, cap = n - 1;
  uint8_t* out = slots + (size_t)b * kLz4Block;
  for (uint32_t i = lane; i < (1u << kLz4HashLog); i += 32) tab[i] = kLz4Empty;
  __syncwarp();
  const int32_t last_start = (int32_t)n - 13;
  uint32_t op = 0, anchor = 0, p = 0;
  bool fits = true;
  while ((int32_t)p <= last_start) {
    const uint32_t pos = p + lane;
    const bool valid = (int32_t)pos <= last_start;
    uint32_t h = kNull, cand = kLz4Empty;
    bool ok = false;
    if (valid) {
      const uint32_t v = lz4_word(src, pos);
      h = lz4_hash(v);
      cand = tab[h];
      ok = cand != kLz4Empty && lz4_word(src, cand) == v;
    }
    const unsigned hit = __ballot_sync(~0u, ok);
    const uint32_t upto = hit ? __ffs(hit) - 1 : 31;  // positions p..p+upto are inserted
    const uint32_t key = valid && lane <= upto ? h : kNull;
    const unsigned same = __match_any_sync(~0u, key);
    if (key != kNull && 31 - __clz(same) == (int)lane) tab[h] = (uint16_t)pos;
    __syncwarp();
    if (!hit) { p += 32; continue; }
    const uint32_t mpos = p + upto, mcand = __shfl_sync(~0u, cand, upto);
    const uint32_t maxlen = n - 5 - mpos;  // mpos <= n - 13, so maxlen >= 8
    uint32_t mlen = 4;
    for (;;) {
      const uint32_t i = mlen + lane;
      const bool stop = i >= maxlen || lz4_byte(src, mpos + i) != lz4_byte(src, mcand + i);
      const unsigned d = __ballot_sync(~0u, stop);
      if (d) { mlen += __ffs(d) - 1; break; }
      mlen += 32;
    }
    if (!(fits = lz4_sequence(out, &op, cap, src, anchor, mpos - anchor, mpos - mcand, mlen, lane))) break;
    p = anchor = mpos + mlen;
    if (lane == 0) tab[lz4_hash(lz4_word(src, p - 2))] = (uint16_t)(p - 2);
    __syncwarp();
  }
  if (fits) fits = lz4_sequence(out, &op, cap, src, anchor, n - anchor, 0, 0, lane);
  if (lane == 0) blk_size[b] = fits ? op : (0x80000000u | n);
}

// One warp per buffer: offset of every block inside its frame (counted from the end of the 7-byte frame header) and the
// frame's whole size (header + blocks with their 4-byte sizes + EndMark).
__global__ void __launch_bounds__(kThreads) k_lz4_layout(const Lz4Buf* __restrict__ bufs, uint32_t nbuf, const uint32_t* __restrict__ blk_size,
                                                         uint64_t* __restrict__ blk_off, uint64_t* __restrict__ frame) {
  const uint32_t lane = threadIdx.x & 31, w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (w >= nbuf) return;
  const Lz4Buf B = bufs[w];
  uint64_t run = 0;
  for (uint32_t i0 = 0; i0 < B.nblk; i0 += 32) {
    const uint32_t i = i0 + lane;
    const uint32_t sz = i < B.nblk ? 4 + (blk_size[B.first + i] & 0x7FFFFFFFu) : 0;
    uint32_t incl = sz;
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t t = __shfl_up_sync(~0u, incl, d);
      if ((int)lane >= d) incl += t;
    }
    if (i < B.nblk) blk_off[B.first + i] = run + incl - sz;
    run += __shfl_sync(~0u, incl, 31);
  }
  if (lane == 0) frame[w] = 7 + run + 4;
}

__device__ __forceinline__ void lz4_warp_copy(uint8_t* dst, const uint8_t* src, uint32_t n, uint32_t lane) {
  uint32_t j = lane;
  for (; j + 96 < n; j += 128) {
    const uint8_t a = (uint8_t)lz4_byte(src, j), b = (uint8_t)lz4_byte(src, j + 32), c = (uint8_t)lz4_byte(src, j + 64), d = (uint8_t)lz4_byte(src, j + 96);
    dst[j] = a; dst[j + 32] = b; dst[j + 64] = c; dst[j + 96] = d;
  }
  for (; j < n; j += 32) dst[j] = (uint8_t)lz4_byte(src, j);
}

// One warp per block: writes the block where the compressed body puts it. buf_dst[i] = offset of buffer i in `body` (bit 63:
// the buffer is stored raw, as -1 and its bytes). The first block of a buffer writes the int64 length prefix and the frame
// header, the last one the EndMark and the zero padding up to the next 8-byte boundary.
__global__ void __launch_bounds__(kThreads) k_lz4_pack(const Lz4Blk* __restrict__ blks, uint32_t nblk, const Lz4Buf* __restrict__ bufs,
                                                       const uint8_t* __restrict__ slots, const uint32_t* __restrict__ blk_size,
                                                       const uint64_t* __restrict__ blk_off, const uint64_t* __restrict__ frame,
                                                       const uint64_t* __restrict__ buf_dst, uint8_t* __restrict__ body) {
  const uint32_t lane = threadIdx.x & 31, b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (b >= nblk) return;
  const Lz4Blk k = blks[b];
  const Lz4Buf B = bufs[k.buf];
  const uint64_t d = buf_dst[k.buf];
  const bool raw = d >> 63, first = b == B.first, last = b + 1 == B.first + B.nblk;
  uint8_t* dst = body + (d & ~(1ull << 63));
  uint64_t end;
  if (raw) {
    if (first && lane == 0) *reinterpret_cast<long long*>(dst) = -1;
    lz4_warp_copy(dst + 8 + (uint64_t)(b - B.first) * kLz4Block, k.src, k.len, lane);
    end = 8 + B.len;
  } else {
    if (first && lane < 15) {  // then the frame header 04 22 4D 18 60 40 82: magic, FLG, BD (64 KiB blocks), HC
      constexpr uint64_t kHdr = 0x00824060184D2204ull;
      dst[lane] = (uint8_t)(lane < 8 ? B.len >> (8 * lane) : kHdr >> (8 * (lane - 8)));
    }
    const uint32_t sz = blk_size[b], n = sz & 0x7FFFFFFFu;
    uint8_t* o = dst + 15 + blk_off[b];
    if (lane < 4) o[lane] = (uint8_t)(sz >> (8 * lane));
    if (sz >> 31) lz4_warp_copy(o + 4, k.src, n, lane);
    else lz4_warp_copy(o + 4, slots + (size_t)b * kLz4Block, n, lane);
    end = 8 + frame[k.buf];
    if (last && lane < 4) dst[end - 4 + lane] = 0;  // EndMark
  }
  if (last)
    for (uint64_t i = end + lane; i < ((end + 7) & ~7ull); i += 32) dst[i] = 0;
}

// Merge groups: one warp per block of this member's share of the frames. buf_dst[i] = offset of buffer i's share in `body` (bit
// 63: the buffer is stored raw, and the member copies its part of the buffer as it is). Writes the block's 4-byte size and its
// bytes at blk_off[b] inside the share; the length prefix, frame header, EndMark and padding are written by the group's root.
__global__ void __launch_bounds__(kThreads) k_lz4_pack_parts(const Lz4Blk* __restrict__ blks, uint32_t nblk, const uint8_t* __restrict__ slots,
                                                             const uint32_t* __restrict__ blk_size, const uint64_t* __restrict__ blk_off,
                                                             const uint64_t* __restrict__ buf_dst, uint8_t* __restrict__ body) {
  const uint32_t lane = threadIdx.x & 31, b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (b >= nblk) return;
  const Lz4Blk k = blks[b];
  const uint64_t d = buf_dst[k.buf];
  if (d >> 63) return;
  const uint32_t sz = blk_size[b], n = sz & 0x7FFFFFFFu;
  uint8_t* o = body + d + blk_off[b];
  if (lane < 4) o[lane] = (uint8_t)(sz >> (8 * lane));
  if (sz >> 31) lz4_warp_copy(o + 4, k.src, n, lane);
  else lz4_warp_copy(o + 4, slots + (size_t)b * kLz4Block, n, lane);
}

// ---------------------------------------------------------------------------------------------
// PA_CFG_RETIRE_STACKS: the device-resident stack registry (records, per-slot last_use words, the frame arena).
// Record updates: upd[i] goes to slot[i]. A record with kStackFree in pad frees its slot. Any other is a registration whose
// `off` counts from `base`, where its frames were uploaded; its last_use starts at seq[i], the batches staged before it was
// registered, so a stack is idle for k batches only once it was registered before them.
__global__ void __launch_bounds__(kThreads) k_stack_scatter(const RegStack* __restrict__ upd, const uint32_t* __restrict__ slot,
                                                            const uint32_t* __restrict__ seq, uint32_t n, unsigned long long base,
                                                            RegStack* __restrict__ recs, uint32_t* __restrict__ last_use) {
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
    RegStack r = upd[i];
    if (!(r.pad & kStackFree)) {
      r.off += base;
      last_use[slot[i]] = seq[i];
    }
    recs[slot[i]] = r;
  }
}

// Idle selection: bit i = slot i is live and its last_use is at most `bound` (neither registered nor named in the window).
// The bitmap goes through WordsF (exclusive popcount prefix) and k_stack_idle_emit writes the handles in slot order.
__global__ void __launch_bounds__(kThreads) k_stack_idle_bits(const RegStack* __restrict__ recs, const uint32_t* __restrict__ last_use, uint32_t n,
                                                              uint32_t bound, uint32_t* __restrict__ bits) {
  const uint32_t n32 = (n + 31u) & ~31u;  // whole warps: the ballot needs every lane
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n32; i += gridDim.x * kThreads) {
    const bool idle = i < n && !(recs[i].pad & kStackFree) && last_use[i] <= bound;
    const uint32_t w = __ballot_sync(0xFFFFFFFFu, idle);
    if ((threadIdx.x & 31u) == 0) bits[i >> 5] = w;
  }
}
// The first `cap` idle slots are retired: their handles go out in slot order and their last_use becomes 0xFFFFFFFF, which keeps
// them out of every later selection while they wait for their grace batch (a row of that batch may overwrite it with a
// sequence number that is inside every later window).
__global__ void __launch_bounds__(kThreads) k_stack_idle_emit(const uint32_t* __restrict__ bits, const uint32_t* __restrict__ wprefix, uint32_t n,
                                                              const RegStack* __restrict__ recs, unsigned long long cap,
                                                              unsigned long long* __restrict__ handles, uint32_t* __restrict__ last_use) {
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads) {
    const uint32_t w = bits[i >> 5];
    if (!((w >> (i & 31u)) & 1u)) continue;
    const uint32_t rank = wprefix[i >> 5] + (uint32_t)__popc(w & ((1u << (i & 31u)) - 1u));
    if (rank >= cap) continue;
    handles[rank] = ((unsigned long long)recs[i].pad << 32) | i;
    last_use[i] = 0xFFFFFFFFu;
  }
}

// Arena compaction: the live stacks' frames move, in slot order, into a fresh buffer. One scan over the slots gives each live
// stack its new offset (frames) and its copy chunks (kCompactChunk ids each), so a 65535-id stack is spread over 256 warps
// instead of holding one.
constexpr uint32_t kCompactChunk = 256;
struct StackLiveF {
  typedef Pair T;  // {chunks, frames}
  const RegStack* recs;
  uint32_t n_slots;
  unsigned long long* new_off;
  uint2* chunks;  // (slot, chunk index in the stack)
  Pair* total_out;
  __device__ uint32_t n() const { return n_slots; }
  __device__ Pair value(uint32_t i) const {
    const RegStack& r = recs[i];
    const uint32_t d = (r.pad & kStackFree) ? 0u : r.depth;
    return Pair{(d + kCompactChunk - 1) / kCompactChunk, d};
  }
  __device__ void emit(uint32_t i, Pair ex, Pair v) const {
    new_off[i] = ex.fr;
    for (uint32_t c = 0; c < v.cnt; c++) chunks[ex.cnt + c] = make_uint2(i, c);
  }
  __device__ void total(int, Pair t) const { *total_out = t; }
};
// one warp per chunk; `words` = 32-bit words per frame id (the arena holds the ids at the ring's width)
__global__ void __launch_bounds__(kThreads) k_stack_compact_copy(const Pair* __restrict__ total, const uint2* __restrict__ chunks, const RegStack* __restrict__ recs,
                                                                 const unsigned long long* __restrict__ new_off, uint32_t words,
                                                                 const uint32_t* __restrict__ src, uint32_t* __restrict__ dst) {
  const uint32_t lane = threadIdx.x & 31u, nc = total->cnt;
  for (uint32_t c = (blockIdx.x * kThreads + threadIdx.x) >> 5; c < nc; c += (gridDim.x * kThreads) >> 5) {
    const uint2 e = chunks[c];
    const unsigned long long j0 = (unsigned long long)e.y * kCompactChunk;
    const uint32_t cnt = min(kCompactChunk, (uint32_t)(recs[e.x].depth - j0)) * words;
    const uint32_t* s = src + (recs[e.x].off + j0) * words;
    uint32_t* d = dst + (new_off[e.x] + j0) * words;
    for (uint32_t k = lane; k < cnt; k += 32) d[k] = s[k];
  }
}
__global__ void __launch_bounds__(kThreads) k_stack_rebase(RegStack* __restrict__ recs, uint32_t n, const unsigned long long* __restrict__ new_off) {
  for (uint32_t i = blockIdx.x * kThreads + threadIdx.x; i < n; i += gridDim.x * kThreads)
    if (!(recs[i].pad & kStackFree)) recs[i].off = new_off[i];
}

}  // namespace pa
