/*
 * parcaagg.h — C ABI of libparcaagg: the H100-native replacement for parca-agent's
 * per-interval sample → Arrow (v2 schema) aggregation path.
 *
 * Drop-in boundary (reference file:line are relative to parca-dev/parca-agent):
 *   - reporter.Reporter as implemented by ParcaReporter, reporter/parca_reporter.go:56
 *     (ReportTraceEvent :219, reportTraceEventV2 :332, writeSampleV2 :368, appendLocationV2 :418,
 *      labelsForTID :568, buildSampleRecordV2 :1742, IPC serialisation :1779-1790 / :1847-1860)
 *   - the Arrow builders in reporter/arrow_v2.go (SampleWriterV2 :500-682,
 *     StacktraceDictBuilderV2 :228-497, FunctionDictBuilderV2 :163-218) and the run-end
 *     wrappers in reporter/arrow.go:14-207.
 *
 * A Go (cgo) shim implementing reporter.Reporter binds exactly these entry points; see
 * INTEGRATION.md. Plain pointers and sizes only; no C++/torch types cross this boundary.
 * Every function returns 0 on success or a negative PA_E* code; pa_agg_last_error() gives text.
 * No exception or abort crosses the boundary. All multi-byte fields are little-endian.
 */
#ifndef PARCAAGG_H
#define PARCAAGG_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PA_ABI_VERSION 3u

/* ---- error codes -------------------------------------------------------------------------- */
#define PA_OK 0
#define PA_EINVAL (-22)   /* bad argument / unknown id */
#define PA_ENOMEM (-12)   /* host or device allocation failed */
#define PA_ENOSPC (-28)   /* ring full (submit) — caller must flush */
#define PA_ENODEV (-19)   /* no usable CUDA device */
#define PA_EIO (-5)       /* CUDA runtime failure; see pa_agg_last_error */
#define PA_ERANGE (-34)   /* batch exceeds Arrow int32 limits (reporter/arrow_v2.go:233-234) */

/* ---- sample kinds: one output row each; replaces the Origin switch of
 *      reportTraceEventV2 (reporter/parca_reporter.go:338-363). The shim expands a
 *      TraceOriginMemory event into up to four rows (:343-360). ------------------------------ */
enum {
  PA_KIND_CPU = 0,          /* TraceOriginSampling :340  value=1      */
  PA_KIND_OFFCPU = 1,       /* TraceOriginOffCPU   :342  value=OffTime */
  PA_KIND_CUDA = 2,         /* TraceOriginCuda     :362  value=OffTime */
  PA_KIND_MEM_INUSE_OBJECTS = 3, /* :351 */
  PA_KIND_MEM_INUSE_SPACE = 4,   /* :354 */
  PA_KIND_MEM_ALLOC_OBJECTS = 5, /* :357 */
  PA_KIND_MEM_ALLOC_SPACE = 6,   /* :358 */
  PA_KIND_COUNT = 7
};

/* ---- frame kinds: which branch of appendLocationV2 (reporter/parca_reporter.go:418-555)
 *      resolves the frame. The frame-type *string* (libpf.FrameType.String(), an un-vendored
 *      dependency) is supplied by the shim as a string id. ----------------------------------- */
enum {
  PA_FRAME_NATIVE = 0,   /* :449-476 */
  PA_FRAME_KERNEL = 1,   /* :478-514 */
  PA_FRAME_ABORT = 2,    /* :432-446 */
  PA_FRAME_OOMPROF = 3,  /* :516-520 */
  PA_FRAME_INTERP = 4    /* :522-551 (python, ruby, jvm, cuda, ...) */
};
#define PA_FRAME_F_MAPPING_FILE 0x1u /* frame.Mapping.Valid() && m.File != {} (:456-462) */
#define PA_FRAME_F_EXEC_KNOWN 0x2u   /* r.executables.Get(FileID) hit (:460, :490) */

#define PA_HASH_PROVIDED 0u /* trace.Hash arrives in the header — the reference's behaviour (:394-395) */
#define PA_HASH_XXH64X2 1u  /* hi=XXH64(frame ids LE, seed 0), lo=XXH64(same, seed 0x9E3779B97F4A7C15) on the GPU */
#define PA_XXH_SEED_LO 0x9E3779B97F4A7C15ull

#define PA_LABEL_DISABLE_CPU 0x1u         /* --metadata-disable-cpu-label (flags/flags.go:317) */
#define PA_LABEL_DISABLE_THREAD_ID 0x2u   /* --metadata-disable-thread-id-label (:318) */
#define PA_LABEL_DISABLE_THREAD_COMM 0x4u /* --metadata-disable-thread-comm-label (:319) */

#define PA_SCHEMA_V2 0u /* inline stacktraces, reporter/arrow_v2.go */
#define PA_SCHEMA_V1 1u /* stacktrace ids only, reporter/arrow.go:260-332 + parca_reporter.go:246-328 (sample record);
                           the follow-up record with the full stacktraces comes from pa_agg_stacktraces */

#define PA_IPC_PLAIN 0u
#define PA_IPC_LZ4_FRAME 1u
#define PA_IPC_LZ4_FRAME_GPU 2u

#define PA_CFG_SINGLE_RING 0x1u /* one ring buffer instead of two: ingest is refused (PA_ENOSPC) while a flush holds the ring.
                                    Halves the pinned host memory; for replay / batch use, not for a live agent */
#define PA_CFG_REGISTERED_STACKS 0x2u /* registered stacks: stacks are registered once (pa_agg_register_stacks) and a sample row
                                    names its stack by id in frame_off; the ring holds 64-byte headers only (no frame ids, no frame
                                    ring, no device frame buffer). Works with both hash modes, both schemas, both frame_id_bytes and
                                    every ipc_compression; the output is byte for byte the record of the same rows with their frame ids
                                    in the ring. Row meaning in this mode: frame_off = a registered stack id; hash_hi / hash_lo and
                                    nframes are ignored (the stack's registration supplies them); pa_agg_acquire takes n_frames == 0
                                    and hands out *frames = NULL; pa_agg_submit ignores `frames` and keeps the caller's frame_off. A row
                                    whose stack id is not registered fails the flush with PA_EINVAL (the next flush works).
                                    max_frames (0 = max_samples * 64) bounds the registered frames instead of the ring.
                                    Not supported (PA_EINVAL): pa_agg_shard_export, pa_agg_stage_device(_parts); and pa_merge_create_*
                                    unless PA_CFG_GROUP_STACKS is set too */
#define PA_CFG_GROUP_STACKS 0x4u /* with PA_CFG_REGISTERED_STACKS only (pa_agg_create fails with PA_EINVAL otherwise): the stack ids
                                    are group-wide, so the aggregator may be a member of a merge group. Every member of such a group
                                    registers the same stacks in the same order (like strings, frames and labelsets), so a row's
                                    frame_off names the same stack on every shard; pa_merge_process checks the count, the arena length
                                    and a digest of (id, depth, frame ids) of the registered stacks and fails with PA_EINVAL on every
                                    rank when they differ. A group cannot mix such members with ring members (pa_merge_create_local
                                    refuses it, multi-process groups fail pa_merge_process on every rank). On its own the aggregator
                                    behaves exactly like a PA_CFG_REGISTERED_STACKS one */
#define PA_CFG_RETIRE_STACKS 0x8u /* with PA_CFG_REGISTERED_STACKS only, and not with PA_CFG_GROUP_STACKS (pa_agg_create fails with
                                    PA_EINVAL otherwise): registered stacks that no batch has named for a while can be retired
                                    (pa_agg_retire_stacks) and their slots reused, so the registry of a long-running agent stays bounded.
                                    A stack is named by a 64-bit handle, generation << 32 | slot, that pa_agg_register_stack_handles
                                    returns; a row puts it in frame_off. A slot that was never reused has generation 0, so its handle is
                                    the id the plain mode would have given. A handle whose slot has been freed or reused never names
                                    another stack: a row that carries one fails its flush with PA_EINVAL (the next flush works).
                                    pa_agg_register_stacks is refused (PA_EINVAL). max_frames bounds the frames of the stacks not yet
                                    freed (live, pending, and retired ones still in their grace batch); the frames freed stacks leave
                                    behind do not count, and the device arena is compacted when they outweigh the live ones. The
                                    output is byte for byte the same as without the flag */
#define PA_CFG_GROUP_RETIRE 0x10u /* only as PA_CFG_REGISTERED_STACKS | PA_CFG_GROUP_STACKS | PA_CFG_GROUP_RETIRE (pa_agg_create fails with
                                    PA_EINVAL otherwise, and with PA_CFG_RETIRE_STACKS): retirement for the members of a merge group.
                                    Stacks are named by handles and registered through pa_agg_register_stack_handles, as with
                                    PA_CFG_RETIRE_STACKS, but the group retires them, collectively (pa_merge_retire_stacks): a stack that
                                    any member's rows named in the idle window stays live, and every member's slots, generations and free
                                    slots stay identical, so identical registrations return identical handles on every member.
                                    pa_agg_retire_stacks is refused (PA_EINVAL); the registry counters of PA_CFG_RETIRE_STACKS work.
                                    pa_merge_process checks the members' slot count, stage count and a digest of every registration
                                    (handle, id, depth, frame ids) and retirement, and fails with PA_EINVAL on every rank when they
                                    differ: a member staged or flushed on its own has left the group's lockstep. A group cannot mix such
                                    members with other members (refused like a mixed PA_CFG_GROUP_STACKS group) */

#define PA_NO_STRING 0xFFFFFFFFu /* "no value"; string id 0 is always the empty string "" */

/* One sample = one (trace, meta) pair handed to ReportTraceEvent (:219): 64 bytes. */
typedef struct pa_sample_hdr {
  uint64_t hash_hi;      /* trace.Hash (libpf.TraceHash) — ignored in PA_HASH_XXH64X2 mode */
  uint64_t hash_lo;
  int64_t timestamp_ns;  /* meta.Timestamp (:397) */
  int64_t value;         /* meta.OffTime / memory value; ignored for PA_KIND_CPU (value=1) */
  uint32_t pid;          /* meta.PID — shard key on >1 GPU */
  uint32_t tid;          /* meta.TID → label thread_id (:621) */
  uint32_t comm_sid;     /* string id of meta.Comm → label thread_name (:624); 0 (= "") drops it */
  uint32_t labelset_id;  /* per-PID cached labels (content of the labels LRU, :569) */
  uint64_t frame_off;    /* index of this sample's first frame id in the batch frame stream;
                            filled by pa_agg_submit / by the producer after pa_agg_acquire.
                            PA_CFG_REGISTERED_STACKS: the registered stack id of this sample (set by the caller) */
  uint32_t cpu;          /* meta.CPU → label cpu (:618) */
  uint16_t nframes;      /* len(trace.Frames) */
  uint8_t kind;          /* PA_KIND_* */
  uint8_t flags;         /* reserved, 0 */
} pa_sample_hdr;

/* One distinct libpf.Frame value (the dedup key of appendLocationV2, :421): 64 bytes.
 * frame ids are dense: the i-th registered frame has id i. The shim guarantees
 * frame-id equality == libpf.Frame value equality (it interns unique.Handle → id). */
typedef struct pa_frame_desc {
  uint8_t kind;                /* PA_FRAME_* */
  uint8_t flags;               /* PA_FRAME_F_* */
  uint16_t reserved0;
  uint32_t type_name_sid;      /* frame.Type.String() */
  uint64_t address_or_lineno;  /* frame.AddressOrLineno (:429) */
  uint32_t function_name_sid;  /* frame.FunctionName ("" = 0) */
  uint32_t source_file_sid;    /* frame.SourceFile */
  uint32_t source_line;        /* frame.SourceLine */
  uint32_t exec_file_name_sid; /* execInfo.FileName when PA_FRAME_F_EXEC_KNOWN */
  uint32_t exec_build_id_sid;  /* execInfo.BuildID ("" → FileID hex, :467-471) */
  uint32_t source_column;      /* frame.SourceColumn (v1 stacktrace record only, :1680, :1727) */
  uint64_t file_id_hi;         /* mf.FileID */
  uint64_t file_id_lo;
  uint32_t mapping_file_name_sid; /* frame.Mapping.File.FileName — v1 interpreted frames with a GNU build id (:1716-1719) */
  uint32_t gnu_build_id_sid;      /* frame.Mapping.File.GnuBuildID ("" = 0: fall back to the frame-type string) */
} pa_frame_desc;

typedef struct pa_label_pair {
  uint32_t name_sid;
  uint32_t value_sid;
} pa_label_pair;

typedef struct pa_agg_config {
  uint32_t abi_version;        /* PA_ABI_VERSION */
  int32_t device;              /* CUDA device ordinal */
  uint32_t hash_mode;          /* PA_HASH_* */
  uint32_t label_flags;        /* PA_LABEL_DISABLE_* */
  uint32_t samples_per_second; /* --profiling-cpu-sampling-frequency (period = 1e9/this, :340) */
  uint32_t n_external_labels;  /* --metadata-external-labels → LabelAll at flush (:1760-1764) */
  const pa_label_pair* external_labels; /* string ids must be registered before the first flush */
  uint64_t max_samples;        /* ring capacity in rows (per buffer; two buffers are kept) */
  uint64_t max_frames;         /* ring capacity in frame ids (per buffer); PA_CFG_REGISTERED_STACKS: capacity of the registered frames */
  uint32_t chunk_samples;      /* H2D/compute overlap granularity; 0 = default */
  uint32_t schema;             /* PA_SCHEMA_V2 (0, default here) or PA_SCHEMA_V1 (--remote-store-use-v2-schema=false,
                                  flags/flags.go:349): which sample record pa_agg_flush builds */
  uint64_t stack_cache_entries; /* v1 only: capacity of the known-stacks store (the `stacks` LRU, cacheSize at
                                  parca_reporter.go:876; main.go:630 keeps it >= 65536). 0 = max(65536, max_samples). Exact LRU:
                                  after every batch and every pa_agg_stacktraces call the store holds the stacks accessed last */
  uint64_t stack_cache_frames;  /* v1 only: capacity of the store's frame arena, in frames. 0 = 128 per entry (4 bytes each: content + one batch of 64-frame stacks). Not a
                                  reference limit: when the live stacks alone exceed it the store starts over from the current batch */
  uint32_t unknown_frame_type_sid; /* v1 only: string id of libpf.UnknownFrame.String() for the "missing stacktrace"
                                  row (:1561); 0 = the literal "unknown" */
  uint32_t flags;              /* PA_CFG_* */
  uint32_t frame_id_bytes;     /* width of one frame id in the ring: 0 or 8 = uint64 (a unique.Handle-sized slot, the default), 4 = uint32.
                                  Frame ids are dense registration indices (< 2^32 by construction), so the narrow ring carries the same
                                  ids in half the PCIe / HBM bytes; stack ids and every output byte are identical (XXH64 is defined over
                                  the ids as little-endian uint64 either way: the kernel widens on load). pa_agg_acquire / pa_agg_submit
                                  then take and hand out uint32 arrays through the same pointers. */
  uint32_t ipc_compression;    /* PA_IPC_PLAIN (0): uncompressed bodies == the offline-mode bytes (:1779-1790), the bit-exact mode.
                                  PA_IPC_LZ4_FRAME (1): bodies wrapped like ipc.WithLZ4() (:1851, the gRPC path) — decodes to the
                                  same record but is NOT byte-identical to the Go writer (different LZ4 encoder). Host work: the
                                  uncompressed stream is copied out, then re-encoded with the system liblz4.so.1.
                                  PA_IPC_LZ4_FRAME_GPU (2): the same framing (ipc.WithLZ4()), with the bodies encoded on the GPU in
                                  independent 64 KiB LZ4 blocks; only the compressed bodies cross PCIe and no liblz4 is needed. It
                                  decodes to the same record and is NOT byte-identical to the Go writer (nor to mode 1). The mode for
                                  the gRPC path. Both modes apply to every result: v2 and v1 sample records and pa_agg_stacktraces.
                                  Merge groups: when EVERY member is PA_IPC_LZ4_FRAME_GPU the merged record is LZ4_FRAME too, byte
                                  for byte the stream one such aggregator makes from the concatenated rows (see pa_merge_* below). A
                                  group that mixes PA_IPC_LZ4_FRAME_GPU members with other members is refused (PA_EINVAL). Groups of
                                  PA_IPC_PLAIN or PA_IPC_LZ4_FRAME members build uncompressed merged records (the host mode is not
                                  applied to them; pa_ipc_compress_lz4 can be). */
} pa_agg_config;

/* Result of one flush; memory is library-owned (pinned host) until pa_agg_release. */
typedef struct pa_agg_result {
  const uint8_t* ipc;        /* uncompressed Arrow IPC stream == offline-mode V2 bytes (:1779-1790) */
  uint64_t ipc_len;
  uint64_t n_rows;           /* record.NumRows(); 0 ⇒ ipc==NULL (reference skips the send, :1842-1845) */
  uint64_t n_unique_stacks;  /* StacktraceDictBuilderV2.UniqueStacktraces() (arrow_v2.go:338) */
  uint64_t n_locations;      /* len(LocationIndex) */
  uint64_t n_functions;      /* funcDict.Len() */
  uint64_t n_location_indices;
  uint32_t gpu_launches;     /* kernels launched for this flush */
  uint32_t reserved;
  double h2d_ms, gpu_ms, d2h_ms, host_ms; /* stage timings of this flush */
} pa_agg_result;

typedef struct pa_agg pa_agg; /* opaque */

/* lifecycle — reporter.New (:836) / Stop (:802) */
int pa_agg_create(const pa_agg_config* cfg, pa_agg** out);
void pa_agg_destroy(pa_agg* a);
const char* pa_agg_last_error(const pa_agg* a);
uint32_t pa_agg_abi_version(void);

/* dictionaries (host → library, append-only, ids dense in registration order).
 * strings: n strings as offsets[n+1] into bytes; *first_id receives the id of the first one. */
int pa_agg_register_strings(pa_agg* a, const uint8_t* bytes, const uint32_t* offsets, uint32_t n, uint32_t* first_id);
int pa_agg_register_frames(pa_agg* a, const pa_frame_desc* descs, uint32_t n, uint64_t* first_frame_id);
/* labelsets: n sets, set i = pairs[offsets[i]..offsets[i+1]) sorted by name (labels.Labels order). */
int pa_agg_register_labelsets(pa_agg* a, const pa_label_pair* pairs, const uint32_t* offsets, uint32_t n, uint32_t* first_id);
/* stacks (PA_CFG_REGISTERED_STACKS only): n stacks, stack i = frames[offsets[i]..offsets[i+1]) (uint32 ids when
 * frame_id_bytes = 4, as in pa_agg_submit); ids are dense and append-only like frame ids, *first_stack_id receives the first.
 * hashes: 2n words hash_hi, hash_lo per stack, as in pa_sample_hdr; required in PA_HASH_PROVIDED mode and NULL in
 * PA_HASH_XXH64X2 mode, where the library computes each id here with the definition the GPU uses for ring rows (XXH64 over the
 * ids as little-endian uint64, seeds 0 and PA_XXH_SEED_LO; pa_xxh64). Thread-safe, may run during a flush; a batch uses the
 * stacks registered when it is processed. All or nothing: a refused call registers no stack.
 * PA_EINVAL: unregistered frame id, aggregator without the flag, hashes given / missing for the hash mode.
 * PA_ERANGE: a stack deeper than 65535. PA_ENOSPC: the registered frames would exceed max_frames. */
int pa_agg_register_stacks(pa_agg* a, const uint64_t* hashes, const uint64_t* frames, const uint64_t* offsets, uint32_t n, uint64_t* first_stack_id);
/* The same inputs, validation and errors as pa_agg_register_stacks, in either registered mode; handles[i] receives the handle of
 * stack i (n entries). Without PA_CFG_RETIRE_STACKS the handles are the consecutive ids. With it, a stack takes the lowest free
 * slot (with that slot's next generation) or else a new slot, so the handles need not be consecutive. */
int pa_agg_register_stack_handles(pa_agg* a, const uint64_t* hashes, const uint64_t* frames, const uint64_t* offsets, uint32_t n, uint64_t* handles);
/* PA_CFG_RETIRE_STACKS only. Call it between flushes, from the flushing thread (ingest and registration may run meanwhile);
 * PA_EINVAL while a staged batch has not been collected, for idle_batches == 0, and on other aggregators.
 * Retires every live stack that is idle for idle_batches batches: registered before the last idle_batches batches were staged,
 * and named by none of them. At most `cap` are retired, lowest slot first; their handles go to handles[] in ascending slot order
 * and their count to *n_retired. Idle stacks beyond `cap` stay live; a later call finds them.
 * Grace rule: rows of the NEXT batch may still name a retired stack and come out exactly right (rows a producer committed before
 * the caller forgot the handle). The stack is freed when the batch after that one is staged; from then on its slot may go to a new
 * registration. The caller drops the returned handles from its own lookup before its next flush.
 * Counters through pa_agg_last_kernel_ms (in *launches, ms = 0, saturating at 2^32 - 1): "stacks_live" (registered and not yet
 * freed), "stacks_free" (free slots), "stack_frames_live" (their frames), "stack_frames_dead" (frames of freed stacks still in the
 * device arena), "stack_compactions" and "stacks_retired" (since creation). "stack_compact" reports the device time (ms) and kernel
 * launches of the last arena compaction. These names fail with PA_EINVAL on aggregators without PA_CFG_RETIRE_STACKS. */
int pa_agg_retire_stacks(pa_agg* a, uint32_t idle_batches, uint64_t* handles, uint64_t cap, uint64_t* n_retired);

/* ingest — ReportTraceEvent (:219). Thread-safe; row order == acquisition order (the mutex at :335).
 * acquire reserves space for n_rows headers / n_frames frame ids in the pinned ring and returns
 * where to write them (no Go pointers are retained: the ring is C-owned). *frame_base is the
 * frame_off of the first reserved frame id. commit publishes the rows. */
int pa_agg_acquire(pa_agg* a, uint64_t n_rows, uint64_t n_frames, pa_sample_hdr** hdrs, uint64_t** frames, uint64_t* frame_base);
int pa_agg_commit(pa_agg* a, uint64_t n_rows);
/* copying convenience: frames of row i are frames[sum(nframes[0..i))..]; frame_off is filled in. */
int pa_agg_submit(pa_agg* a, const pa_sample_hdr* hdrs, const uint64_t* frames, uint64_t n_rows);

/* flush — buildSampleRecordV2 (:1742) + IPC (:1779-1790): swap the ring buffer under the ingest
 * lock, run the GPU pipeline on the detached buffer, return the finished IPC stream. */
int pa_agg_flush(pa_agg* a, pa_agg_result* out);
void pa_agg_release(pa_agg* a, pa_agg_result* res);

/* v1 schema only — buildStacktraceRecord (:1545-1739) + LocationsWriter.NewRecord (arrow.go:230-254) + IPC
 * (:1336-1349 offline, :1470-1500 gRPC): the record {stacktrace_id: Binary, is_complete: Bool, locations:
 * List<Struct<...>>} for n_ids 16-byte stack ids (big-endian hi||lo, as in the sample record's stacktrace_id
 * dictionary), resolved against the device-resident store of known stacks that every v1 flush feeds (the
 * `stacks` LRU, :224-227). An id that is not (or no longer) in the store yields the reference's
 * "missing stacktrace" row (:1556-1573). out->n_rows = n_ids, out->n_locations = flattened locations.
 * The result replaces the previous flush/stacktraces result (same pinned output buffer). */
int pa_agg_stacktraces(pa_agg* a, const uint8_t* ids, uint64_t n_ids, pa_agg_result* out);
/* v1: the unique stack ids of the batch most recently processed, first-occurrence order (== the stacktrace_id
 * dictionary of its sample record, the ids the reference walks at :1307-1328). out has 16*n bytes. */
int pa_agg_last_stack_ids(pa_agg* a, uint8_t* out, uint64_t n);

/* bench / profiling hooks: the same pipeline split in its three stages.
 * stage = swap + H2D only; process = kernels only on the HBM-resident batch (repeatable);
 * collect = D2H + IPC framing. flush == stage; process; collect. */
int pa_agg_stage(pa_agg* a);
int pa_agg_process(pa_agg* a);
int pa_agg_collect(pa_agg* a, pa_agg_result* out);
/* device time (ms, CUDA events on the compute stream) of named kernel groups during the last
 * process(): names are "hash", "header", "rank", "locations", "labels", "dicts", "total". "lz4" reports the compression kernels of
 * the last collect / pa_agg_stacktraces in PA_IPC_LZ4_FRAME_GPU mode. Two more names report counters of the
 * v1 stack store since creation in *launches (ms = 0): "store_compactions", "store_evictions". Two more report the label
 * column plan in *launches (ms = 0): "label_columns", the labelset-derived label columns planned for the last pass (a pass plans
 * the label names the previous batch's rows used plus every name registered since; at most 246 label columns, cpu / thread_id /
 * thread_name included, per batch), and "label_replans", the passes redone since creation because a batch's rows used a
 * label name the plan had left out. */
int pa_agg_last_kernel_ms(const pa_agg* a, const char* name, double* ms, uint32_t* launches);
/* copies the per-row 128-bit stack ids (big-endian hi‖lo, 16 B per row) of the staged batch. */
int pa_agg_debug_stack_ids(pa_agg* a, uint8_t* out, uint64_t n_rows);
/* per-unique-stack occurrence counts in first-occurrence order (the "count per stack" side table;
 * not part of the reference's record — see SURVEY §0.2 — and therefore computed on demand by a separate
 * kernel over the batch most recently processed, not on the flush path). out has n_unique_stacks entries. */
int pa_agg_debug_stack_counts(pa_agg* a, uint32_t* out, uint64_t n);
/* the same batch as (labelset, stack) -> count: one entry per distinct pair in first-occurrence order; stack is the
 * first-occurrence ordinal of the stack (index into the counts above). Also on demand and off the flush path. Up to
 * `cap` entries are written; *n_pairs receives the number of distinct pairs (call again with a larger cap if it is bigger). */
int pa_agg_debug_pair_counts(pa_agg* a, uint32_t* labelset_ids, uint32_t* stack_ordinals, uint32_t* counts, uint64_t cap, uint64_t* n_pairs);

/* ---- multi-GPU, one merged batch for an ARBITRARY interleaving of the shards' rows (round-1 path; moves 72 B per row to
 * the merging GPU — prefer pa_merge_* below, which exchanges dictionary keys only) -------------------------------------
 * The sample stream is sharded by pid hash, one aggregator per GPU. Per-shard batches (mode A) need nothing more. For
 * ONE batch that is bit-identical to the unsharded stream's, every shard aggregator (PA_SCHEMA_V2) runs stage + process,
 * exports its rows and the frames of its unique stacks into device buffers the caller owns, the caller moves them to
 * the merging GPU (NCCL send/recv over NVLink: 64 B per row + 8 B per unique-stack frame) and places the rows at their
 * positions in the global order, and a PA_HASH_PROVIDED aggregator there stages that union from device memory and
 * runs the usual process + collect. All aggregators must have been registered the same strings / frames / labelsets. */
/* sizes of what pa_agg_shard_export will write for the batch last processed (rows, frame ids) */
int pa_agg_shard_sizes(pa_agg* a, uint64_t* n_rows, uint64_t* n_frames);
/* hdr_out: n_rows pa_sample_hdr (device memory) with hash_hi/lo = the stack id, nframes = the kept stack's depth and
 * frame_off = frame_base + offset of the stack's frames inside frames_out; frames_out: n_frames uint64 (device).
 * Synchronous: the buffers are complete when the call returns. */
int pa_agg_shard_export(pa_agg* a, uint64_t frame_base, pa_sample_hdr* hdr_out, uint64_t* frames_out);
/* drop the staged batch without building its record (a shard whose rows have been exported does not need its own) */
int pa_agg_discard(pa_agg* a);
/* stage a batch that already lives in device memory (rows in final order, frame_off relative to frames) instead of the
 * pinned ring; the caller's writes to both buffers must have completed. Follow with pa_agg_process + pa_agg_collect. */
int pa_agg_stage_device(pa_agg* a, const pa_sample_hdr* hdr, uint64_t n_rows, const uint64_t* frames, uint64_t n_frames);

/* the same, with the scatter to global row order done by the library: part p holds n_rows headers whose positions in the
 * merged batch are global_row[i] (all parts together must cover 0..n_rows_total-1 exactly once) and the frames its
 * headers' frame_off point into, already based so that the parts' frame blocks concatenate in part order. */
typedef struct pa_device_part {
  const pa_sample_hdr* hdr;
  const uint64_t* global_row;
  uint64_t n_rows;
  const uint64_t* frames;
  uint64_t n_frames;
} pa_device_part;
int pa_agg_stage_device_parts(pa_agg* a, const pa_device_part* parts, uint32_t n_parts, uint64_t n_rows_total);

/* ---- multi-GPU, one merged batch with an O(unique keys) exchange (SURVEY section 8e; "mode B, slices") ------------------
 * A group of shard aggregators (one schema, identical string / frame / labelset registrations, one per GPU ring) builds
 * ONE record batch: the reference's record (reporter/parca_reporter.go:1742-1790) for the sample stream
 * [shard 0's rows, shard 1's rows, ...]. Rows never leave the GPU that ingested them; only dictionary keys cross NVLink
 * (stack ids to their owner shard and back as one merged list, min-reductions of the first-occurrence tables, thread-id lists,
 * per-column run edges). Every first-occurrence dictionary index (arrow_v2.go:191, :302; parca_reporter.go:425) and every run
 * (arrow.go:97-131, merged across shard borders) comes out exactly as the reference would produce it on that stream.
 *   pa_merge_create_local : every member in this process and on ONE device (device copies instead of NCCL)
 *   pa_merge_create_nccl  : one member per call; NCCL (libnccl.so.2, loaded on first use) over NVLink / NVSwitch. Rank 0
 *                           obtains the 128-byte id from pa_merge_nccl_unique_id and hands it to every rank (the host agent's job).
 * Per interval, on every rank: pa_agg_stage (or ingest + pa_merge_flush) -> pa_merge_process -> pa_merge_plan -> pa_merge_collect.
 * All three are collective. pa_merge_collect writes this process's members' parts of the stream into `base`, a buffer of at
 * least *ipc_len bytes that ALL processes of the group share (e.g. a POSIX shared-memory mapping; it is page-locked on first
 * use); rank 0 adds the dictionaries and the metadata, and gets out->ipc == base. base == NULL: groups whose members all live
 * in this process use a library-owned pinned buffer.
 * LZ4 groups (every member PA_IPC_LZ4_FRAME_GPU): the record and dictionary batch bodies are LZ4_FRAME-compressed on the members'
 * GPUs, on each buffer's own 64 KiB block grid, so the stream is byte-identical to one PA_IPC_LZ4_FRAME_GPU aggregator's on the
 * concatenated rows. pa_merge_plan runs the compression (a block that crosses a shard border is assembled by the shard that holds
 * its first byte, from the following shards' heads, exchanged once) and returns the COMPRESSED *ipc_len, the same on every
 * rank; pa_merge_collect packs each member's blocks and copies them to their places, rank 0 adds metadata and framing.
 * pa_agg_last_kernel_ms(member, "lz4", ...) reports each member's share of the compression kernels, and "lz4_heads" (in
 * *launches, ms = 0) the bytes of block heads the member sent in the last plan. Mixed groups: pa_merge_create_local refuses
 * them (the reason goes to the PA_IPC_LZ4_FRAME_GPU members' pa_agg_last_error); groups with one member per process find out
 * in pa_merge_process, which then fails with PA_EINVAL on every rank before any work.
 * v1 groups (every member PA_SCHEMA_V1, with equal store sizes: stack_cache_entries / stack_cache_frames as they resolve — left
 * at 0 they follow max_samples, so members with different rings need explicit, equal values): the group behaves, interval by
 * interval, like ONE v1 aggregator fed the concatenated rows — the sample record, pa_agg_stacktraces, pa_agg_last_stack_ids and
 * the "store_evictions" / "store_compactions" counters. Every member holds a full copy of the group's known-stacks store and
 * pa_merge_process applies the merged batch's accesses to each copy (it exchanges the global last row of every merged stack and
 * the frames of the stacks the store lacks; pa_agg_last_kernel_ms(member, "store_frames", ...) reports, in *launches, the frame
 * ids the member sent in the last pa_merge_process). PA_CFG_GROUP_STACKS groups send one 8-byte offset into the registered frame
 * arena per stack instead of its frames (every member holds the same arena): "store_refs" reports those offsets the same way,
 * and "store_frames" is 0. An error any member's store update finds (e.g. an unregistered frame id,
 * seen only by the shard that sends that stack's frames) fails pa_merge_process on every rank. After a merged interval pa_agg_last_stack_ids on any member returns the merged dictionary, and a member
 * flushed on its own continues from the group's store. A group that mixes schemas, or v1 members with different store sizes, is
 * refused like a mixed LZ4 group (pa_merge_create_local at once, with the reason in every member's pa_agg_last_error;
 * multi-process groups in pa_merge_process on every rank).
 *   pa_merge_create_host  : one member per call; the caller supplies the four collectives on HOST buffers (MPI, gloo, sockets ...):
 *                           the library stages device buffers through pinned memory around them. For hosts without NCCL, and for
 *                           exercising the multi-process path on one GPU (two processes may share a device). */
typedef struct pa_merge pa_merge;
/* Collectives over the `world` ranks of the group, on host memory; every callback returns 0 on success. Byte counts.
 *   allgather         recv[r*bytes .. ) = rank r's send
 *   allgatherv        recv[displs[r] .. +counts[r]) = rank r's send (counts[my rank] bytes)
 *   alltoallv         send[sdispls[r] .. +scounts[r]) goes to rank r; recv[rdispls[r] .. +rcounts[r]) comes from rank r
 *   allreduce_min_u32 element-wise minimum over all ranks, in place */
typedef struct pa_merge_host_transport {
  void* user;
  int (*allgather)(void* user, const void* send, void* recv, uint64_t bytes);
  int (*allgatherv)(void* user, const void* send, void* recv, const uint64_t* counts, const uint64_t* displs);
  int (*alltoallv)(void* user, const void* send, const uint64_t* scounts, const uint64_t* sdispls, void* recv, const uint64_t* rcounts, const uint64_t* rdispls);
  int (*allreduce_min_u32)(void* user, uint32_t* buf, uint64_t count);
} pa_merge_host_transport;
int pa_merge_create_host(pa_agg* member, const pa_merge_host_transport* t, uint32_t rank, uint32_t world, pa_merge** out);
/* one member per call; the exchange runs through ONE POSIX shared-memory segment `name` ("/...", created by rank 0, mapped and page-locked by
 * every rank): each GPU copies its keys into its own mailbox and the blocks it needs out of the others' over its own PCIe link, with
 * process-shared barriers in between. Needs nothing but CUDA and /dev/shm. mailbox_bytes: 0 = 64 MiB per rank (larger payloads go in rounds). */
int pa_merge_create_shm(pa_agg* member, const char* name, uint32_t rank, uint32_t world, uint64_t mailbox_bytes, pa_merge** out);
int pa_merge_create_local(pa_agg* const* members, uint32_t n, pa_merge** out);
int pa_merge_nccl_unique_id(uint8_t* id128);
int pa_merge_create_nccl(pa_agg* member, const uint8_t* id128, uint32_t rank, uint32_t world, pa_merge** out);
void pa_merge_destroy(pa_merge* m);
const char* pa_merge_last_error(const pa_merge* m);
int pa_merge_process(pa_merge* m);
int pa_merge_plan(pa_merge* m, uint64_t* ipc_len);
int pa_merge_collect(pa_merge* m, uint8_t* base, uint64_t cap, pa_agg_result* out);
/* in-process groups: ring swap + H2D of every member, the merged pass, plan and collect in one call */
int pa_merge_flush(pa_merge* m, pa_agg_result* out);
/* PA_CFG_GROUP_RETIRE groups, between intervals (collective: every rank calls it after pa_merge_collect, with the same arguments).
 * pa_agg_retire_stacks for the whole group, with the same rules (idle window, cap, lowest slot first, grace batch): a stack is idle
 * when no member's rows named it in the window. Every rank receives the same handles in handles[] (ascending slot order) and
 * *n_retired, and every member frees the same slots at the same stage. PA_EINVAL on every rank, with nothing retired, for
 * idle_batches == 0, a member whose staged batch is not collected, a member without the flag, and ranks that disagree on
 * idle_batches, cap, stage count or uploaded slot count. handles[] receives at most min(cap, uploaded slots) entries, so a caller
 * that wants every idle stack may pass cap = UINT64_MAX (the same on every rank) with room for its member's slots. Registrations
 * may run concurrently on any member (the registry digest keeps registrations and retirements apart, so their interleaving on
 * each member does not matter). The caller drops the returned handles from its lookup before the next interval's rows are
 * written. */
int pa_merge_retire_stacks(pa_merge* m, uint32_t idle_batches, uint64_t* handles, uint64_t cap, uint64_t* n_retired);
/* v1 groups, between intervals (collective): the stacktrace record (pa_agg_stacktraces) for rank 0's request. Rank 0 passes the
 * server's ids, the other ranks NULL / 0 (the ids reach them in one all-gather). Every member applies the request's accesses to
 * its copy of the store, and each rank's *out is the record its own member built: the same bytes on every rank (in-process
 * groups: member 0's). The result is that member's, as if it came from pa_agg_stacktraces on it: out->ipc lives in the member's
 * pinned output buffer, is replaced by its next flush / collect / stacktrace request, and is released with
 * pa_agg_release(member, out). PA_EINVAL for v2 groups, and before the merged batch is collected. */
int pa_merge_stacktraces(pa_merge* m, const uint8_t* ids, uint64_t n_ids, pa_agg_result* out);
/* wall-clock of the last pa_merge_process, the part of it spent waiting in the three size exchanges, the payload bytes this
 * process's members sent to other ranks (NCCL groups), and the merged row count */
int pa_merge_last_stats(const pa_merge* m, double* wall_ms, double* exchange_wait_ms, uint64_t* nvlink_bytes, uint64_t* n_rows_total);

/* LZ4_FRAME body compression of a finished, uncompressed stream written by this library (what PA_IPC_LZ4_FRAME applies to
 * every result). Host only; uses the system liblz4.so.1 through dlopen and fails with PA_EIO when it is missing. *out is
 * malloc'ed; release it with pa_ipc_free. Flagged: not byte-identical to arrow-go + pierrec/lz4, only record-identical. */
int pa_ipc_compress_lz4(const uint8_t* ipc, uint64_t len, uint8_t** out, uint64_t* out_len);
void pa_ipc_free(uint8_t* p);

/* host helpers restating reference functions (no GPU involved) */
/* maybeFixTruncation (reporter/parca_reporter.go:190-216): returns the fixed length, or -1. */
int64_t pa_fix_truncation(const uint8_t* s, uint64_t len, uint64_t max_len);
uint64_t pa_xxh64(const void* data, uint64_t len, uint64_t seed);

#ifdef __cplusplus
}
#endif
#endif /* PARCAAGG_H */
