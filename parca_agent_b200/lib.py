"""ctypes binding of libparcaagg.so (include/parcaagg.h) — the product's only compute path.

There is deliberately no CPU fallback: if the CUDA library is missing or no device is usable,
importing/constructing fails loudly. Nothing here imports the test oracle.
"""
import ctypes as C
import os

import numpy as np

from . import abi

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libparcaagg.so")
_LIB = None

EXPORTS = [
    "pa_agg_create", "pa_agg_destroy", "pa_agg_last_error", "pa_agg_abi_version", "pa_agg_register_strings",
    "pa_agg_register_frames", "pa_agg_register_labelsets", "pa_agg_register_stacks", "pa_agg_acquire", "pa_agg_commit", "pa_agg_submit",
    "pa_agg_flush", "pa_agg_release", "pa_agg_stage", "pa_agg_process", "pa_agg_collect", "pa_agg_last_kernel_ms",
    "pa_agg_debug_stack_ids", "pa_agg_debug_stack_counts", "pa_agg_debug_pair_counts", "pa_agg_stacktraces", "pa_agg_last_stack_ids", "pa_agg_shard_sizes", "pa_agg_shard_export", "pa_agg_stage_device", "pa_agg_stage_device_parts", "pa_agg_discard", "pa_ipc_compress_lz4", "pa_ipc_free", "pa_fix_truncation", "pa_xxh64",
    "pa_merge_create_local", "pa_merge_nccl_unique_id", "pa_merge_create_nccl", "pa_merge_destroy", "pa_merge_last_error", "pa_merge_process",
    "pa_merge_plan", "pa_merge_collect", "pa_merge_flush", "pa_merge_last_stats", "pa_merge_create_host", "pa_merge_create_shm",
    "pa_merge_stacktraces", "pa_agg_register_stack_handles", "pa_agg_retire_stacks", "pa_merge_retire_stacks",
]


class PaError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("libparcaagg error %d: %s" % (code, msg))
        self.code = code


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError("libparcaagg.so is not built (%s). Run `python -c 'import __graft_entry__ as g; g.build()'`; "
                               "there is no CPU fallback." % LIB_PATH)
        L = C.CDLL(LIB_PATH)
        vp, u32p, u64p = C.c_void_p, C.POINTER(C.c_uint32), C.POINTER(C.c_uint64)
        L.pa_agg_create.argtypes = [C.POINTER(abi.PaAggConfig), C.POINTER(vp)]
        L.pa_agg_destroy.argtypes = [vp]
        L.pa_agg_destroy.restype = None
        L.pa_agg_last_error.argtypes = [vp]
        L.pa_agg_last_error.restype = C.c_char_p
        L.pa_agg_abi_version.restype = C.c_uint32
        L.pa_agg_register_strings.argtypes = [vp, C.c_char_p, vp, C.c_uint32, u32p]
        L.pa_agg_register_frames.argtypes = [vp, vp, C.c_uint32, u64p]
        L.pa_agg_register_labelsets.argtypes = [vp, vp, vp, C.c_uint32, u32p]
        L.pa_agg_register_stacks.argtypes = [vp, vp, vp, vp, C.c_uint32, u64p]
        L.pa_agg_register_stack_handles.argtypes = [vp, vp, vp, vp, C.c_uint32, vp]
        L.pa_agg_retire_stacks.argtypes = [vp, C.c_uint32, vp, C.c_uint64, u64p]
        L.pa_merge_retire_stacks.argtypes = [vp, C.c_uint32, vp, C.c_uint64, u64p]
        L.pa_agg_acquire.argtypes = [vp, C.c_uint64, C.c_uint64, C.POINTER(vp), C.POINTER(vp), u64p]
        L.pa_agg_commit.argtypes = [vp, C.c_uint64]
        L.pa_agg_submit.argtypes = [vp, vp, vp, C.c_uint64]
        L.pa_agg_flush.argtypes = [vp, C.POINTER(abi.PaAggResult)]
        L.pa_agg_release.argtypes = [vp, C.POINTER(abi.PaAggResult)]
        L.pa_agg_release.restype = None
        L.pa_agg_stage.argtypes = [vp]
        L.pa_agg_process.argtypes = [vp]
        L.pa_agg_collect.argtypes = [vp, C.POINTER(abi.PaAggResult)]
        L.pa_agg_last_kernel_ms.argtypes = [vp, C.c_char_p, C.POINTER(C.c_double), u32p]
        L.pa_agg_debug_stack_ids.argtypes = [vp, vp, C.c_uint64]
        L.pa_agg_debug_stack_counts.argtypes = [vp, vp, C.c_uint64]
        L.pa_agg_debug_pair_counts.argtypes = [vp, vp, vp, vp, C.c_uint64, u64p]
        L.pa_agg_shard_sizes.argtypes = [vp, u64p, u64p]
        L.pa_agg_shard_export.argtypes = [vp, C.c_uint64, vp, vp]
        L.pa_agg_discard.argtypes = [vp]
        L.pa_ipc_compress_lz4.argtypes = [C.c_char_p, C.c_uint64, C.POINTER(C.POINTER(C.c_uint8)), u64p]
        L.pa_ipc_free.argtypes = [C.POINTER(C.c_uint8)]
        L.pa_ipc_free.restype = None
        L.pa_agg_stage_device_parts.argtypes = [vp, C.POINTER(abi.PaDevicePart), C.c_uint32, C.c_uint64]
        L.pa_agg_stage_device.argtypes = [vp, vp, C.c_uint64, vp, C.c_uint64]
        L.pa_agg_stacktraces.argtypes = [vp, C.c_char_p, C.c_uint64, C.POINTER(abi.PaAggResult)]
        L.pa_agg_last_stack_ids.argtypes = [vp, vp, C.c_uint64]
        L.pa_fix_truncation.argtypes = [C.c_char_p, C.c_uint64, C.c_uint64]
        L.pa_fix_truncation.restype = C.c_int64
        L.pa_xxh64.argtypes = [vp, C.c_uint64, C.c_uint64]
        L.pa_xxh64.restype = C.c_uint64
        L.pa_merge_create_local.argtypes = [C.POINTER(vp), C.c_uint32, C.POINTER(vp)]
        L.pa_merge_nccl_unique_id.argtypes = [C.c_char_p]
        L.pa_merge_create_nccl.argtypes = [vp, C.c_char_p, C.c_uint32, C.c_uint32, C.POINTER(vp)]
        L.pa_merge_create_host.argtypes = [vp, vp, C.c_uint32, C.c_uint32, C.POINTER(vp)]
        L.pa_merge_create_shm.argtypes = [vp, C.c_char_p, C.c_uint32, C.c_uint32, C.c_uint64, C.POINTER(vp)]
        L.pa_merge_destroy.argtypes = [vp]
        L.pa_merge_destroy.restype = None
        L.pa_merge_last_error.argtypes = [vp]
        L.pa_merge_last_error.restype = C.c_char_p
        L.pa_merge_process.argtypes = [vp]
        L.pa_merge_plan.argtypes = [vp, u64p]
        L.pa_merge_collect.argtypes = [vp, vp, C.c_uint64, C.POINTER(abi.PaAggResult)]
        L.pa_merge_flush.argtypes = [vp, C.POINTER(abi.PaAggResult)]
        L.pa_merge_last_stats.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_double), u64p, u64p]
        L.pa_merge_stacktraces.argtypes = [vp, C.c_char_p, C.c_uint64, C.POINTER(abi.PaAggResult)]
        _LIB = L
    return _LIB


class Result:
    """One flushed batch. `ipc` is a zero-copy view of library-owned pinned memory, valid until the next flush."""

    def __init__(self, raw):
        self.n_rows = int(raw.n_rows)
        self.n_unique_stacks = int(raw.n_unique_stacks)
        self.n_locations = int(raw.n_locations)
        self.n_functions = int(raw.n_functions)
        self.n_location_indices = int(raw.n_location_indices)
        self.gpu_launches = int(raw.gpu_launches)
        self.h2d_ms, self.gpu_ms, self.d2h_ms, self.host_ms = raw.h2d_ms, raw.gpu_ms, raw.d2h_ms, raw.host_ms
        n = int(raw.ipc_len)
        self.ipc_len = n
        self.ipc = np.ctypeslib.as_array(raw.ipc, shape=(n,)) if n else np.zeros(0, np.uint8)

    def ipc_bytes(self):
        return self.ipc.tobytes()


class Aggregator:
    """Thin object wrapper over one pa_agg handle."""

    def __init__(self, device=0, hash_mode=abi.PA_HASH_XXH64X2, label_flags=0, samples_per_second=19, external_labels=(),
                 max_samples=1 << 20, max_frames=0, chunk_samples=0, schema=abi.PA_SCHEMA_V2, stack_cache_entries=0, stack_cache_frames=0,
                 unknown_frame_type_sid=0, ipc_compression=abi.PA_IPC_PLAIN, frame_id_bytes=8, flags=0):
        L = lib()
        ext = (abi.PaLabelPair * max(1, len(external_labels)))()
        for i, (n, v) in enumerate(external_labels):
            ext[i].name_sid, ext[i].value_sid = int(n), int(v)
        cfg = abi.PaAggConfig(abi_version=abi.PA_ABI_VERSION, device=device, hash_mode=hash_mode, label_flags=label_flags,
                              samples_per_second=samples_per_second, n_external_labels=len(external_labels), external_labels=ext,
                              max_samples=max_samples, max_frames=max_frames, chunk_samples=chunk_samples, schema=schema,
                              stack_cache_entries=stack_cache_entries, stack_cache_frames=stack_cache_frames, unknown_frame_type_sid=unknown_frame_type_sid,
                              ipc_compression=ipc_compression, frame_id_bytes=frame_id_bytes, flags=flags)
        h = C.c_void_p()
        rc = L.pa_agg_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise PaError(rc, "pa_agg_create failed (no CUDA device, bad config or out of memory)")
        self.h = h
        self.max_samples = max_samples
        self.id_dtype = np.uint32 if frame_id_bytes == 4 else np.uint64  # what the ring holds per frame id
        self.registered = bool(flags & abi.PA_CFG_REGISTERED_STACKS)

    def _ck(self, rc):
        if rc != 0:
            raise PaError(rc, (lib().pa_agg_last_error(self.h) or b"").decode(errors="replace"))

    def close(self):
        if getattr(self, "h", None):
            lib().pa_agg_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- registration
    def register_strings(self, strs):
        blob, offs = abi.pack_strings(list(strs))
        first = C.c_uint32()
        self._ck(lib().pa_agg_register_strings(self.h, blob, offs.ctypes.data, len(strs), C.byref(first)))
        return first.value

    def register_frames(self, descs):
        descs = np.ascontiguousarray(descs, dtype=abi.FRAME_DTYPE)
        first = C.c_uint64()
        self._ck(lib().pa_agg_register_frames(self.h, descs.ctypes.data, len(descs), C.byref(first)))
        return first.value

    def register_labelsets(self, labelsets):
        pairs, offs = abi.pack_labelsets(labelsets)
        first = C.c_uint32()
        self._ck(lib().pa_agg_register_labelsets(self.h, pairs.ctypes.data, offs.ctypes.data, len(labelsets), C.byref(first)))
        return first.value

    def register_stacks(self, frames, offsets, hashes=None):
        """PA_CFG_REGISTERED_STACKS: stack i = frames[offsets[i]:offsets[i+1]]; hashes (n, 2) [hash_hi, hash_lo] in
        PA_HASH_PROVIDED mode, None in PA_HASH_XXH64X2 mode. Returns the id of the first stack."""
        frames = np.ascontiguousarray(frames, dtype=self.id_dtype)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = len(offsets) - 1
        if hashes is not None:
            hashes = np.ascontiguousarray(hashes, dtype=np.uint64).reshape(-1)
        first = C.c_uint64()
        self._ck(lib().pa_agg_register_stacks(self.h, None if hashes is None else hashes.ctypes.data, frames.ctypes.data if len(frames) else None,
                                              offsets.ctypes.data, n, C.byref(first)))
        return first.value

    def register_stack_handles(self, frames, offsets, hashes=None):
        """register_stacks for either registered mode: a uint64 array with the handle of each stack (PA_CFG_RETIRE_STACKS:
        generation << 32 | slot; otherwise the consecutive ids)."""
        frames = np.ascontiguousarray(frames, dtype=self.id_dtype)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        n = len(offsets) - 1
        if hashes is not None:
            hashes = np.ascontiguousarray(hashes, dtype=np.uint64).reshape(-1)
        out = np.zeros(max(n, 1), dtype=np.uint64)
        self._ck(lib().pa_agg_register_stack_handles(self.h, None if hashes is None else hashes.ctypes.data, frames.ctypes.data if len(frames) else None,
                                                     offsets.ctypes.data, n, out.ctypes.data))
        return out[:n]

    def retire_stacks(self, idle_batches, cap=None):
        """PA_CFG_RETIRE_STACKS: retire the stacks idle for `idle_batches` batches (at most `cap`, default all); returns their
        handles in slot order. Drop them from any lookup before the next flush."""
        cap = self.stack_counters()["stacks_live"] if cap is None else cap
        out = np.zeros(max(cap, 1), dtype=np.uint64)
        n = C.c_uint64()
        self._ck(lib().pa_agg_retire_stacks(self.h, idle_batches, out.ctypes.data, cap, C.byref(n)))
        return out[:n.value]

    def stack_counters(self):
        """PA_CFG_RETIRE_STACKS: the stack registry's counters (pa_agg_last_kernel_ms names)."""
        return {k: self.kernel_ms(k)[1] for k in ("stacks_live", "stacks_free", "stack_frames_live", "stack_frames_dead", "stack_compactions", "stacks_retired")}

    # ---- ingest
    def submit(self, hdrs, frame_ids):
        hdrs = np.ascontiguousarray(hdrs, dtype=abi.HDR_DTYPE)
        frame_ids = np.ascontiguousarray(frame_ids, dtype=self.id_dtype)
        self._keep = (hdrs, frame_ids)
        self._ck(lib().pa_agg_submit(self.h, hdrs.ctypes.data, frame_ids.ctypes.data, len(hdrs)))

    def acquire(self, n_rows, n_frames):
        """Reserve ring space; returns (hdr view, frame-id view, frame_base). Write, then commit()."""
        ph, pf, base = C.c_void_p(), C.c_void_p(), C.c_uint64()
        self._ck(lib().pa_agg_acquire(self.h, n_rows, n_frames, C.byref(ph), C.byref(pf), C.byref(base)))
        hv = np.ctypeslib.as_array(C.cast(ph, C.POINTER(C.c_uint8)), shape=(max(n_rows, 1) * 64,))[:n_rows * 64].view(abi.HDR_DTYPE)
        ctype = C.c_uint32 if self.id_dtype == np.uint32 else C.c_uint64
        if not pf.value:  # registered stacks: the ring holds no frame ids
            return hv, np.zeros(0, self.id_dtype), base.value
        fv = np.ctypeslib.as_array(C.cast(pf, C.POINTER(ctype)), shape=(max(n_frames, 1),))[:n_frames]
        return hv, fv, base.value

    def commit(self, n_rows):
        self._ck(lib().pa_agg_commit(self.h, n_rows))

    # ---- flush and its three stages
    def _result(self, fn):
        raw = abi.PaAggResult()
        self._ck(fn(self.h, C.byref(raw)))
        return Result(raw)

    def flush(self):
        return self._result(lib().pa_agg_flush)

    def stage(self):
        self._ck(lib().pa_agg_stage(self.h))

    def process(self):
        self._ck(lib().pa_agg_process(self.h))

    def collect(self):
        return self._result(lib().pa_agg_collect)

    def debug_pair_counts(self, cap):
        """(labelset id, stack ordinal, count) of every distinct pair of the processed batch, first-occurrence order."""
        ls, st, ct = (np.zeros(max(cap, 1), dtype=np.uint32) for _ in range(3))
        n = C.c_uint64()
        self._ck(lib().pa_agg_debug_pair_counts(self.h, ls.ctypes.data, st.ctypes.data, ct.ctypes.data, cap, C.byref(n)))
        m = min(int(n.value), cap)
        return ls[:m], st[:m], ct[:m], int(n.value)

    # ---- mode B building blocks (device pointers are plain integers, e.g. torch.Tensor.data_ptr())
    def shard_sizes(self):
        nr, nf = C.c_uint64(), C.c_uint64()
        self._ck(lib().pa_agg_shard_sizes(self.h, C.byref(nr), C.byref(nf)))
        return int(nr.value), int(nf.value)

    def shard_export(self, frame_base, hdr_ptr, frames_ptr):
        self._ck(lib().pa_agg_shard_export(self.h, frame_base, hdr_ptr, frames_ptr))

    def stage_device_parts(self, parts, n_rows_total):
        """parts: list of (hdr_ptr, global_row_ptr, n_rows, frames_ptr, n_frames) device buffers; rows are scattered to global order."""
        arr = (abi.PaDevicePart * max(len(parts), 1))()
        for i, (h, g, n, f, nf) in enumerate(parts):
            arr[i] = abi.PaDevicePart(h, g, n, f, nf)
        self._ck(lib().pa_agg_stage_device_parts(self.h, arr, len(parts), n_rows_total))

    def discard(self):
        self._ck(lib().pa_agg_discard(self.h))

    def stage_device(self, hdr_ptr, n_rows, frames_ptr, n_frames):
        self._ck(lib().pa_agg_stage_device(self.h, hdr_ptr, n_rows, frames_ptr, n_frames))

    def stacktraces(self, ids):
        """v1: the stacktrace record for the concatenated 16-byte ids (buildStacktraceRecord)."""
        ids = bytes(ids)
        assert len(ids) % 16 == 0
        raw = abi.PaAggResult()
        self._ck(lib().pa_agg_stacktraces(self.h, ids, len(ids) // 16, C.byref(raw)))
        return Result(raw)

    def last_stack_ids(self, n):
        out = np.zeros((n, 16), dtype=np.uint8)
        self._ck(lib().pa_agg_last_stack_ids(self.h, out.ctypes.data, n))
        return out

    def kernel_ms(self, name):
        ms, n = C.c_double(), C.c_uint32()
        self._ck(lib().pa_agg_last_kernel_ms(self.h, name.encode(), C.byref(ms), C.byref(n)))
        return ms.value, n.value

    def debug_stack_ids(self, n_rows):
        out = np.zeros((n_rows, 16), dtype=np.uint8)
        self._ck(lib().pa_agg_debug_stack_ids(self.h, out.ctypes.data, n_rows))
        return out

    def debug_stack_counts(self, n):
        out = np.zeros(n, dtype=np.uint32)
        self._ck(lib().pa_agg_debug_stack_counts(self.h, out.ctypes.data, n))
        return out


class MergeGroup:
    """Shard aggregators that build ONE merged record batch (mode B, include/parcaagg.h pa_merge_*). The merged batch is the
    record of the stream [member 0's rows, member 1's rows, ...]; only dictionary keys are exchanged between the GPUs."""

    def __init__(self, handle, members):
        self.h, self.members = handle, list(members)

    @classmethod
    def local(cls, members):
        """All members in this process, on one device (device copies instead of NCCL)."""
        arr = (C.c_void_p * len(members))(*[m.h for m in members])
        h = C.c_void_p()
        rc = lib().pa_merge_create_local(arr, len(members), C.byref(h))
        if rc != 0:
            raise PaError(rc, "pa_merge_create_local failed")
        return cls(h, members)

    @staticmethod
    def nccl_unique_id():
        buf = C.create_string_buffer(128)
        rc = lib().pa_merge_nccl_unique_id(buf)
        if rc != 0:
            raise PaError(rc, "pa_merge_nccl_unique_id failed (libnccl.so.2 not loadable?)")
        return buf.raw

    @classmethod
    def nccl(cls, member, unique_id, rank, world):
        """One member per process / per GPU; `unique_id` comes from rank 0's nccl_unique_id()."""
        h = C.c_void_p()
        rc = lib().pa_merge_create_nccl(member.h, bytes(unique_id), rank, world, C.byref(h))
        if rc != 0:
            raise PaError(rc, "pa_merge_create_nccl failed")
        return cls(h, [member])

    @classmethod
    def host(cls, member, transport, rank, world):
        """One member per process; `transport` provides the collectives on host buffers (host_transport.GlooTransport)."""
        h = C.c_void_p()
        rc = lib().pa_merge_create_host(member.h, C.byref(transport.struct), rank, world, C.byref(h))
        if rc != 0:
            raise PaError(rc, "pa_merge_create_host failed")
        g = cls(h, [member])
        g._transport = transport  # the callbacks must outlive the group
        return g

    @classmethod
    def shm(cls, member, name, rank, world, mailbox_bytes=0):
        """One member per process; the exchange goes through the POSIX shared-memory segment `name` ("/..."), which rank 0 creates
        and every rank page-locks: GPU -> own mailbox -> the other GPUs, each over its own PCIe link. No NCCL, no sockets."""
        h = C.c_void_p()
        rc = lib().pa_merge_create_shm(member.h, name.encode(), rank, world, mailbox_bytes, C.byref(h))
        if rc != 0:
            raise PaError(rc, "pa_merge_create_shm failed")
        return cls(h, [member])

    def _ck(self, rc):
        if rc != 0:
            extra = "; ".join(getattr(getattr(self, "_transport", None), "errors", []) or [])
            raise PaError(rc, (lib().pa_merge_last_error(self.h) or b"").decode(errors="replace") + (" | " + extra if extra else ""))

    def process(self):
        self._ck(lib().pa_merge_process(self.h))

    def plan(self):
        n = C.c_uint64()
        self._ck(lib().pa_merge_plan(self.h, C.byref(n)))
        return int(n.value)

    def collect(self, base_ptr=None, cap=0):
        raw = abi.PaAggResult()
        self._ck(lib().pa_merge_collect(self.h, base_ptr, cap, C.byref(raw)))
        return Result(raw) if raw.ipc else _HeadlessResult(raw)

    def flush(self):
        raw = abi.PaAggResult()
        self._ck(lib().pa_merge_flush(self.h, C.byref(raw)))
        return Result(raw)

    def stacktraces(self, ids=None):
        """v1 groups (collective): the stacktrace record for rank 0's concatenated 16-byte ids; other ranks pass None. Every rank
        gets its own member's record (the same bytes everywhere), valid until that member's next flush or request."""
        ids = b"" if ids is None else bytes(ids)
        assert len(ids) % 16 == 0
        raw = abi.PaAggResult()
        self._ck(lib().pa_merge_stacktraces(self.h, ids or None, len(ids) // 16, C.byref(raw)))
        return Result(raw)

    def retire_stacks(self, idle_batches, cap=None):
        """PA_CFG_GROUP_RETIRE groups (collective, after collect): retire the stacks no member named for `idle_batches` batches
        (at most `cap`, default all); returns their handles in slot order, the same on every rank. Drop them from the lookup
        before the next interval. The default cap is the same on every rank (ranks must agree on it); the handle buffer is
        sized by this member's slots, never fewer than the uploaded slots the call selects from."""
        if cap is None:
            c = self.members[0].stack_counters()
            cap, room = 2**64 - 1, c["stacks_live"] + c["stacks_free"]
        else:
            room = cap
        out = np.zeros(max(room, 1), dtype=np.uint64)
        n = C.c_uint64()
        self._ck(lib().pa_merge_retire_stacks(self.h, idle_batches, out.ctypes.data, cap, C.byref(n)))
        return out[:n.value]

    def stats(self):
        wall, wait, nb, nr = C.c_double(), C.c_double(), C.c_uint64(), C.c_uint64()
        self._ck(lib().pa_merge_last_stats(self.h, C.byref(wall), C.byref(wait), C.byref(nb), C.byref(nr)))
        return {"wall_ms": wall.value, "exchange_wait_ms": wait.value, "nvlink_bytes": int(nb.value), "rows": int(nr.value)}

    def close(self):
        if getattr(self, "h", None):
            lib().pa_merge_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class _HeadlessResult(Result):
    """Result on a rank that does not hold the stream (every rank but 0 of a multi-process merge)."""

    def __init__(self, raw):
        n = int(raw.ipc_len)
        raw.ipc_len = 0
        super().__init__(raw)
        self.ipc_len = n


class StackForm:
    """A workload's rows in registered-stacks form: stack i = frames[offsets[i]:offsets[i+1]] with the stack id
    hashes[i] = (hash_hi, hash_lo) its rows carry, and stack_of_row[r] = the stack row r names (its frame_off)."""

    def __init__(self, hashes, frames, offsets, stack_of_row):
        self.hashes, self.frames, self.offsets, self.stack_of_row = hashes, frames, offsets, stack_of_row


def stack_form(w):
    """Workloads with a stack table register the table, with the id of each stack taken from the rows that name it (stacks no
    row names get id 0); the others (explicit frame streams) are deduplicated on (hash_hi, hash_lo, frame ids)."""
    if w._frame_ids is None:
        t = np.ascontiguousarray(w.stack_table, dtype=np.uint64)
        hashes = np.zeros((t.shape[0], 2), dtype=np.uint64)
        hashes[w.stack_choice, 0] = w.hdrs["hash_hi"]
        hashes[w.stack_choice, 1] = w.hdrs["hash_lo"]
        offsets = np.arange(t.shape[0] + 1, dtype=np.uint64) * np.uint64(t.shape[1])
        return StackForm(hashes, t.reshape(-1), offsets, np.asarray(w.stack_choice, dtype=np.uint64))
    ids = w.frame_ids
    index, hashes, parts = {}, [], []
    of_row = np.zeros(w.n, dtype=np.uint64)
    for r, (hi, lo, off, nf) in enumerate(zip(w.hdrs["hash_hi"].tolist(), w.hdrs["hash_lo"].tolist(), w.hdrs["frame_off"].tolist(), w.hdrs["nframes"].tolist())):
        fr = ids[off:off + nf]
        key = (hi, lo, fr.tobytes())
        s = index.get(key)
        if s is None:
            s = index[key] = len(parts)
            hashes.append((hi, lo))
            parts.append(fr)
        of_row[r] = s
    offsets = np.zeros(len(parts) + 1, dtype=np.uint64)
    offsets[1:] = np.cumsum([len(p) for p in parts], dtype=np.uint64)
    frames = np.concatenate(parts).astype(np.uint64) if parts else np.zeros(0, np.uint64)
    return StackForm(np.asarray(hashes, dtype=np.uint64).reshape(-1, 2), frames, offsets, of_row)


def group_stack_form(parts):
    """PA_CFG_GROUP_STACKS: (one StackForm over the union of the parts' stacks, [each part's stack_of_row in it]). Every member
    of a merge group registers that form, so a row names the same stack on every shard; in PA_HASH_PROVIDED mode a stack's id
    comes from whichever part's rows name it. The form's own stack_of_row is that of the concatenated parts (one aggregator fed
    [part 0's rows, part 1's rows, ...])."""
    parts = list(parts)
    t0 = parts[0].stack_table if parts else None
    if parts and all(p._frame_ids is None and (p.stack_table is t0 or np.array_equal(p.stack_table, t0)) for p in parts):
        t = np.ascontiguousarray(t0, dtype=np.uint64)  # one shared stack table: register it once
        hashes = np.zeros((t.shape[0], 2), dtype=np.uint64)
        for p in parts:
            hashes[p.stack_choice, 0] = p.hdrs["hash_hi"]
            hashes[p.stack_choice, 1] = p.hdrs["hash_lo"]
        offsets = np.arange(t.shape[0] + 1, dtype=np.uint64) * np.uint64(t.shape[1])
        rows = [np.asarray(p.stack_choice, dtype=np.uint64) for p in parts]
        return StackForm(hashes, t.reshape(-1), offsets, np.concatenate(rows)), rows
    index, hashes, stacks, rows = {}, [], [], []
    for p in parts:  # each part's own stacks, deduplicated across the parts on (hash_hi, hash_lo, frame ids) as stack_form does
        sf = stack_form(p)
        offs = sf.offsets.astype(np.int64)
        remap = np.zeros(len(offs) - 1, dtype=np.uint64)
        for s, (hi, lo) in enumerate(sf.hashes.tolist()):
            fr = np.asarray(sf.frames[offs[s]:offs[s + 1]], dtype=np.uint64)
            key = (hi, lo, fr.tobytes())
            g = index.get(key)
            if g is None:
                g = index[key] = len(stacks)
                hashes.append((hi, lo))
                stacks.append(fr)
            remap[s] = g
        rows.append(remap[np.asarray(sf.stack_of_row, dtype=np.int64)])
    offsets = np.zeros(len(stacks) + 1, dtype=np.uint64)
    offsets[1:] = np.cumsum([len(f) for f in stacks], dtype=np.uint64)
    frames = np.concatenate(stacks) if stacks else np.zeros(0, np.uint64)
    of_row = np.concatenate(rows) if rows else np.zeros(0, np.uint64)
    return StackForm(np.asarray(hashes, dtype=np.uint64).reshape(-1, 2), frames, offsets, of_row), rows


def expand_stack_form(hdrs, sf):
    """The ring form of rows in registered-stacks form: (headers with hash_hi / hash_lo / nframes / frame_off of their stack,
    concatenated frame ids) — what an aggregator without PA_CFG_REGISTERED_STACKS ingests for the same samples."""
    hd = np.array(hdrs, dtype=abi.HDR_DTYPE, copy=True)
    s = np.asarray(sf.stack_of_row, dtype=np.int64)
    start, end = sf.offsets[:-1].astype(np.int64), sf.offsets[1:].astype(np.int64)
    nf = (end - start)[s]
    hd["hash_hi"], hd["hash_lo"] = sf.hashes[s, 0], sf.hashes[s, 1]
    hd["nframes"] = nf
    off = np.zeros(len(s), dtype=np.int64)
    if len(s):
        off[1:] = np.cumsum(nf)[:-1]
    hd["frame_off"] = off.astype(np.uint64)
    total = int(nf.sum())
    idx = np.repeat(start[s], nf) + (np.arange(total, dtype=np.int64) - np.repeat(off, nf))
    return hd, np.asarray(sf.frames, dtype=np.uint64)[idx]


def from_workload(w, device=0, max_samples=None, max_frames=None, chunk_samples=0, registered_stacks=False, group_form=None, group_retire=False,
                  flags=0, **kw):
    """Aggregator with the workload's dictionaries registered (string id 0 == "" is implicit). registered_stacks: a
    PA_CFG_REGISTERED_STACKS aggregator with the workload's stacks registered too (stack_form); max_frames then defaults to
    the registered frames. group_form: a PA_CFG_REGISTERED_STACKS | PA_CFG_GROUP_STACKS aggregator that registers this
    StackForm (group_stack_form) instead, as every member of its merge group does; with group_retire, PA_CFG_GROUP_RETIRE too
    (a fresh registry hands out handles equal to the form's stack numbers)."""
    sf = group_form if group_form is not None else stack_form(w) if registered_stacks else None
    if group_form is not None:
        flags |= abi.PA_CFG_REGISTERED_STACKS | abi.PA_CFG_GROUP_STACKS | (abi.PA_CFG_GROUP_RETIRE if group_retire else 0)
    n = max(1, w.n if max_samples is None else max_samples)
    nf = max(1, (len(sf.frames) if sf else w.n_frame_ids) if max_frames is None else max_frames)
    a = Aggregator(device=device, hash_mode=w.hash_mode, label_flags=w.label_flags, samples_per_second=w.samples_per_second,
                   external_labels=w.external_labels, max_samples=n, max_frames=nf, chunk_samples=chunk_samples, schema=getattr(w, "schema", 0),
                   flags=flags | (abi.PA_CFG_REGISTERED_STACKS if sf is not None else 0), **kw)
    first = a.register_strings(w.strings[1:])
    assert first == 1, first
    a.register_frames(w.frames)
    a.register_labelsets(w.labelsets)
    if sf is not None:
        a.stack_form = sf
        a.register_stack_handles(sf.frames, sf.offsets, sf.hashes if w.hash_mode == abi.PA_HASH_PROVIDED else None)
    return a


def load(a, w, stack_of_row=None):
    """Write the workload's rows straight into the pinned ring (no intermediate copy of the frame stream). On a registered-stacks
    aggregator the rows name registered stacks (stack_of_row, by default those from_workload(w, registered_stacks=True)
    registered) and the ring gets no frames; a merge group member fed one part of a group_stack_form takes that part's
    stack_of_row."""
    if a.registered:
        hv, _, _ = a.acquire(w.n, 0)
        hv[:] = w.hdrs
        hv["frame_off"] = a.stack_form.stack_of_row if stack_of_row is None else stack_of_row
        a.commit(w.n)
        return
    hv, fv, base = a.acquire(w.n, w.n_frame_ids)
    hv[:] = w.hdrs
    if base:
        hv["frame_off"] += np.uint64(base)
    if w.n_frame_ids:
        w.write_frames(fv)
    a.commit(w.n)


def run(w, device=0, chunk_samples=0, **kw):
    """Whole-batch convenience used by tests: returns (ipc bytes, Result)."""
    a = from_workload(w, device=device, chunk_samples=chunk_samples, **kw)
    load(a, w)
    r = a.flush()
    data = r.ipc_bytes()
    a.close()
    return data, r


def compress_lz4(ipc):
    """LZ4_FRAME body compression of an uncompressed stream (host only; record-identical, not Go-byte-identical)."""
    p, n = C.POINTER(C.c_uint8)(), C.c_uint64()
    rc = lib().pa_ipc_compress_lz4(bytes(ipc), len(ipc), C.byref(p), C.byref(n))
    if rc != 0:
        raise PaError(rc, "pa_ipc_compress_lz4 failed")
    try:
        return C.string_at(p, n.value)
    finally:
        lib().pa_ipc_free(p)


def fix_truncation(s, max_len):
    n = lib().pa_fix_truncation(s, len(s), max_len)
    return (None, False) if n < 0 else (s[:n], True)


def xxh64(data, seed=0):
    buf = (C.c_char * len(data)).from_buffer_copy(data) if data else None
    return int(lib().pa_xxh64(buf, len(data), seed))
