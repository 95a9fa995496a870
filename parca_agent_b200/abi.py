"""ctypes/numpy mirror of include/parcaagg.h (struct layouts and constants only).

Shared by the product binding (parca_agent_b200.lib), the synthetic workload generator and the
test-side oracle wrapper. No compute lives here.
"""
import ctypes as C

import numpy as np

PA_ABI_VERSION = 3
PA_CFG_SINGLE_RING = 1
PA_CFG_REGISTERED_STACKS = 2
PA_CFG_GROUP_STACKS = 4
PA_CFG_RETIRE_STACKS = 8
PA_CFG_GROUP_RETIRE = 16

PA_KIND_CPU, PA_KIND_OFFCPU, PA_KIND_CUDA = 0, 1, 2
PA_KIND_MEM_INUSE_OBJECTS, PA_KIND_MEM_INUSE_SPACE, PA_KIND_MEM_ALLOC_OBJECTS, PA_KIND_MEM_ALLOC_SPACE = 3, 4, 5, 6

PA_FRAME_NATIVE, PA_FRAME_KERNEL, PA_FRAME_ABORT, PA_FRAME_OOMPROF, PA_FRAME_INTERP = 0, 1, 2, 3, 4
PA_FRAME_F_MAPPING_FILE, PA_FRAME_F_EXEC_KNOWN = 1, 2

PA_HASH_PROVIDED, PA_HASH_XXH64X2 = 0, 1
PA_XXH_SEED_LO = 0x9E3779B97F4A7C15

PA_LABEL_DISABLE_CPU, PA_LABEL_DISABLE_THREAD_ID, PA_LABEL_DISABLE_THREAD_COMM = 1, 2, 4
PA_SCHEMA_V2, PA_SCHEMA_V1 = 0, 1
PA_IPC_PLAIN, PA_IPC_LZ4_FRAME, PA_IPC_LZ4_FRAME_GPU = 0, 1, 2
PA_NO_STRING = 0xFFFFFFFF

# struct pa_sample_hdr (64 B)
HDR_DTYPE = np.dtype([
    ("hash_hi", "<u8"), ("hash_lo", "<u8"), ("timestamp_ns", "<i8"), ("value", "<i8"),
    ("pid", "<u4"), ("tid", "<u4"), ("comm_sid", "<u4"), ("labelset_id", "<u4"),
    ("frame_off", "<u8"), ("cpu", "<u4"), ("nframes", "<u2"), ("kind", "u1"), ("flags", "u1"),
])
assert HDR_DTYPE.itemsize == 64

# struct pa_frame_desc (64 B)
FRAME_DTYPE = np.dtype([
    ("kind", "u1"), ("flags", "u1"), ("reserved0", "<u2"), ("type_name_sid", "<u4"),
    ("address_or_lineno", "<u8"), ("function_name_sid", "<u4"), ("source_file_sid", "<u4"),
    ("source_line", "<u4"), ("exec_file_name_sid", "<u4"), ("exec_build_id_sid", "<u4"), ("source_column", "<u4"),
    ("file_id_hi", "<u8"), ("file_id_lo", "<u8"), ("mapping_file_name_sid", "<u4"), ("gnu_build_id_sid", "<u4"),
])
assert FRAME_DTYPE.itemsize == 64

PAIR_DTYPE = np.dtype([("name_sid", "<u4"), ("value_sid", "<u4")])


class PaLabelPair(C.Structure):
    _fields_ = [("name_sid", C.c_uint32), ("value_sid", C.c_uint32)]


class PaAggConfig(C.Structure):
    _fields_ = [
        ("abi_version", C.c_uint32), ("device", C.c_int32), ("hash_mode", C.c_uint32), ("label_flags", C.c_uint32),
        ("samples_per_second", C.c_uint32), ("n_external_labels", C.c_uint32),
        ("external_labels", C.POINTER(PaLabelPair)),
        ("max_samples", C.c_uint64), ("max_frames", C.c_uint64), ("chunk_samples", C.c_uint32), ("schema", C.c_uint32),
        ("stack_cache_entries", C.c_uint64), ("stack_cache_frames", C.c_uint64), ("unknown_frame_type_sid", C.c_uint32), ("flags", C.c_uint32),
        ("frame_id_bytes", C.c_uint32), ("ipc_compression", C.c_uint32),
    ]


class PaAggResult(C.Structure):
    _fields_ = [
        ("ipc", C.POINTER(C.c_uint8)), ("ipc_len", C.c_uint64), ("n_rows", C.c_uint64),
        ("n_unique_stacks", C.c_uint64), ("n_locations", C.c_uint64), ("n_functions", C.c_uint64),
        ("n_location_indices", C.c_uint64), ("gpu_launches", C.c_uint32), ("reserved", C.c_uint32),
        ("h2d_ms", C.c_double), ("gpu_ms", C.c_double), ("d2h_ms", C.c_double), ("host_ms", C.c_double),
    ]


class PaDevicePart(C.Structure):
    _fields_ = [("hdr", C.c_void_p), ("global_row", C.c_void_p), ("n_rows", C.c_uint64), ("frames", C.c_void_p), ("n_frames", C.c_uint64)]


def pack_strings(strs):
    """list[bytes] → (bytes blob, uint32 offsets[n+1])."""
    offs = np.zeros(len(strs) + 1, dtype=np.uint32)
    if strs:
        offs[1:] = np.cumsum([len(s) for s in strs], dtype=np.uint64).astype(np.uint32)
    return b"".join(strs), offs


def pack_labelsets(labelsets):
    """list[list[(name_sid, value_sid)]] → (pairs array, uint32 offsets[n+1])."""
    offs = np.zeros(len(labelsets) + 1, dtype=np.uint32)
    flat = []
    for i, ls in enumerate(labelsets):
        flat.extend(ls)
        offs[i + 1] = len(flat)
    pairs = np.zeros(len(flat), dtype=PAIR_DTYPE)
    if flat:
        arr = np.asarray(flat, dtype=np.uint32).reshape(-1, 2)
        pairs["name_sid"] = arr[:, 0]
        pairs["value_sid"] = arr[:, 1]
    return pairs, offs
