"""Flush cost of a merged config-4 record on one GPU in three ways: (a) a plain merge group, (b) a merge group of
PA_IPC_LZ4_FRAME_GPU members (bodies compressed on the device, on the whole buffers' 64 KiB block grid), (c) the plain merge
followed by pa_ipc_compress_lz4 on the host (liblz4).

S config-4 shards (synth.config4_part) go into two in-process groups, one per member mode, on the same GPU. The modes are
flushed in rotating order, run after run; each line gives the median and range of the pa_merge_flush wall time (stage +
process + plan + collect, synchronous; for (c) plus the host compression), the stream sizes, the members' "lz4" kernel time
and the bytes of block heads the members exchanged. Then both groups are freed and one PA_IPC_LZ4_FRAME_GPU aggregator takes
the concatenated rows of the same shards: its sha256 must equal (b)'s.

usage: python tools/bench_merge_lz4.py [--shards 3] [--rows 12500000] [--runs 3] [--out FILE]"""
import argparse
import ctypes as C
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from parca_agent_b200 import abi, lib, synth  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def host_lz4(res):
    """pa_ipc_compress_lz4 straight from the result's pinned buffer: (ms, compressed bytes)."""
    p, n = C.POINTER(C.c_uint8)(), C.c_uint64()
    t0 = time.perf_counter()
    rc = lib.lib().pa_ipc_compress_lz4(res.ipc.ctypes.data_as(C.c_char_p), res.ipc_len, C.byref(p), C.byref(n))
    ms = (time.perf_counter() - t0) * 1e3
    if rc != 0:
        raise lib.PaError(rc, "pa_ipc_compress_lz4 failed")
    lib.lib().pa_ipc_free(p)
    return ms, int(n.value)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shards", type=int, default=3)
    ap.add_argument("--rows", type=int, default=12_500_000, help="rows per shard")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    dev = card()
    S = args.shards
    parts = [synth.config4_part(r, S, rows_per_gpu=args.rows) for r in range(S)]
    for p in parts[1:]:  # the tables are equal by construction: keep one copy
        p.strings, p.frames, p.labelsets, p.stack_table = parts[0].strings, parts[0].frames, parts[0].labelsets, parts[0].stack_table
    groups = {}
    for name, mode in (("plain", abi.PA_IPC_PLAIN), ("lz4_gpu", abi.PA_IPC_LZ4_FRAME_GPU)):
        aggs = [lib.from_workload(p, device=0, max_samples=p.n, max_frames=p.n_frame_ids, chunk_samples=1 << 20, flags=abi.PA_CFG_SINGLE_RING,
                                  ipc_compression=mode) for p in parts]
        groups[name] = (aggs, lib.MergeGroup.local(aggs))
    t = {"plain": [], "lz4_gpu": [], "plain_then_host_lz4": []}
    last = {}

    def flush(name):
        aggs, g = groups["plain" if name == "plain_then_host_lz4" else name]
        for a, p in zip(aggs, parts):
            lib.load(a, p)
        t0 = time.perf_counter()
        r = g.flush()
        ms = (time.perf_counter() - t0) * 1e3
        rec = {"ms": ms, "bytes": r.ipc_len}
        if name == "plain_then_host_lz4":
            hms, n = host_lz4(r)
            rec.update(ms=ms + hms, host_lz4_ms=hms, bytes=n)
        if name == "lz4_gpu":
            k = [a.kernel_ms("lz4") for a in aggs]
            rec.update(lz4_ms=[round(x[0], 3) for x in k], lz4_launches=[x[1] for x in k], heads_bytes=[a.kernel_ms("lz4_heads")[1] for a in aggs])
            last["digest"] = hashlib.sha256(r.ipc).hexdigest()
        if name == "plain":
            last["plain_bytes"] = r.ipc_len
        return rec

    order = list(t)
    for name in order:  # warm-up: module loads, table growth, pinned output allocation
        flush(name)
    for k in range(args.runs):
        for name in order[k % 3:] + order[:k % 3]:
            t[name].append(flush(name))
    lines = []
    for name in order:
        ms = np.array([x["ms"] for x in t[name]])
        rec = {"mode": name, "shards": S, "rows": S * args.rows, "runs": args.runs, "flush_ms_median": round(float(np.median(ms)), 1),
               "flush_ms_min": round(float(ms.min()), 1), "flush_ms_max": round(float(ms.max()), 1), "ipc_bytes": t[name][-1]["bytes"],
               "ratio_vs_plain": round(t[name][-1]["bytes"] / last["plain_bytes"], 4), "card": dev}
        if name == "plain_then_host_lz4":
            rec["host_lz4_ms_median"] = round(float(np.median([x["host_lz4_ms"] for x in t[name]])), 1)
        if name == "lz4_gpu":
            rec.update({k: t[name][-1][k] for k in ("lz4_ms", "lz4_launches", "heads_bytes")})
            rec["sha256"] = last["digest"]
        lines.append(rec)
        print(json.dumps(rec), flush=True)
    peak = torch.cuda.mem_get_info()
    for aggs, g in groups.values():
        g.close()
        for a in aggs:
            a.close()
    # the same rows through one aggregator
    w = synth.concat(parts)
    parts = None
    a = lib.from_workload(w, device=0, max_samples=w.n, max_frames=w.n_frame_ids, chunk_samples=1 << 20, flags=abi.PA_CFG_SINGLE_RING,
                          ipc_compression=abi.PA_IPC_LZ4_FRAME_GPU)
    lib.load(a, w)
    r = a.flush()
    single = hashlib.sha256(r.ipc).hexdigest()
    a.close()
    rec = {"check": "merged lz4_gpu stream == one PA_IPC_LZ4_FRAME_GPU aggregator on the concatenated rows", "rows": w.n, "sha256": single,
           "identical": single == last["digest"], "device_free_bytes_with_both_groups": peak[0], "device_total_bytes": peak[1], "card": dev}
    lines.append(rec)
    print(json.dumps(rec), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")
    if not rec["identical"]:
        sys.exit(1)


if __name__ == "__main__":
    main()
