"""Flush cost of a merged v1 record at config-4 shard size on one GPU: (a) an in-process merge group of PA_SCHEMA_V1 members
(sample record + the replicated known-stacks store), (b) the same shards as a PA_SCHEMA_V2 group, (c) one v1 aggregator on the
concatenated rows. Also: a pa_merge_stacktraces of every id of the interval, and the bytes of the store exchange (frame ids the
members sent) in the first interval and in a repeat of it.

The groups are flushed in rotating order after one warm-up interval each; lines give the median and range of the pa_merge_flush
wall time (stage + process + plan + collect, synchronous). The device memory each v1 member takes (ring, tables and its copy of
the store, with the default stack_cache_entries) is what bounds how many v1 shards fit on one card. Then the groups are freed and
one v1 aggregator takes the concatenated rows: its sha256 must equal the v1 group's.

usage: python tools/bench_merge_v1.py [--shards 3] [--rows 12500000] [--runs 3] [--out FILE]"""
import argparse
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
    lines = []

    def emit(rec):
        rec["card"] = dev
        lines.append(rec)
        print(json.dumps(rec), flush=True)

    groups, member_bytes = {}, {}
    for name, schema in (("v1", abi.PA_SCHEMA_V1), ("v2", abi.PA_SCHEMA_V2)):
        free0 = torch.cuda.mem_get_info()[0]
        aggs = []
        for p in parts:
            p.schema = schema
            aggs.append(lib.from_workload(p, device=0, max_samples=p.n, max_frames=p.n_frame_ids, chunk_samples=1 << 20, flags=abi.PA_CFG_SINGLE_RING))
        member_bytes[name] = (free0 - torch.cuda.mem_get_info()[0]) // S
        groups[name] = (aggs, lib.MergeGroup.local(aggs))
    last = {}

    def flush(name):
        aggs, g = groups[name]
        for a, p in zip(aggs, parts):
            lib.load(a, p)
        t0 = time.perf_counter()
        r = g.flush()
        ms = (time.perf_counter() - t0) * 1e3
        if name == "v1":
            last["digest"] = hashlib.sha256(r.ipc).hexdigest()
            last["n_unique"] = r.n_unique_stacks
            last["frames_sent"] = [a.kernel_ms("store_frames")[1] for a in aggs]
        return {"ms": ms, "bytes": r.ipc_len}

    t = {"v1": [], "v2": []}
    for name in t:  # warm-up = the first interval: every stack is new to the store
        flush(name)
    first = last["frames_sent"]
    for k in range(args.runs):
        for name in (("v1", "v2") if k % 2 == 0 else ("v2", "v1")):
            t[name].append(flush(name))
    for name in t:
        ms = np.array([x["ms"] for x in t[name]])
        rec = {"mode": "merged_" + name, "shards": S, "rows": S * args.rows, "runs": args.runs, "flush_ms_median": round(float(np.median(ms)), 1),
               "flush_ms_min": round(float(ms.min()), 1), "flush_ms_max": round(float(ms.max()), 1), "ipc_bytes": t[name][-1]["bytes"],
               "device_bytes_per_member": int(member_bytes[name])}
        if name == "v1":
            rec.update(sha256=last["digest"], store_exchange_bytes_first_interval=4 * sum(first), store_exchange_bytes_repeat_interval=4 * sum(last["frames_sent"]))
        emit(rec)
    # a request for every id of the interval (offline mode's walk of the merged dictionary)
    aggs, g = groups["v1"]
    blob = aggs[0].last_stack_ids(last["n_unique"]).tobytes()
    st = []
    for _ in range(args.runs):
        t0 = time.perf_counter()
        r = g.stacktraces(blob)
        st.append((time.perf_counter() - t0) * 1e3)
    emit({"mode": "merge_stacktraces_all_ids", "ids": last["n_unique"], "ms_median": round(float(np.median(st)), 1), "ipc_bytes": r.ipc_len,
          "n_locations": r.n_locations})
    free, total = torch.cuda.mem_get_info()
    for aggs, g in groups.values():
        g.close()
        for a in aggs:
            a.close()
    # the same rows through one v1 aggregator
    w = synth.concat(parts)
    parts = None
    w.schema = abi.PA_SCHEMA_V1
    a = lib.from_workload(w, device=0, max_samples=w.n, max_frames=w.n_frame_ids, chunk_samples=1 << 20, flags=abi.PA_CFG_SINGLE_RING)
    single_ms, digest = [], None
    for _ in range(args.runs + 1):
        lib.load(a, w)
        t0 = time.perf_counter()
        r = a.flush()
        single_ms.append((time.perf_counter() - t0) * 1e3)
        digest = hashlib.sha256(r.ipc).hexdigest()
    a.close()
    ms = np.array(single_ms[1:])
    emit({"mode": "single_v1", "rows": w.n, "flush_ms_median": round(float(np.median(ms)), 1), "flush_ms_min": round(float(ms.min()), 1),
          "flush_ms_max": round(float(ms.max()), 1), "sha256": digest, "identical_to_merged_v1": digest == last["digest"],
          "device_free_bytes_with_both_groups": int(free), "device_total_bytes": int(total)})
    if args.out:
        with open(args.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")
    if digest != last["digest"]:
        sys.exit(1)


if __name__ == "__main__":
    main()
