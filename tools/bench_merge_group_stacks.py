"""Merge groups of registered stacks with group-wide ids (PA_CFG_GROUP_STACKS) against ring groups, at config-4 shard size on
one GPU. Config-4 shards of --rows rows each (pid-sharded parts of one 8-GPU config-4 interval):

  (a) --shards members as a ring group and as a group-stacks group (v2): pa_merge_flush median and range (stage + process + plan
      + collect, synchronous; the groups alternate after one warm-up interval each), and the device memory each member takes:
      at create, and after the warm-up flush, which adds the device mirrors of the registered tables (the registered stacks'
      records and arena among them), the per-flush scratch and the group's exchange buffers;
  (b) the same shards as v1 groups: the bytes of the store exchange in the cold first interval (4 B per frame id for the ring
      group, one 8-byte handle per stack for the group-stacks group) and in a repeat of it;
  (c) all 8 shards of the interval (8 x --rows rows, which a ring group cannot hold on one 80 GB card) as ONE group-stacks group,
      built member by member until the card is full; then the group is freed and one group-stacks aggregator takes the
      concatenated rows of the shards that fitted: its sha256 must equal the group's.

usage: python tools/bench_merge_group_stacks.py [--shards 3] [--rows 12500000] [--runs 3] [--full 8] [--out FILE]"""
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

FLAGS = abi.PA_CFG_SINGLE_RING


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shards", type=int, default=3)
    ap.add_argument("--rows", type=int, default=12_500_000, help="rows per shard")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--full", type=int, default=8, help="shards of the interval tried as one group-stacks group (0: skip)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    dev = card()
    world = max(args.full, args.shards)
    parts = [synth.config4_part(r, world, rows_per_gpu=args.rows) for r in range(world)]
    for p in parts[1:]:  # the tables are equal by construction: keep one copy
        p.strings, p.frames, p.labelsets, p.stack_table = parts[0].strings, parts[0].frames, parts[0].labelsets, parts[0].stack_table
    form, sor = lib.group_stack_form(parts)
    S = args.shards
    lines = []

    def emit(rec):
        rec["card"] = dev
        lines.append(rec)
        print(json.dumps(rec), flush=True)

    def make(mode, k, schema=abi.PA_SCHEMA_V2):
        p = parts[k]
        p.schema = schema
        if mode == "ring":
            return lib.from_workload(p, device=0, max_samples=p.n, max_frames=p.n_frame_ids, chunk_samples=1 << 20, flags=FLAGS)
        return lib.from_workload(p, device=0, max_samples=p.n, chunk_samples=1 << 20, flags=FLAGS, group_form=form)

    def load(mode, a, k):
        lib.load(a, parts[k]) if mode == "ring" else lib.load(a, parts[k], stack_of_row=sor[k])

    # ---- (a) v2 flush time and device memory per member
    groups, create_bytes, member_bytes, digests = {}, {}, {}, {}

    def flush(mode):
        aggs, g = groups[mode]
        for k, a in enumerate(aggs):
            load(mode, a, k)
        t0 = time.perf_counter()
        r = g.flush()
        ms = (time.perf_counter() - t0) * 1e3
        digests[mode] = hashlib.sha256(r.ipc).hexdigest()
        return ms, r.ipc_len

    t = {"ring": [], "group_stacks": []}
    for mode in t:  # one mode at a time: create, warm-up flush, then what the members hold
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        aggs = [make(mode, k) for k in range(S)]
        torch.cuda.synchronize()
        create_bytes[mode] = (free0 - torch.cuda.mem_get_info()[0]) // S
        groups[mode] = (aggs, lib.MergeGroup.local(aggs))
        flush(mode)
        torch.cuda.synchronize()
        member_bytes[mode] = (free0 - torch.cuda.mem_get_info()[0]) // S
    for k in range(args.runs):
        for mode in (("ring", "group_stacks") if k % 2 == 0 else ("group_stacks", "ring")):
            t[mode].append(flush(mode))
    for mode in t:
        ms = np.array([x[0] for x in t[mode]])
        emit({"mode": "merged_v2_" + mode, "shards": S, "rows": S * args.rows, "runs": args.runs, "flush_ms_median": round(float(np.median(ms)), 1),
              "flush_ms_min": round(float(ms.min()), 1), "flush_ms_max": round(float(ms.max()), 1), "ipc_bytes": t[mode][-1][1],
              "device_bytes_per_member_at_create": int(create_bytes[mode]), "device_bytes_per_member_after_flush": int(member_bytes[mode]),
              "sha256": digests[mode]})
    same = digests["ring"] == digests["group_stacks"]
    for aggs, g in groups.values():
        g.close()
        for a in aggs:
            a.close()
    groups = {}
    # ---- (b) v1 store exchange, cold and repeated interval
    for mode in ("ring", "group_stacks"):
        aggs = [make(mode, k, abi.PA_SCHEMA_V1) for k in range(S)]
        g = lib.MergeGroup.local(aggs)
        sent = []
        for _ in range(2):
            for k, a in enumerate(aggs):
                load(mode, a, k)
            t0 = time.perf_counter()
            r = g.flush()
            ms = (time.perf_counter() - t0) * 1e3
            sent.append((4 * sum(a.kernel_ms("store_frames")[1] for a in aggs) + 8 * sum(a.kernel_ms("store_refs")[1] for a in aggs), round(ms, 1)))
        emit({"mode": "merged_v1_" + mode, "shards": S, "rows": S * args.rows, "n_unique": r.n_unique_stacks,
              "store_exchange_bytes_cold": sent[0][0], "store_exchange_bytes_repeat": sent[1][0], "flush_ms_cold": sent[0][1], "flush_ms_repeat": sent[1][1]})
        g.close()
        for a in aggs:
            a.close()
    for p in parts:
        p.schema = abi.PA_SCHEMA_V2
    # ---- (c) the whole interval as one group-stacks group, then one aggregator on the same rows
    ok = same
    if args.full:
        aggs, err = [], None
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        for k in range(args.full):
            try:
                aggs.append(make("group_stacks", k))
            except lib.PaError as e:
                err = str(e)
                break
        used = free0 - torch.cuda.mem_get_info()[0]
        n = len(aggs)
        rec = {"mode": "full_interval_group_stacks", "shards_tried": args.full, "shards_fitted": n, "rows": n * args.rows,
               "device_bytes_per_member_at_create": int(used // max(n, 1)), "create_error": err}
        digest = None
        try:
            if n:
                g = lib.MergeGroup.local(aggs)
                for k, a in enumerate(aggs):
                    load("group_stacks", a, k)
                t0 = time.perf_counter()
                r = g.flush()
                rec["flush_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
                digest = rec["sha256"] = hashlib.sha256(r.ipc).hexdigest()
                torch.cuda.synchronize()
                rec["device_bytes_per_member_after_flush"] = int((free0 - torch.cuda.mem_get_info()[0]) // n)
                g.close()
        except lib.PaError as e:
            rec["flush_error"] = str(e)
        for a in aggs:
            a.close()
        aggs = None
        torch.cuda.synchronize()
        if digest:  # one group-stacks aggregator on the concatenated rows of the shards that fitted
            w = synth.concat(parts[:n])
            of_row = np.concatenate(sor[:n])
            parts = None
            try:
                a = lib.from_workload(w, device=0, max_samples=w.n, chunk_samples=1 << 20, flags=FLAGS, group_form=form)
                lib.load(a, w, stack_of_row=of_row)
                t0 = time.perf_counter()
                r = a.flush()
                rec["single_flush_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
                rec["single_sha256"] = hashlib.sha256(r.ipc).hexdigest()
                rec["identical_to_single"] = rec["single_sha256"] == digest
                ok = ok and rec["identical_to_single"]
                a.close()
            except lib.PaError as e:
                rec["single_error"] = str(e)
        emit(rec)
    emit({"mode": "summary", "ring_and_group_stacks_identical": same, "ok": ok})
    if args.out:
        with open(args.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
