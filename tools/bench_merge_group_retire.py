"""Merge groups whose members retire registered stacks together (PA_CFG_GROUP_RETIRE), at config-4 shard size on one GPU.
Config-4 shards of --rows rows each (pid-sharded parts of one 8-GPU config-4 interval, 1 M stacks of 64 ids, XXH64 ids):

  (a) --shards members as a plain group-stacks group and as a group-retire group on the same rows (v2): pa_merge_flush median and
      range (stage + process + plan + collect, synchronous; the groups alternate after one warm-up interval each);
  (b) pa_merge_retire_stacks on the group-retire group with every registered slot on the device (the stacks no row named are
      idle), then the flush after the grace batch, whose stage frees them and compacts the arena: its wall time and each member's
      "stack_compact" device time;
  (c) a --churn-interval churn of a fresh group-retire group over a stack window that shifts every interval (stacks entering the
      window are registered into freed slots, retire(2) after each flush): device memory in use and stack_frames_live per
      interval, and the merged sha256 of every interval against one PA_CFG_RETIRE_STACKS aggregator on the concatenated rows.

usage: python tools/bench_merge_group_retire.py [--shards 3] [--rows 12500000] [--runs 3] [--churn 20] [--churn-rows 2000000] [--out FILE]"""
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
    ap.add_argument("--churn", type=int, default=20, help="intervals of the churn run (0: skip)")
    ap.add_argument("--churn-rows", type=int, default=2_000_000, help="rows per shard and interval of the churn run")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "the benchmark needs a CUDA device"
    dev = card()
    S = args.shards
    parts = [synth.config4_part(r, 8, rows_per_gpu=args.rows) for r in range(S)]
    for p in parts[1:]:  # the tables are equal by construction: keep one copy
        p.strings, p.frames, p.labelsets, p.stack_table = parts[0].strings, parts[0].frames, parts[0].labelsets, parts[0].stack_table
    form, sor = lib.group_stack_form(parts)
    lines = []

    def emit(rec):
        rec["card"] = dev
        lines.append(rec)
        print(json.dumps(rec), flush=True)

    def make(k, retire):
        return lib.from_workload(parts[k], device=0, max_samples=parts[k].n, chunk_samples=1 << 20, flags=FLAGS, group_form=form, group_retire=retire)

    # ---- (a) flush time, group-retire members against plain group-stacks members
    groups, digests, t = {}, {}, {"group_stacks": [], "group_retire": []}

    def flush(mode):
        aggs, g = groups[mode]
        for k, a in enumerate(aggs):
            lib.load(a, parts[k], stack_of_row=sor[k])
        t0 = time.perf_counter()
        r = g.flush()
        ms = (time.perf_counter() - t0) * 1e3
        digests[mode] = hashlib.sha256(r.ipc).hexdigest()
        return ms

    for mode in t:
        aggs = [make(k, mode == "group_retire") for k in range(S)]
        groups[mode] = (aggs, lib.MergeGroup.local(aggs))
        flush(mode)
    for k in range(args.runs):
        for mode in (("group_stacks", "group_retire") if k % 2 == 0 else ("group_retire", "group_stacks")):
            t[mode].append(flush(mode))
    for mode in t:
        ms = np.array(t[mode])
        emit({"mode": "merged_v2_" + mode, "shards": S, "rows": S * args.rows, "runs": args.runs, "flush_ms_median": round(float(np.median(ms)), 1),
              "flush_ms_min": round(float(ms.min()), 1), "flush_ms_max": round(float(ms.max()), 1), "sha256": digests[mode]})
    ok = digests["group_stacks"] == digests["group_retire"]
    aggs, g = groups.pop("group_stacks")
    g.close()
    for a in aggs:
        a.close()
    # ---- (b) retirement over every slot, then the stage that frees the retired stacks and compacts the arena
    aggs, g = groups.pop("group_retire")
    slots = aggs[0].stack_counters()["stacks_live"]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    gone = g.retire_stacks(1)
    retire_ms = (time.perf_counter() - t0) * 1e3
    grace_ms = flush("group_retire")
    free_ms = flush("group_retire")  # (this stage frees them; the rows name only live stacks)
    emit({"mode": "group_retire_stacks", "shards": S, "slots": int(slots), "retired": int(len(gone)), "retire_ms": round(retire_ms, 2),
          "grace_flush_ms": round(grace_ms, 1), "freeing_flush_ms": round(free_ms, 1),
          "stack_compact_ms": [round(a.kernel_ms("stack_compact")[0], 3) for a in aggs], "counters": aggs[0].stack_counters()})
    g.close()
    for a in aggs:
        a.close()
    # ---- (c) churn over a shifting window, against one retiring aggregator
    if args.churn:
        n_st, R = len(form.hashes), args.churn_rows
        win, step = n_st // 4, n_st // 16
        offs = form.offsets.astype(np.int64)
        rng = np.random.Generator(np.random.PCG64(3))
        opts = dict(device=0, max_samples=R * S, max_frames=(win + 4 * step) * 64 * 2, chunk_samples=1 << 20, flags=FLAGS)
        members = [lib.from_workload(parts[0].head(0), **dict(opts, max_samples=R, flags=FLAGS | abi.PA_CFG_REGISTERED_STACKS |
                                                             abi.PA_CFG_GROUP_STACKS | abi.PA_CFG_GROUP_RETIRE)) for _ in range(S)]
        single = lib.from_workload(parts[0].head(0), **dict(opts, flags=FLAGS | abi.PA_CFG_REGISTERED_STACKS | abi.PA_CFG_RETIRE_STACKS))
        g = lib.MergeGroup.local(members)
        lookup, same = {}, True
        for k in range(args.churn):
            window = (np.arange(win) + k * step) % n_st
            new = [int(s) for s in window if int(s) not in lookup]
            if new:
                fr = np.concatenate([form.frames[offs[s]:offs[s + 1]] for s in new]).astype(np.uint64)
                o = np.zeros(len(new) + 1, dtype=np.uint64)
                o[1:] = np.cumsum(offs[np.array(new) + 1] - offs[np.array(new)])
                hs = [a.register_stack_handles(fr, o) for a in members + [single]]
                assert all(np.array_equal(h, hs[0]) for h in hs)
                lookup.update(zip(new, (int(x) for x in hs[0])))
            handles = np.array([lookup[int(s)] for s in rng.choice(window, R * S)], dtype=np.uint64)
            for i, a in enumerate(members):
                hv, _, _ = a.acquire(R, 0)
                hv[:] = parts[i].hdrs[:R]
                hv["frame_off"] = handles[i * R:(i + 1) * R]
                a.commit(R)
            hv, _, _ = single.acquire(R * S, 0)
            for i in range(S):
                hv[i * R:(i + 1) * R] = parts[i].hdrs[:R]
            hv["frame_off"] = handles
            single.commit(R * S)
            t0 = time.perf_counter()
            r = g.flush()
            ms = (time.perf_counter() - t0) * 1e3
            got = hashlib.sha256(r.ipc).hexdigest()
            want = hashlib.sha256(single.flush().ipc).hexdigest()
            same = same and got == want
            gone = [int(x) for x in g.retire_stacks(2)]
            assert gone == [int(x) for x in single.retire_stacks(2)]
            gs = set(gone)
            lookup = {s: h for s, h in lookup.items() if h not in gs}
            torch.cuda.synchronize()
            free, total = torch.cuda.mem_get_info()
            c = members[0].stack_counters()
            emit({"mode": "churn", "interval": k, "flush_ms": round(ms, 1), "retired": len(gone), "stacks_live": c["stacks_live"],
                  "stack_frames_live": c["stack_frames_live"], "stack_frames_dead": c["stack_frames_dead"], "stack_compactions": c["stack_compactions"],
                  "device_bytes_in_use": int(total - free), "identical_to_single": got == want})
        ok = ok and same
        g.close()
        for a in members + [single]:
            a.close()
    emit({"mode": "summary", "group_stacks_and_group_retire_identical": digests["group_stacks"] == digests["group_retire"], "ok": ok})
    if args.out:
        with open(args.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")
    if not ok:
        sys.exit(1)


if __name__ == "__main__":
    main()
