"""Stack retirement (PA_CFG_RETIRE_STACKS) on one GPU. Three parts, one JSON line each; the card's name, power limit and max SM
clock are read in the same run.

  step    configs 2 and 3 at full size: a plain registered aggregator and a retire one (the stack table registered once) take
          the same rows; every timed step ingests, stages, processes and collects them again, so each batch has a new sequence
          number and k_header<true, true> stores it into every named slot's last_use word, as in real use. Median "total" and
          "header" device times of the alternating steps; the difference is the cost of the generation check and the last_use
          store. The two streams' sha256 must be equal.
  retire  1M stacks x 64 ids registered; one batch names about half of them, pa_agg_retire_stacks(1) retires the rest (wall time
          of the call, which ends in a device synchronise), and the stage after the grace batch frees them and compacts the arena
          ("stack_compact" device time; bytes = 2 x the live arena bytes, against the 3.35 TB/s data-sheet HBM3 figure).
  churn   intervals of config-3-shaped rows over a rotating stack population, the lookup cleared every fifth interval as the
          reporter clears its stack cache; retire_stacks(1) after each flush. Per interval: device memory in use, the registry
          counters, and whether the stream's sha256 equals the ring-mode stream of the same rows. A plain registered aggregator
          with the same max_frames is fed the same registrations; the interval at which it fails with PA_ENOSPC is reported.

usage: python tools/bench_stack_retirement.py [--rows 10000000] [--steps 10] [--churn-rows 2000000] [--intervals 20]
                                              [--parts step retire churn] [--out FILE]"""
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

REG, RETIRE = abi.PA_CFG_REGISTERED_STACKS, abi.PA_CFG_RETIRE_STACKS
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def step(cfg, rows, steps):
    w = synth.config2(n=rows) if cfg == 2 else synth.config3(n=rows)
    aggs = {"registered": lib.from_workload(w, chunk_samples=1 << 20, registered_stacks=True),
            "retire": lib.from_workload(w, chunk_samples=1 << 20, registered_stacks=True, flags=RETIRE)}
    digest, t = {}, {k: {"total": [], "header": []} for k in aggs}
    for k, a in aggs.items():  # warm-up
        lib.load(a, w)
        digest[k] = hashlib.sha256(a.flush().ipc_bytes()).hexdigest()
    for i in range(steps):
        for k in (list(aggs) if i % 2 == 0 else list(aggs)[::-1]):
            a = aggs[k]
            lib.load(a, w)
            a.stage()  # a new batch: a new sequence number
            a.process()
            for name in ("total", "header"):
                t[k][name].append(a.kernel_ms(name)[0])
            a.collect()
    out = {"part": "step", "config": cfg, "rows": w.n, "steps": steps, "same_stream": digest["registered"] == digest["retire"]}
    for k, a in aggs.items():
        out[k] = {n: float(np.median(v)) for n, v in t[k].items()}
        a.close()
    out["header_delta_ms"] = out["retire"]["header"] - out["registered"]["header"]
    out["total_delta_ms"] = out["retire"]["total"] - out["registered"]["total"]
    return out


def retire_and_compact(n_stacks=1_000_000, depth=64):
    w = synth.config2(n=1000)
    a = lib.from_workload(w.head(0), max_samples=1 << 20, max_frames=n_stacks * depth, flags=REG | RETIRE)
    rng = np.random.Generator(np.random.PCG64(1))
    frames = rng.integers(0, len(w.frames), n_stacks * depth).astype(np.uint64)
    offsets = np.arange(n_stacks + 1, dtype=np.uint64) * np.uint64(depth)
    t0 = time.perf_counter()
    h = a.register_stack_handles(frames, offsets)
    reg_ms = (time.perf_counter() - t0) * 1e3
    keep = h[(np.arange(n_stacks) % 2 == 0) & (np.arange(n_stacks) < int(n_stacks * 0.98))]  # a little under half stay live
    hdr = np.array(w.hdrs[np.arange(len(keep)) % w.n], copy=True)

    def batch():
        hv, _, _ = a.acquire(len(keep), 0)
        hv[:] = hdr
        hv["frame_off"] = keep
        a.commit(len(keep))

    batch()
    a.flush()
    t0 = time.perf_counter()
    gone = a.retire_stacks(1)
    retire_ms = (time.perf_counter() - t0) * 1e3
    batch()
    a.flush()  # the grace batch
    batch()
    t0 = time.perf_counter()
    a.stage()  # frees the retired stacks; the dead frames now outweigh the live ones: compaction
    stage_ms = (time.perf_counter() - t0) * 1e3
    a.process()
    a.collect()
    c = a.stack_counters()
    ms, launches = a.kernel_ms("stack_compact")
    moved = 2 * c["stack_frames_live"] * 8
    a.close()
    return {"part": "retire", "stacks": n_stacks, "depth": depth, "register_ms": reg_ms, "retired": len(gone), "retire_ms": retire_ms,
            "stage_ms": stage_ms, "compact_ms": ms, "compact_launches": launches, "compactions": c["stack_compactions"],
            "compact_bytes": moved, "compact_bytes_per_s": moved / (ms * 1e-3) if ms else None,
            "compact_share_of_hbm": moved / (ms * 1e-3) / HBM_BYTES_PER_S if ms else None, "counters": c}


def churn(rows, intervals, window=100_000, shift=20_000):
    import torch
    w = synth.config3(n=rows)
    sf = lib.stack_form(w)
    U = len(sf.hashes)
    depth = np.diff(sf.offsets.astype(np.int64))
    max_frames = int(64 * (2 * window + 3 * shift))  # the window, its duplicates after a cleared lookup, stacks in grace
    a = lib.from_workload(w.head(0), max_samples=rows, max_frames=max_frames, flags=REG | RETIRE, chunk_samples=1 << 20)
    plain = lib.from_workload(w.head(0), max_samples=1, max_frames=max_frames, flags=REG)
    ring = lib.from_workload(w.head(0), max_samples=rows, max_frames=rows * 64, chunk_samples=1 << 20)
    lookup = np.full(U, -1, dtype=np.int64)
    plain_enospc, out = None, []
    for k in range(intervals):
        if k % 5 == 4:
            lookup[:] = -1
        win = (k * shift + np.arange(window)) % U
        stacks = (k * shift + np.asarray(w.stack_choice, np.int64) % window) % U
        fresh = win[lookup[win] < 0]
        offs = sf.offsets.astype(np.int64)
        fr = np.concatenate([sf.frames[offs[s]:offs[s + 1]] for s in fresh]) if len(fresh) else np.zeros(0, np.uint64)
        o = np.zeros(len(fresh) + 1, dtype=np.uint64)
        o[1:] = np.cumsum(depth[fresh])
        lookup[fresh] = a.register_stack_handles(fr, o).astype(np.int64)
        if plain_enospc is None:
            try:
                plain.register_stacks(fr, o)
            except lib.PaError as e:
                assert e.code == -28
                plain_enospc = k
        hv, _, _ = a.acquire(w.n, 0)
        hv[:] = w.hdrs
        hv["frame_off"] = lookup[stacks].astype(np.uint64)
        a.commit(w.n)
        got = hashlib.sha256(a.flush().ipc_bytes()).hexdigest()
        hd, ids = lib.expand_stack_form(w.hdrs, lib.StackForm(sf.hashes, sf.frames, sf.offsets, stacks.astype(np.uint64)))
        hv, fv, _ = ring.acquire(w.n, len(ids))
        hv[:] = hd
        fv[:] = ids
        ring.commit(w.n)
        want = hashlib.sha256(ring.flush().ipc_bytes()).hexdigest()
        gone = a.retire_stacks(1)
        lookup[np.isin(lookup, gone.astype(np.int64))] = -1
        free, total = torch.cuda.mem_get_info()
        out.append({"interval": k, "registered": int(len(fresh)), "retired": int(len(gone)), "same_stream": got == want,
                    "device_used_bytes": int(total - free), **a.stack_counters()})
    a.close(); plain.close(); ring.close()
    return {"part": "churn", "rows": rows, "intervals": intervals, "window": window, "shift": shift, "max_frames": max_frames,
            "plain_enospc_interval": plain_enospc, "all_same": all(x["same_stream"] for x in out), "per_interval": out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--churn-rows", type=int, default=2_000_000)
    ap.add_argument("--intervals", type=int, default=20)
    ap.add_argument("--parts", nargs="+", default=["step", "retire", "churn"], choices=["step", "retire", "churn"])
    ap.add_argument("--out")
    args = ap.parse_args()
    lines = [{"card": card()}]
    print(json.dumps(lines[0]), flush=True)
    if "step" in args.parts:
        for cfg in (2, 3):
            lines.append(step(cfg, args.rows, args.steps))
            print(json.dumps(lines[-1]), flush=True)
    if "retire" in args.parts:
        lines.append(retire_and_compact())
        print(json.dumps(lines[-1]), flush=True)
    if "churn" in args.parts:
        lines.append(churn(args.churn_rows, args.intervals))
        print(json.dumps({k: v for k, v in lines[-1].items() if k != "per_interval"}), flush=True)
        for x in lines[-1]["per_interval"]:
            print(json.dumps({k: x[k] for k in ("interval", "same_stream", "device_used_bytes", "stacks_live", "stack_frames_live",
                                                 "stack_frames_dead", "stack_compactions")}), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for x in lines:
                f.write(json.dumps(x) + "\n")


if __name__ == "__main__":
    main()
