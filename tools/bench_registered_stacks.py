"""Ring rows vs registered stacks (PA_CFG_REGISTERED_STACKS) on one GPU, at full size: configs 2 and 3, uint64 and uint32 frame
ids, both hash modes. The ring aggregator ingests headers + frame ids; the registered one has the workload's stack table
registered once and ingests 64-byte headers that name their stack.

For every (config, id width, hash mode) both aggregators hold the same batch and run alternately, run after run, so that drift
of the shared host hits them alike. Each result line gives, per mode: the median and range of the pa_agg_flush wall time and its
h2d / gpu / d2h / host split (as the result reports it), the resident step (pa_agg_stage once, then pa_agg_process repeated:
"total", "header" and "hash" device times), the pinned ring bytes the aggregator holds, and the sha256 of the stream (the two
must be equal). The card's name, power limit and max SM clock are read in the same run.

Producer side: tests/cpp/bench_reporter_stacks.cpp (compiled into a temporary directory) feeds the C++ reporter mirror into a
config-2-shaped aggregator (2M samples, 64 frames, 100k stacks, 262,144 frames), ring rows and registered stacks alternately.

usage: python tools/bench_registered_stacks.py [--configs 2 3] [--rows 10000000] [--runs 5] [--steps 10] [--reporter-runs 2]
                                               [--reporter-only] [--out FILE]"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from parca_agent_b200 import abi, lib, synth  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def pinned_ring_bytes(w, registered, idb):
    """What pa_agg_create pins for the ring (two buffers): headers, plus the frame-id ring unless stacks are registered."""
    per = w.n * 64 + (0 if registered else w.n_frame_ids * idb + 64)
    return 2 * per


def med(xs):
    return {"median": float(np.median(xs)), "min": float(np.min(xs)), "max": float(np.max(xs))}


def bench(cfg, rows, idb, mode, runs, steps):
    w = synth.config2(n=rows, hash_mode=mode) if cfg == 2 else synth.config3(n=rows, hash_mode=mode)
    aggs = {"ring": lib.from_workload(w, frame_id_bytes=idb, chunk_samples=1 << 20),
            "registered": lib.from_workload(w, frame_id_bytes=idb, chunk_samples=1 << 20, registered_stacks=True)}
    t = {k: [] for k in aggs}
    digest = {}

    def flush(k):
        a = aggs[k]
        lib.load(a, w)
        t0 = time.perf_counter()
        r = a.flush()
        ms = (time.perf_counter() - t0) * 1e3
        return ms, r

    for k in aggs:  # warm-up: module loads, arena growth, pinned output allocation
        flush(k)
    order = list(aggs)
    for i in range(runs):
        for k in (order if i % 2 == 0 else order[::-1]):
            ms, r = flush(k)
            t[k].append((ms, r.h2d_ms, r.gpu_ms, r.d2h_ms, r.host_ms))
            if i == runs - 1:
                digest[k] = hashlib.sha256(r.ipc_bytes()).hexdigest()
    out = {"config": cfg, "rows": w.n, "frame_id_bytes": idb, "hash_mode": "provided" if mode == abi.PA_HASH_PROVIDED else "xxh64x2",
           "runs": runs, "same_stream": digest["ring"] == digest["registered"]}
    for k, a in aggs.items():
        x = np.asarray(t[k])
        res = {"flush_ms": med(x[:, 0]), "h2d_ms": float(np.median(x[:, 1])), "gpu_ms": float(np.median(x[:, 2])),
               "d2h_ms": float(np.median(x[:, 3])), "host_ms": float(np.median(x[:, 4])),
               "e2e_samples_per_s": w.n / (float(np.median(x[:, 0])) * 1e-3),
               "pinned_ring_bytes": pinned_ring_bytes(w, k == "registered", idb), "sha256": digest[k]}
        lib.load(a, w)
        a.stage()
        tot, hdr, hsh = [], [], []
        for _ in range(steps + 2):
            a.process()
            tot.append(a.kernel_ms("total")[0]); hdr.append(a.kernel_ms("header")[0]); hsh.append(a.kernel_ms("hash")[0])
        a.collect()
        res["resident_step_ms"] = {"total": med(tot[2:]), "header": med(hdr[2:]), "hash": med(hsh[2:])}
        out[k] = res
        a.close()
    return out


def reporter(runs):
    """ReportTraceEvent rates with ring rows and with registered stacks, alternating (one JSON line each)"""
    out = []
    with tempfile.TemporaryDirectory() as d:
        exe = os.path.join(d, "bench_reporter_stacks")
        libdir = os.path.join(ROOT, "parca_agent_b200")
        subprocess.run(["g++", "-O2", "-std=c++17", "-o", exe, os.path.join(ROOT, "tests", "cpp", "bench_reporter_stacks.cpp"), "-L" + libdir,
                        "-lparcaagg", "-Wl,-rpath," + libdir, "-lpthread"], check=True)
        for _ in range(runs):
            for rows in ("ring", "stacks"):
                p = subprocess.run([exe, "2000000", "64", "100000", "262144", "gpu", "handle", rows], capture_output=True, text=True, timeout=600)
                out.append(json.loads(p.stdout.strip().splitlines()[-1]) if p.returncode == 0 else {"rows": rows, "error": p.stderr[-300:]})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", type=int, nargs="+", default=[2, 3])
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--reporter-runs", type=int, default=2)
    ap.add_argument("--reporter-only", action="store_true", help="only the producer-side comparison")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs a CUDA device"
    lines = []
    for cfg in ([] if args.reporter_only else args.configs):
        for idb in (8, 4):
            for mode in (abi.PA_HASH_XXH64X2, abi.PA_HASH_PROVIDED):
                r = bench(cfg, args.rows, idb, mode, args.runs, args.steps)
                r["card"] = card()
                print(json.dumps(r), flush=True)
                lines.append(r)
    for r in reporter(args.reporter_runs):
        r["card"] = card()
        print(json.dumps(r), flush=True)
        lines.append(r)
    if args.out:
        with open(args.out, "w") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
