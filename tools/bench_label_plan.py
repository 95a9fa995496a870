"""The per-batch label column plan on one GPU, against the parent build's lifetime plan. Every part prints one JSON line; the
card's name, power limit and max SM clock are read in the same run.

  span     config-2 rows whose registered labelsets span 10, 100 and 240 lifetime label names, 10 of them named by the rows
           (64 labelsets over the same 10 names, the rest registered and never named). This build and the parent build
           (--parent-lib, compiled from the parent commit) run in alternating worker processes on the same seeded rows: median
           "labels" and "total" device times of the timed flushes, the process's device memory after the first flush
           (nvidia-smi), and the sha256 of each stream, which must be equal between the builds.
  wide     the same with 5000 lifetime names (this build only: the parent fails every flush past 246).
  replan   one aggregator, 240 lifetime names: wall time of flushes whose prediction holds and of flushes that miss (the rows
           name an old labelset each other flush), and the replans counted.
  churn    50 intervals of config-2-shaped rows with pod-label churn (each interval registers six labelsets over 34 new names
           and its rows name them): per interval the planned label columns, the replans so far, "labels" / "total" device times
           and device memory.

usage: python tools/bench_label_plan.py [--rows 10000000] [--steps 10] [--warmup 3] [--rounds 2] [--parent-lib PATH]
                                        [--parts span wide replan churn] [--out FILE]"""
import argparse
import dataclasses
import hashlib
import json
import os
import pickle
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from parca_agent_b200 import abi, lib, synth  # noqa: E402

USED = 10


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def device_mib():
    """This process's device memory (MiB) as nvidia-smi reports it; None when it cannot tell."""
    q = subprocess.run(["nvidia-smi", "--query-compute-apps=pid,used_memory", "--format=csv,noheader,nounits"], capture_output=True, text=True)
    for line in q.stdout.splitlines():
        f = [x.strip() for x in line.split(",")]
        if len(f) == 2 and f[0] == str(os.getpid()):
            return int(f[1])
    return None


def spanned(w, n_names, seed=1):
    """w's rows on 64 labelsets over the same USED names; more labelsets register the other n_names - USED names."""
    st = synth.StringTable()
    st.strings, st.index = list(w.strings), {s: i for i, s in enumerate(w.strings)}
    names = [st.sid("pod_label_%05d" % k) for k in range(n_names)]
    vals = [st.sid("v%d" % k) for k in range(64)]
    rng = np.random.Generator(np.random.PCG64(seed))
    named = [[(names[k], vals[int(rng.integers(0, 64))]) for k in range(USED)] for _ in range(64)]
    rest = [[(names[k], vals[0]) for k in range(j, min(j + 20, n_names))] for j in range(USED, n_names, 20)]
    hd = w.hdrs.copy()
    hd["labelset_id"] = hd["labelset_id"] % 64
    return dataclasses.replace(w, strings=st.strings, labelsets=named + rest, hdrs=hd)


def _replace(w, **kw):
    return dataclasses.replace(w, **kw)


def timed_flushes(a, w, warmup, steps):
    labels, total, digest, mib = [], [], None, None
    for i in range(warmup + steps):
        lib.load(a, w)
        r = a.flush()
        d = hashlib.sha256(r.ipc_bytes()).hexdigest()
        if digest is None:
            digest, mib = d, device_mib()
        assert d == digest, "the stream changed between flushes of the same rows"
        if i >= warmup:
            labels.append(a.kernel_ms("labels")[0])
            total.append(a.kernel_ms("total")[0])
    return {"labels_ms": float(np.median(labels)), "total_ms": float(np.median(total)), "device_mib_after_first_flush": mib, "sha256": digest}


def worker(args):
    """One arm of one part, in its own process (the parent build is loaded instead of this one with --lib)."""
    out = {"lib": "this" if os.path.abspath(args.lib) == os.path.abspath(lib.LIB_PATH) else "parent"}
    lib.LIB_PATH = args.lib
    with open(args.cache, "rb") as f:
        w = pickle.load(f)
    try:
        a = lib.from_workload(w)
        out.update(timed_flushes(a, w, args.warmup, args.steps))
        try:
            out["label_columns"] = a.kernel_ms("label_columns")[1]
        except lib.PaError:
            pass
        a.close()
    except lib.PaError as e:
        out["error"] = str(e)
    print(json.dumps(out))


def run_worker(cache, libpath, args):
    cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--cache", cache, "--lib", libpath, "--steps", str(args.steps), "--warmup", str(args.warmup)]
    p = subprocess.run(cmd, capture_output=True, text=True)
    if p.returncode:
        return {"error": p.stderr.strip().splitlines()[-1] if p.stderr.strip() else "exit %d" % p.returncode}
    return json.loads(p.stdout.strip().splitlines()[-1])


def part_span(args, base, tmp, spans, arms):
    out = []
    for n_names in spans:
        cache = os.path.join(tmp, "span_%d.pkl" % n_names)
        with open(cache, "wb") as f:
            pickle.dump(spanned(base, n_names), f)
        res = {arm: [] for arm in arms}
        for _ in range(args.rounds):  # alternate the builds
            for arm, path in arms.items():
                res[arm].append(run_worker(cache, path, args))
        line = {"part": "span" if len(arms) > 1 else "wide", "lifetime_names": n_names, "used_names": USED, "rows": base.n}
        for arm, rs in res.items():
            ok = [r for r in rs if "error" not in r]
            line[arm] = {"labels_ms": [r["labels_ms"] for r in ok], "total_ms": [r["total_ms"] for r in ok],
                         "device_mib_after_first_flush": [r["device_mib_after_first_flush"] for r in ok],
                         "sha256": sorted({r["sha256"] for r in ok}), "label_columns": sorted({r.get("label_columns") for r in ok} - {None}),
                         "errors": [r["error"] for r in rs if "error" in r]}
        if len(arms) > 1:
            line["same_stream"] = line["this"]["sha256"] == line["parent"]["sha256"] and len(line["this"]["sha256"]) == 1
        out.append(line)
        print(json.dumps(line), flush=True)
    return out


def part_replan(args, base):
    w = spanned(base, 240)
    old = _replace(w, hdrs=w.hdrs.copy())
    old.hdrs["labelset_id"][::997] = len(w.labelsets) - 1  # an old labelset over names no recent batch named
    a = lib.from_workload(w)
    hit, miss = [], []
    for i in range(args.warmup + 2 * args.steps):
        x = old if i % 2 else w
        lib.load(a, x)
        t0 = time.perf_counter()
        a.flush()
        dt = (time.perf_counter() - t0) * 1e3
        if i >= args.warmup:
            (miss if i % 2 else hit).append(dt)
    line = {"part": "replan", "rows": w.n, "flush_wall_ms_hit": float(np.median(hit)), "flush_wall_ms_miss": float(np.median(miss)),
            "label_replans": a.kernel_ms("label_replans")[1]}
    a.close()
    print(json.dumps(line), flush=True)
    return line


def part_churn(args, base, n_intervals=50, window=34):
    st = synth.StringTable()
    st.strings, st.index = list(base.strings), {s: i for i, s in enumerate(base.strings)}
    names = [st.sid("pod_label_%05d" % k) for k in range(window * n_intervals)]
    vals = [st.sid("v%d" % k) for k in range(16)]
    w0 = _replace(base, strings=st.strings, labelsets=[])
    rng = np.random.Generator(np.random.PCG64(7))
    a = lib.from_workload(w0)
    n_ls, lines = 0, []
    for i in range(n_intervals):
        win = names[window * i:window * (i + 1)]
        new = [[(win[c], vals[int(rng.integers(0, 16))]) for c in part] for part in np.array_split(np.arange(window), 6)]
        a.register_labelsets(new)
        hd = base.hdrs.copy()
        hd["labelset_id"] = n_ls + hd["labelset_id"] % len(new)
        n_ls += len(new)
        lib.load(a, _replace(w0, hdrs=hd))
        a.flush()
        lines.append({"interval": i, "label_columns": a.kernel_ms("label_columns")[1], "label_replans": a.kernel_ms("label_replans")[1],
                      "labels_ms": a.kernel_ms("labels")[0], "total_ms": a.kernel_ms("total")[0], "device_mib": device_mib()})
    a.close()
    line = {"part": "churn", "rows": base.n, "intervals": lines, "lifetime_names": window * n_intervals}
    print(json.dumps(line), flush=True)
    return line


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--churn-rows", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--parent-lib", help="libparcaagg.so built from the parent commit (the span part needs it)")
    ap.add_argument("--parts", nargs="+", default=["span", "wide", "replan", "churn"])
    ap.add_argument("--out")
    ap.add_argument("--worker", action="store_true")
    ap.add_argument("--cache")
    ap.add_argument("--lib")
    args = ap.parse_args()
    if args.worker:
        return worker(args)
    head = {"card": card(), "rows": args.rows, "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds}
    print(json.dumps(head), flush=True)
    results = [head]
    base = synth.config2(n=args.rows)
    with tempfile.TemporaryDirectory() as tmp:
        if "span" in args.parts:
            if not args.parent_lib or not os.path.exists(args.parent_lib):
                raise SystemExit("--parent-lib %s: build the parent commit's libparcaagg.so first" % args.parent_lib)
            results += part_span(args, base, tmp, (10, 100, 240), {"this": lib.LIB_PATH, "parent": args.parent_lib})
        if "wide" in args.parts:
            results += part_span(args, base, tmp, (5000,), {"this": lib.LIB_PATH})
    if "replan" in args.parts:
        results.append(part_replan(args, base))
    if "churn" in args.parts:
        results.append(part_churn(args, synth.config2(n=args.churn_rows)))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
