"""End-to-end flush cost of the three IPC body modes on one GPU: PA_IPC_PLAIN, PA_IPC_LZ4_FRAME (host liblz4 after the
copy-out) and PA_IPC_LZ4_FRAME_GPU (bodies compressed on the device, only the compressed bytes copied out).

One aggregator per mode holds the same batch; the modes are flushed in rotating order, run after run, so that drift of the
shared host hits them alike. Each result line gives the median and the range over the runs of the pa_agg_flush wall time
(stage + process + collect, synchronous), the device time of the "lz4" kernels, the copy-out and host times the result
reports, and the stream sizes. The GPU-LZ4 stream of the last run is checked buffer by buffer against the plain stream.

usage: python tools/bench_lz4.py [--configs 2 3] [--rows 10000000] [--runs 5] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from parca_agent_b200 import abi, lib, synth  # noqa: E402

MODES = {"plain": abi.PA_IPC_PLAIN, "lz4_host": abi.PA_IPC_LZ4_FRAME, "lz4_gpu": abi.PA_IPC_LZ4_FRAME_GPU}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def bench(cfg, rows, runs):
    from test_ipc_lz4_gpu import check_buffers
    w = synth.config2(n=rows) if cfg == 2 else synth.config3(n=rows)
    aggs = {}
    for name, mode in MODES.items():
        aggs[name] = lib.from_workload(w, ipc_compression=mode, flags=abi.PA_CFG_SINGLE_RING)
    t = {name: [] for name in MODES}
    last = {}

    def flush(name):
        a = aggs[name]
        lib.load(a, w)
        t0 = time.perf_counter()
        r = a.flush()
        ms = (time.perf_counter() - t0) * 1e3
        lz4_ms, lz4_launches = a.kernel_ms("lz4")
        return ms, r, lz4_ms, lz4_launches

    for name in MODES:  # warm-up: module loads, arena growth, pinned output allocation
        flush(name)
    order = list(MODES)
    for k in range(runs):
        for name in order[k % 3:] + order[:k % 3]:
            ms, r, lz4_ms, lz4_launches = flush(name)
            t[name].append((ms, r.d2h_ms, r.host_ms, lz4_ms, lz4_launches, r.ipc_len, r.gpu_ms))
            if k == runs - 1 and name in ("plain", "lz4_gpu"):
                last[name] = r.ipc_bytes()
    host_len = t["lz4_host"][-1][5]
    plain_len = t["plain"][-1][5]
    out = []
    for name in MODES:
        a = np.array(t[name], dtype=np.float64)
        med = np.median(a, axis=0)
        rec = {"config": cfg, "rows": rows, "mode": name, "runs": runs, "flush_ms_median": round(med[0], 2),
               "flush_ms_min": round(a[:, 0].min(), 2), "flush_ms_max": round(a[:, 0].max(), 2),
               "samples_per_s": round(rows / (med[0] / 1e3)), "gpu_ms": round(med[6], 3), "d2h_ms": round(med[1], 2), "host_ms": round(med[2], 2),
               "ipc_bytes": int(a[-1, 5]), "ratio_vs_plain": round(a[-1, 5] / plain_len, 4), "ratio_vs_host_lz4": round(a[-1, 5] / host_len, 4)}
        if name == "lz4_gpu":
            rec.update({"lz4_kernel_ms": round(med[3], 3), "lz4_launches": int(a[-1, 4]), "lz4_uncompressed_GBps": round(plain_len / (med[3] / 1e3) / 1e9, 1)})
        out.append(rec)
    stats = check_buffers(last["lz4_gpu"], last["plain"], python_decoder=False)
    out[-1]["checked_buffers"] = stats
    for a in aggs.values():
        a.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", type=int, nargs="+", default=[2, 3], choices=[2, 3])
    ap.add_argument("--rows", type=int, default=10_000_000)
    ap.add_argument("--runs", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    dev = card()
    lines = []
    for cfg in args.configs:
        for rec in bench(cfg, args.rows, args.runs):
            rec["card"] = dev
            lines.append(rec)
            print(json.dumps(rec), flush=True)
    if args.out:
        with open(args.out, "w") as f:
            for rec in lines:
                f.write(json.dumps(rec) + "\n")


if __name__ == "__main__":
    main()
