"""Run under torch.distributed.run with the gloo backend: the per-batch label column plan in a merge group of one member per
PROCESS, through pa_merge_create_host (collectives on host buffers over gloo) or, with PA_MERGE_TRANSPORT=shm,
pa_merge_create_shm (PA_SHM_MAILBOX bytes per rank). All ranks may share ONE GPU (PA_ONE_GPU=1). Every rank lives through the
same pod-label churn (test_label_plan.churn): each interval registers new labelsets on every member, its small labelset is
named by rank 0's rows only and, every seventh interval, an old labelset (a miss) by the last rank's rows only. After the
fifth interval each member flushes a batch of its own, so the members predict the next merged batch from different names.
Rank 0 compares every merged stream with the oracle fed the same registrations; every rank must report the same
"label_columns" and add the same number to "label_replans" in every merged batch."""
import ctypes
import os
import sys
from multiprocessing import resource_tracker, shared_memory

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import oracle_py  # noqa: E402
from parca_agent_b200 import lib  # noqa: E402
from parca_agent_b200.host_transport import GlooTransport  # noqa: E402
from test_label_plan import churn, oracle_flush, oracle_register_labelsets, spans  # noqa: E402


def main():
    local = 0 if os.environ.get("PA_ONE_GPU") == "1" else int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    kind = os.environ.get("PA_MERGE_TRANSPORT", "gloo")
    transport = GlooTransport()
    seg = ["/pa_label_plan_%d" % os.getpid()]
    dist.broadcast_object_list(seg, src=0)
    w0, ivs = churn(seed=21, n_intervals=12, rows=3000, world=world, empty_at=())
    a = lib.from_workload(w0, device=local, max_samples=3000)
    group = lib.MergeGroup.shm(a, seg[0], rank, world, int(os.environ.get("PA_SHM_MAILBOX", "0"))) if kind == "shm" else \
        lib.MergeGroup.host(a, transport, rank, world)
    o = oracle_py.Oracle(w0) if rank == 0 else None
    shm, cap_bytes = None, 0
    for k, iv in enumerate(ivs):
        a.register_labelsets(iv.new_labelsets)
        if o is not None:
            oracle_register_labelsets(o, iv.new_labelsets)
        replans0 = a.kernel_ms("label_replans")[1]  # (a member's own flushes may replan too: compare what this batch adds)
        lib.load(a, iv.w.rows(spans(iv.w.n, world)[rank]))
        a.stage()
        group.process()
        n = group.plan()
        if shm is None or n > cap_bytes:  # the group's shared output buffer, sized for this interval
            cap_bytes = max(n, 1 << 20)
            names = [None]
            if rank == 0:
                if shm is not None:
                    shm.close(); shm.unlink()
                shm = shared_memory.SharedMemory(create=True, size=cap_bytes)
                names[0] = shm.name
            dist.broadcast_object_list(names, src=0)
            if rank != 0:
                if shm is not None:
                    shm.close()
                shm = shared_memory.SharedMemory(name=names[0])
                resource_tracker.unregister(shm._name, "shared_memory")  # attached, not owned
        view = ctypes.c_char.from_buffer(shm.buf)
        group.collect(ctypes.addressof(view), cap_bytes)
        del view
        dist.barrier()
        if rank == 0:
            assert bytes(shm.buf[:n]) == oracle_flush(o, iv.w), "interval %d: merged stream differs from the oracle" % k
        counters = [None] * world
        dist.all_gather_object(counters, (a.kernel_ms("label_columns")[1], a.kernel_ms("label_replans")[1] - replans0))
        assert all(c == counters[0] for c in counters), "interval %d: members disagree on the plan %s" % (k, counters)
        if rank == 0:
            print("interval %d ok: %d bytes, label_columns %d, replans %d" % (k, n, counters[0][0], counters[0][1]), flush=True)
        if k == 5:  # every member flushes rows of an earlier interval of its own
            mine = ivs[k - 1 - rank]
            lib.load(a, mine.w.rows(spans(mine.w.n, world)[rank]))
            a.flush()
        dist.barrier()
    group.close()
    a.close()
    if o is not None:
        o.close()
    shm.close()
    if rank == 0:
        try:
            shm.unlink()
        except FileNotFoundError:
            pass
    assert not transport.errors, transport.errors
    if rank == 0:
        print("label-plan ok world=%d transport=%s" % (world, kind))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
