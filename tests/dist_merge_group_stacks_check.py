"""Run under torch.distributed.run with the gloo backend: merge groups of PA_CFG_GROUP_STACKS members, one shard aggregator per
PROCESS, through pa_merge_create_host (collectives on host buffers over gloo) or, with PA_MERGE_TRANSPORT=shm,
pa_merge_create_shm (PA_SHM_MAILBOX bytes per rank; small values make every exchange take many rounds). All ranks may share
ONE GPU (PA_ONE_GPU=1). Every rank registers the same group_stack_form. A v2 group, a v1 group over several intervals against a
small store (with stacktrace requests from rank 0) and a PA_IPC_LZ4_FRAME_GPU group: every rank's bytes must equal one
group-stacks aggregator's on [shard 0 rows, shard 1 rows, ...], driven through the same calls. Then a group where the last rank
registered one frame id differently: pa_merge_process must fail with PA_EINVAL on every rank."""
import ctypes
import hashlib
import os
import sys
from multiprocessing import resource_tracker, shared_memory

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from parca_agent_b200 import abi, lib, synth  # noqa: E402
from parca_agent_b200.host_transport import GlooTransport  # noqa: E402

V1 = abi.PA_SCHEMA_V1


def main():
    local = 0 if os.environ.get("PA_ONE_GPU") == "1" else int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    kind = os.environ.get("PA_MERGE_TRANSPORT", "gloo")
    transport = GlooTransport()
    seg = ["/pa_merge_gs_%d" % os.getpid()]
    dist.broadcast_object_list(seg, src=0)

    def group_of(a, ci):
        if kind == "shm":
            return lib.MergeGroup.shm(a, "%s_%d" % (seg[0], ci), rank, world, int(os.environ.get("PA_SHM_MAILBOX", "0")))
        return lib.MergeGroup.host(a, transport, rank, world)

    def same_everywhere(data, what):
        digests = [None] * world
        dist.all_gather_object(digests, (len(data), hashlib.sha256(data).hexdigest()))
        assert all(d == digests[0] for d in digests), "%s: ranks disagree %s" % (what, digests)

    v1 = synth.config2(n=9000, u=2500, p=4096)
    v1.schema = V1
    cases = [("v2", synth.edge_workload(seed=71, n=4000, hash_mode=abi.PA_HASH_PROVIDED, external=False), 0, abi.PA_IPC_PLAIN, 2),
             ("v1", v1, 300, abi.PA_IPC_PLAIN, 5),
             ("lz4", synth.config1().head(30_000), 0, abi.PA_IPC_LZ4_FRAME_GPU, 2)]
    for ci, (name, w, cap, comp, intervals) in enumerate(cases):
        form, _ = lib.group_stack_form([w])  # the same form on every rank
        opts = dict(device=local, max_samples=w.n, stack_cache_entries=cap, ipc_compression=comp, group_form=form)
        a = lib.from_workload(w, **opts)
        single = lib.from_workload(w, **opts) if rank == 0 else None
        group = group_of(a, ci)
        rng = np.random.Generator(np.random.PCG64(7 + ci))  # the same rows on every rank
        probe_rng = np.random.Generator(np.random.PCG64(70 + ci))
        seen, shm, cap_bytes, refs = [], None, 0, 0
        for k in range(intervals):
            rows = np.sort(rng.choice(w.n, min(w.n, 900 if k == 2 else 250), replace=False))
            cuts = np.sort(rng.choice(len(rows) + 1, world - 1, replace=True))
            if k == 1 and world > 2:  # an empty shard in the middle of the group
                cuts[0] = cuts[1] = cuts[0]
            idx = np.split(rows, cuts)
            lib.load(a, w.rows(idx[rank]), stack_of_row=form.stack_of_row[idx[rank]])
            a.stage()
            group.process()
            n = group.plan()
            if shm is None or n > cap_bytes:
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
            res = group.collect(ctypes.addressof(view), cap_bytes)
            del view
            dist.barrier()
            blob = want_st = counters = None
            if rank == 0:
                got = bytes(shm.buf[:n])
                ref = w.rows(np.concatenate(idx))
                lib.load(single, ref, stack_of_row=form.stack_of_row[np.concatenate(idx)])
                r1 = single.flush()
                assert got == r1.ipc_bytes(), "%s interval %d: merged record differs from the single group-stacks aggregator's" % (name, k)
                if w.schema == V1:
                    ids = [bytes(x) for x in single.last_stack_ids(r1.n_unique_stacks)]
                    assert res.n_unique_stacks == len(ids) and a.last_stack_ids(len(ids)).tobytes() == b"".join(ids)
                    seen += [i for i in ids if i not in set(seen)]
                    probe = [seen[int(j)] for j in probe_rng.choice(len(seen), min(len(seen), 100), replace=False)] + [b"\xEE\x01" * 8]
                    blob = b"".join(probe)
                    want_st = single.stacktraces(blob).ipc_bytes()
                    counters = [single.kernel_ms(c)[1] for c in ("store_evictions", "store_compactions")]
            dist.barrier()
            if w.schema == V1:
                same_everywhere(a.last_stack_ids(res.n_unique_stacks).tobytes(), "merged stacktrace_id dictionary")
                st = group.stacktraces(blob).ipc_bytes()
                same_everywhere(st, "stacktrace record")
                if rank == 0:
                    assert st == want_st, "%s interval %d: merged stacktrace record differs" % (name, k)
                objs = [counters]
                dist.broadcast_object_list(objs, src=0)
                assert [a.kernel_ms(c)[1] for c in ("store_evictions", "store_compactions")] == objs[0]
                assert a.kernel_ms("store_frames")[1] == 0
                refs += a.kernel_ms("store_refs")[1]
            if rank == 0:
                print("case %s interval %d ok: %d rows, %d bytes" % (name, k, res.n_rows, n), flush=True)
            dist.barrier()
        if w.schema == V1:
            total = [None] * world
            dist.all_gather_object(total, refs)
            assert sum(total) > 0, "a cold v1 store must have received stack references"
        group.close()
        a.close()
        if single is not None:
            single.close()
        shm.close()
        if rank == 0:
            try:
                shm.unlink()
            except FileNotFoundError:
                pass
        dist.barrier()

    # the last rank registered one frame id differently: every rank fails in the first size exchange, before any work
    w = synth.edge_workload(seed=72, n=2000, hash_mode=abi.PA_HASH_XXH64X2, external=False)
    form, _ = lib.group_stack_form([w])
    if rank == world - 1:
        fr = np.array(form.frames, copy=True)
        fr[len(fr) // 2] = (int(fr[len(fr) // 2]) + 1) % len(w.frames)
        form = lib.StackForm(form.hashes, fr, form.offsets, form.stack_of_row)
    a = lib.from_workload(w, device=local, group_form=form)
    group = group_of(a, len(cases))
    part = np.arange(rank * 100, rank * 100 + 100)
    lib.load(a, w.rows(part), stack_of_row=form.stack_of_row[part])
    a.stage()
    try:
        group.process()
        raise AssertionError("the group must fail on every rank")
    except lib.PaError as e:
        assert e.code == -22 and "identical stacks" in str(e), str(e)
    a.discard()
    group.close()
    lib.load(a, w, stack_of_row=form.stack_of_row)  # the member still flushes alone
    assert a.flush().n_rows == w.n
    a.close()
    dist.barrier()
    assert not transport.errors, transport.errors
    if rank == 0:
        print("merge-group-stacks ok world=%d transport=%s" % (world, kind))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
