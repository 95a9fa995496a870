"""Run under torch.distributed.run with the gloo backend: a merge group of PA_CFG_GROUP_RETIRE members, one shard aggregator per
PROCESS, through pa_merge_create_host (collectives on host buffers over gloo) or, with PA_MERGE_TRANSPORT=shm,
pa_merge_create_shm. All ranks may share ONE GPU (PA_ONE_GPU=1). Every rank registers the same stacks and gets the same handles;
a churn sequence retires after every interval, and rank 0's stream must equal one PA_CFG_RETIRE_STACKS aggregator's on
[shard 0 rows, shard 1 rows, ...] with the same calls. Then refusals that every rank must see alike: ranks that pass different
idle_batches or different caps, a retired handle on the last rank after its grace batch, and a group that mixes in a plain
group-stacks member. A registration that lands before the retire call on rank 0 and after it elsewhere must not split the group."""
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

REG, GROUP = abi.PA_CFG_REGISTERED_STACKS, abi.PA_CFG_REGISTERED_STACKS | abi.PA_CFG_GROUP_STACKS | abi.PA_CFG_GROUP_RETIRE
EINVAL = -22


def main():
    local = 0 if os.environ.get("PA_ONE_GPU") == "1" else int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    kind = os.environ.get("PA_MERGE_TRANSPORT", "gloo")
    transport = GlooTransport()
    seg = ["/pa_merge_gr_%d" % os.getpid()]
    dist.broadcast_object_list(seg, src=0)

    def group_of(a, ci):
        if kind == "shm":
            return lib.MergeGroup.shm(a, "%s_%d" % (seg[0], ci), rank, world)
        return lib.MergeGroup.host(a, transport, rank, world)

    def same_everywhere(obj, what):
        got = [None] * world
        dist.all_gather_object(got, obj)
        assert all(x == got[0] for x in got), "%s: ranks disagree %s" % (what, got)

    def fails_everywhere(fn, text):
        try:
            fn()
            ok = None
        except lib.PaError as e:
            ok = (e.code, text in str(e))
        same_everywhere(ok, "refusal")
        assert ok == (EINVAL, True), ok

    w = synth.ragged(n=6_000, u=1_200, p=4_096, max_depth=70, hash_mode=abi.PA_HASH_XXH64X2)
    w.schema = abi.PA_SCHEMA_V1
    sf = lib.stack_form(w)
    opts = dict(device=local, max_samples=2_000, max_frames=1_000_000, stack_cache_entries=400)
    a = lib.from_workload(w.head(0), flags=GROUP, **opts)
    single = lib.from_workload(w.head(0), flags=REG | abi.PA_CFG_RETIRE_STACKS, **opts) if rank == 0 else None
    group = group_of(a, 0)
    rng = np.random.Generator(np.random.PCG64(17))  # the same draws on every rank
    lookup, shm, cap_bytes = {}, None, 0

    def register(stacks):
        if not stacks:
            return
        offs = sf.offsets.astype(np.int64)
        parts = [sf.frames[offs[s]:offs[s + 1]] for s in stacks]
        o = np.zeros(len(stacks) + 1, dtype=np.uint64)
        o[1:] = np.cumsum([len(p) for p in parts])
        fr = np.concatenate(parts).astype(np.uint64)
        h = [int(x) for x in a.register_stack_handles(fr, o)]
        same_everywhere(h, "registered handles")
        if single is not None:
            assert [int(x) for x in single.register_stack_handles(fr, o)] == h
        lookup.update(zip(stacks, h))

    def load(agg, hdrs, handles):
        hv, _, _ = agg.acquire(len(hdrs), 0)
        hv[:] = hdrs
        hv["frame_off"] = handles
        agg.commit(len(hdrs))

    def interval(window, n):
        nonlocal shm, cap_bytes
        register([int(s) for s in dict.fromkeys(window.tolist()) if int(s) not in lookup])
        hdrs = np.array(w.hdrs[np.sort(rng.choice(w.n, n, replace=False))], copy=True)
        handles = np.array([lookup[int(s)] for s in rng.choice(window, n)], dtype=np.uint64)
        cuts = np.sort(rng.choice(n + 1, world - 1, replace=True))
        load(a, np.split(hdrs, cuts)[rank], np.split(handles, cuts)[rank])
        a.stage()
        group.process()
        size = group.plan()
        if shm is None or size > cap_bytes:
            cap_bytes = max(size, 1 << 20)
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
        if rank == 0:
            load(single, hdrs, handles)
            r1 = single.flush()
            assert bytes(shm.buf[:size]) == r1.ipc_bytes(), "merged record differs from the single retiring aggregator's"
            assert res.n_unique_stacks == r1.n_unique_stacks
            ids = single.last_stack_ids(r1.n_unique_stacks).tobytes()
        dist.barrier()
        blob = [ids if rank == 0 else None]
        dist.broadcast_object_list(blob, src=0)
        st = group.stacktraces(blob[0] if rank == 0 else None).ipc_bytes()
        same_everywhere(hashlib.sha256(st).hexdigest(), "stacktrace record")
        if rank == 0:
            assert st == single.stacktraces(blob[0]).ipc_bytes()
        return hdrs, handles, cuts

    retired = 0
    for k in range(8):
        window = (np.arange(300) + 90 * k) % len(sf.hashes)
        interval(window, 1_200)
        got = [int(x) for x in group.retire_stacks(1 + k % 2)]
        same_everywhere(got, "retired handles")
        if rank == 0:
            assert got == [int(x) for x in single.retire_stacks(1 + k % 2)]
        gone = set(got)
        lookup = {s: h for s, h in lookup.items() if h not in gone}
        retired += len(got)
        same_everywhere(a.stack_counters(), "registry counters")
        if rank == 0:
            assert a.stack_counters() == single.stack_counters()
            print("interval %d ok: %d retired" % (k, len(got)), flush=True)
    assert retired > 300

    # ranks that disagree on idle_batches: every rank is refused, and nothing is retired
    before = a.stack_counters()["stacks_retired"]
    fails_everywhere(lambda: group.retire_stacks(1 if rank else 2), "the same idle_batches")
    fails_everywhere(lambda: group.retire_stacks(1, cap=10 + rank), "the same idle_batches, cap")
    assert a.stack_counters()["stacks_retired"] == before

    # a registration that lands before the retire call on rank 0 and after it on the other ranks: the next interval still works
    fresh = [int(s) for s in range(len(sf.hashes)) if int(s) not in lookup][:3]
    offs = sf.offsets.astype(np.int64)
    fo = np.zeros(len(fresh) + 1, dtype=np.uint64)
    fo[1:] = np.cumsum([offs[s + 1] - offs[s] for s in fresh])
    ff = np.concatenate([sf.frames[offs[s]:offs[s + 1]] for s in fresh]).astype(np.uint64)
    early = [int(x) for x in a.register_stack_handles(ff, fo)] if rank == 0 else None
    if single is not None:
        assert [int(x) for x in single.register_stack_handles(ff, fo)] == early
    got = [int(x) for x in group.retire_stacks(1)]
    same_everywhere(got, "retired handles")
    if rank == 0:
        assert got == [int(x) for x in single.retire_stacks(1)]
    h = early if rank == 0 else [int(x) for x in a.register_stack_handles(ff, fo)]
    same_everywhere(h, "handles registered around the retire call")
    lookup = {s: x for s, x in lookup.items() if x not in set(got)}
    lookup.update(zip(fresh, h))
    interval(np.array(fresh + list(lookup)[:20]), 200)

    # a retired handle on the last rank, one batch after its grace batch: every rank fails, the next interval works
    window = np.arange(40)
    interval(window, 200)
    got = [int(x) for x in group.retire_stacks(1, 5)]
    assert len(got) == 5
    if rank == 0:
        assert got == [int(x) for x in single.retire_stacks(1, 5)]
    interval(window, 200)  # the grace batch (its rows may still name them)
    hdrs = np.array(w.hdrs[:10], copy=True)
    live = [h for h in lookup.values() if h not in set(got)]
    load(a, hdrs, [got[0] if rank == world - 1 else live[0]] * 10)
    a.stage()
    fails_everywhere(group.process, "unregistered stack id")
    a.discard()
    if rank == 0:  # the single aggregator stays in step: the same failed batch
        load(single, hdrs, [got[0]] * 10)
        try:
            single.flush()
            raise AssertionError("the stale handle must fail")
        except lib.PaError as e:
            assert e.code == EINVAL
    lookup = {s: h for s, h in lookup.items() if h not in set(got)}
    interval(np.arange(40, 80), 200)
    group.close()
    a.close()
    if single is not None:
        single.close()

    # a group that mixes in a plain group-stacks member: pa_merge_process fails on every rank, before any work
    form, _ = lib.group_stack_form([w])
    b = lib.from_workload(w, device=local, group_form=form, group_retire=rank != 1)
    group = group_of(b, 1)
    part = np.arange(rank * 50, rank * 50 + 50)
    lib.load(b, w.rows(part), stack_of_row=form.stack_of_row[part])
    b.stage()
    fails_everywhere(group.process, "PA_CFG_GROUP_RETIRE")
    b.discard()
    group.close()
    b.close()
    shm.close()
    if rank == 0:
        try:
            shm.unlink()
        except FileNotFoundError:
            pass
    dist.barrier()
    assert not transport.errors, transport.errors
    if rank == 0:
        print("merge-group-retire ok world=%d transport=%s" % (world, kind))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
