"""Run under torch.distributed.run with the gloo backend: merge groups of PA_SCHEMA_V1 members, one shard aggregator per PROCESS,
through pa_merge_create_host (collectives on host buffers over gloo) or, with PA_MERGE_TRANSPORT=shm, pa_merge_create_shm
(PA_SHM_MAILBOX bytes per rank; small values make the store exchange take many rounds). All ranks may share ONE GPU
(PA_ONE_GPU=1). Several intervals against a small store, with stacktrace requests in between (rank 0's ids only): every rank's
sample-record and stacktrace-record bytes must be identical and equal one v1 aggregator's on [shard 0 rows, shard 1 rows, ...]
driven through the same calls, and every rank's member must return the same merged stacktrace_id dictionary. Then three groups
that pa_merge_process must fail with PA_EINVAL on every rank: mixed schemas, v1 members with different store sizes, and a frame
id that is not registered, in stacks whose first occurrence (and so whose frames' trip to the store) is on the last rank only."""
import ctypes
import dataclasses
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
    seg = ["/pa_merge_v1_%d" % os.getpid()]
    dist.broadcast_object_list(seg, src=0)

    def group_of(a, ci):
        if kind == "shm":
            return lib.MergeGroup.shm(a, "%s_%d" % (seg[0], ci), rank, world, int(os.environ.get("PA_SHM_MAILBOX", "0")))
        return lib.MergeGroup.host(a, transport, rank, world)

    def same_everywhere(data, what):
        """every rank's bytes equal rank 0's"""
        digests = [None] * world
        dist.all_gather_object(digests, (len(data), hashlib.sha256(data).hexdigest()))
        assert all(d == digests[0] for d in digests), "%s: ranks disagree %s" % (what, digests)

    cases = [(synth.config2(n=9000, u=2500, p=4096), 300, 6),
             (synth.edge_workload(seed=44, n=4000, hash_mode=abi.PA_HASH_PROVIDED, external=False), 0, 2)]
    for ci, (w, cap, intervals) in enumerate(cases):
        w.schema = V1
        opts = dict(device=local, max_samples=w.n, max_frames=w.n_frame_ids, stack_cache_entries=cap)
        a = lib.from_workload(w, **opts)
        single = lib.from_workload(w, **opts) if rank == 0 else None
        group = group_of(a, ci)
        rng = np.random.Generator(np.random.PCG64(5 + ci))  # the same rows on every rank
        probe_rng = np.random.Generator(np.random.PCG64(50 + ci))  # rank 0's requests
        seen, shm, cap_bytes = [], None, 0
        for k in range(intervals):
            rows = np.sort(rng.choice(w.n, min(w.n, 900 if k == 2 else 250), replace=False))
            cuts = np.sort(rng.choice(len(rows) + 1, world - 1, replace=True))
            if k == 1 and world > 2:  # an empty shard in the middle of the group
                cuts[0] = cuts[1] = cuts[0]
            idx = np.split(rows, cuts)
            part = w.rows(idx[rank])
            part.schema = V1
            lib.load(a, part)
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
            res = group.collect(ctypes.addressof(view), cap_bytes)
            del view
            dist.barrier()
            if rank == 0:
                got = bytes(shm.buf[:n])
                ref = w.rows(np.concatenate(idx))
                ref.schema = V1
                lib.load(single, ref)
                r1 = single.flush()
                assert got == r1.ipc_bytes(), "%s interval %d: merged sample record differs from the single aggregator's" % (w.name, k)
                ids = [bytes(x) for x in single.last_stack_ids(r1.n_unique_stacks)]
                assert res.n_unique_stacks == len(ids) and a.last_stack_ids(len(ids)).tobytes() == b"".join(ids)
                seen += [i for i in ids if i not in set(seen)]
                probe = [seen[int(j)] for j in probe_rng.choice(len(seen), min(len(seen), 100), replace=False)] + [b"\xEE\x01" * 8]
                blob = b"".join(probe)
                want_st = single.stacktraces(blob).ipc_bytes()
                counters = [single.kernel_ms(c)[1] for c in ("store_evictions", "store_compactions")]
            else:
                blob, want_st, counters = None, None, None
            dist.barrier()
            same_everywhere(a.last_stack_ids(res.n_unique_stacks).tobytes(), "merged stacktrace_id dictionary")  # == rank 0's, checked above
            st = group.stacktraces(blob).ipc_bytes()
            same_everywhere(st, "stacktrace record")
            if rank == 0:
                assert st == want_st, "%s interval %d: merged stacktrace record differs from the single aggregator's" % (w.name, k)
            got_counters = [a.kernel_ms(c)[1] for c in ("store_evictions", "store_compactions")]
            objs = [counters]
            dist.broadcast_object_list(objs, src=0)
            assert got_counters == objs[0], (got_counters, objs[0])
            if rank == 0:
                print("case %s interval %d ok: %d rows, %d bytes, %d frame ids sent by rank 0, counters %s" % (
                    w.name, k, res.n_rows, n, a.kernel_ms("store_frames")[1], got_counters), flush=True)
            dist.barrier()
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
    def refused(a, part, ci, text):
        """every rank's pa_merge_process fails with PA_EINVAL and `text`; the members stay usable"""
        group = group_of(a, ci)
        lib.load(a, part)
        a.stage()
        try:
            group.process()
            raise AssertionError("the group must fail on every rank: " + text)
        except lib.PaError as e:
            assert e.code == -22 and text in str(e), str(e)
        a.discard()
        group.close()
        a.close()
        dist.barrier()

    # groups refused in the first size exchange, before any work: mixed schemas; v1 members with different store sizes
    w = synth.edge_workload(seed=45, n=2000, hash_mode=abi.PA_HASH_XXH64X2, external=False)
    if rank == world - 1:
        w.schema = V1
    refused(lib.from_workload(w, device=local), w.head(100), len(cases), "PA_SCHEMA_V1 and PA_SCHEMA_V2")
    w.schema = V1
    refused(lib.from_workload(w, device=local, stack_cache_entries=2000 if rank == world - 1 else 1000), w.head(100), len(cases) + 1,
            "stack_cache_entries")
    # an unregistered frame id that only the last rank sees (it holds the first occurrence of every stack carrying it, so only it
    # packs those frames for the store): like one v1 aggregator, the group fails, and on every rank
    w = synth.edge_workload(seed=46, n=2000, hash_mode=abi.PA_HASH_XXH64X2, external=False)
    w.schema = V1
    fids = np.asarray(w.frame_ids)
    off, nf = w.hdrs["frame_off"].astype(np.int64), w.hdrs["nframes"].astype(np.int64)
    top = int(fids.max())
    first = next(i for i in range(w.n) if nf[i] and int(fids[off[i]:off[i] + nf[i]].max()) == top)
    idx = [np.zeros(0, np.int64)] * world
    idx[:world - 1] = np.array_split(np.arange(first), world - 1) if world > 1 else []
    idx[world - 1] = np.arange(first, w.n)
    registered = dataclasses.replace(w, frames=w.frames[:top])  # frame ids 0 .. top-1
    part = w.rows(idx[rank])
    refused(lib.from_workload(registered, device=local, max_samples=w.n, max_frames=w.n_frame_ids), part, len(cases) + 2, "unregistered frame id")
    assert not transport.errors, transport.errors
    if rank == 0:
        print("merge-v1 ok world=%d transport=%s" % (world, kind))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
