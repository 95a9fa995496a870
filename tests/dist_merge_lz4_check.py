"""Run under torch.distributed.run with the gloo backend: merge groups of PA_IPC_LZ4_FRAME_GPU members, one shard aggregator per
PROCESS, through pa_merge_create_host (collectives on host buffers over gloo) or, with PA_MERGE_TRANSPORT=shm,
pa_merge_create_shm (PA_SHM_MAILBOX bytes per rank; small values make the heads exchange take many rounds). All ranks may share
ONE GPU (PA_ONE_GPU=1). The merged stream goes to POSIX shared memory sized by pa_merge_plan's compressed length; rank 0
checks it, byte for byte, against one PA_IPC_LZ4_FRAME_GPU aggregator on [shard 0 rows, shard 1 rows, ...], and decodes it
against the CPU oracle's plain stream. The last case mixes modes: pa_merge_process must fail with PA_EINVAL on every rank."""
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
from parca_agent_b200 import abi, lib, sharded, synth  # noqa: E402
from parca_agent_b200.host_transport import GlooTransport  # noqa: E402
from test_ipc_lz4_gpu import check_buffers  # noqa: E402

LZ4 = abi.PA_IPC_LZ4_FRAME_GPU


def main():
    local = 0 if os.environ.get("PA_ONE_GPU") == "1" else int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    rank, world = dist.get_rank(), dist.get_world_size()
    kind = os.environ.get("PA_MERGE_TRANSPORT", "gloo")
    transport = GlooTransport()
    seg = ["/pa_merge_lz4_%d" % os.getpid()]
    dist.broadcast_object_list(seg, src=0)

    def group_of(a, ci):
        if kind == "shm":
            return lib.MergeGroup.shm(a, "%s_%d" % (seg[0], ci), rank, world, int(os.environ.get("PA_SHM_MAILBOX", "0")))
        return lib.MergeGroup.host(a, transport, rank, world)

    cases = [synth.edge_workload(seed=43, n=5000, hash_mode=abi.PA_HASH_PROVIDED, external=False),
             synth.edge_workload(seed=44, n=4000, hash_mode=abi.PA_HASH_XXH64X2, external=False),
             synth.config3(n=120_000, u=9_000, p=4_096, npids=96, lsets=6),
             synth.config2(n=300_000, u=20_000, p=32_768)]
    for ci, w in enumerate(cases):
        idx = sharded.shard_rows(w, world)
        if ci == 1:  # an empty shard in the middle of the group
            idx = [idx[0]] + [np.zeros(0, np.int64)] * (world - 2) + [np.concatenate(idx[1:])] if world > 2 else idx
        part = w.rows(idx[rank])
        a = lib.from_workload(part, device=local, frame_id_bytes=4 if ci == 2 else 8, ipc_compression=LZ4)
        group = group_of(a, ci)
        ref = w.rows(np.concatenate(idx))
        want, plain = (lib.run(ref, device=local, frame_id_bytes=4 if ci == 2 else 8, ipc_compression=LZ4)[0], oracle_py.run(ref)[0]) if rank == 0 else (None, None)
        shm = None
        for rep in range(2):
            lib.load(a, part)
            a.stage()
            group.process()
            n = group.plan()
            if shm is None:
                names = [None]
                if rank == 0:
                    shm = shared_memory.SharedMemory(create=True, size=max(n, 1))
                    names[0] = shm.name
                dist.broadcast_object_list(names, src=0)
                if rank != 0:
                    shm = shared_memory.SharedMemory(name=names[0])
                    resource_tracker.unregister(shm._name, "shared_memory")  # attached, not owned: Python < 3.13 would unlink it when this process exits
            view = ctypes.c_char.from_buffer(shm.buf)
            res = group.collect(ctypes.addressof(view), n)
            del view
            dist.barrier()
            if rank == 0:
                got = bytes(shm.buf[:n])
                assert n == len(want) and got == want, "merged GPU-LZ4 stream differs from the single aggregator's (%s, rep %d): %d vs %d bytes" % (w.name, rep, n, len(want))
                check_buffers(got, plain, python_decoder=len(plain) < (4 << 20))
                assert res.n_rows == w.n
                print("case %s rep %d ok: %d rows, %d compressed bytes, %d plain, %d head bytes sent" % (
                    w.name, rep, res.n_rows, n, len(plain), a.kernel_ms("lz4_heads")[1]), flush=True)
            dist.barrier()
        group.close()
        a.close()
        shm.close()
        if rank == 0:
            try:
                shm.unlink()
            except FileNotFoundError:
                pass
    # a group that mixes modes: every rank's pa_merge_process fails before any work
    w = synth.edge_workload(seed=45, n=2000, hash_mode=abi.PA_HASH_XXH64X2, external=False)
    part = w.rows(sharded.shard_rows(w, world)[rank])
    a = lib.from_workload(part, device=local, ipc_compression=LZ4 if rank == world - 1 else abi.PA_IPC_PLAIN)
    group = group_of(a, len(cases))
    lib.load(a, part)
    a.stage()
    try:
        group.process()
        raise AssertionError("a mixed group must be refused")
    except lib.PaError as e:
        assert e.code == -22 and "PA_IPC_LZ4_FRAME_GPU" in str(e), str(e)
    a.discard()
    group.close()
    a.close()
    dist.barrier()
    assert not transport.errors, transport.errors
    if rank == 0:
        print("merge-lz4 ok world=%d transport=%s" % (world, kind))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
