"""Small end-to-end cases for compute-sanitizer (memcheck / racecheck are 10-100x slower than a normal run): the kernels and host paths
added in round 2 — early copy-out during a multi-chunk flush, the v1 LRU store (evictions, revivals, compaction, over-full batch),
the pipelined / bulk-copy-staged hash variants, the narrow ring, a 3-shard merged record.

usage: PA_EARLY_D2H_ALWAYS=1 compute-sanitizer --tool memcheck python tools/sanitize_small.py [plain|lz4_gpu|merge_lz4_gpu|merge_v1|registered|merge_group_stacks|merge_group_retire]
lz4_gpu: small flushes with the bodies compressed on the device (PA_IPC_LZ4_FRAME_GPU) instead: a multi-chunk v2 batch, the
narrow ring, and a v1 batch with its stacktrace record, each checked against the oracle's plain stream.
merge_lz4_gpu: a small in-process merge group of PA_IPC_LZ4_FRAME_GPU members whose shard cuts put blocks across part borders
(heads exchange, crossing blocks, an empty shard), checked against one such aggregator on the concatenated rows.
merge_v1: in-process groups of PA_SCHEMA_V1 members over several intervals against a small store (evictions, compaction, an
over-full batch, stacktrace requests), plain and PA_IPC_LZ4_FRAME_GPU, checked against one v1 aggregator and the oracle.
registered: PA_CFG_REGISTERED_STACKS aggregators (both hash modes, the narrow ring, small chunks, v1) against the oracle, and a
row naming an unregistered stack id followed by a clean flush.
merge_group_stacks: in-process groups of PA_CFG_GROUP_STACKS members — a v2 interval over three shards with an empty one, and
v1 intervals against a small store (stack references instead of frames), checked against one group-stacks aggregator, a ring
group and the oracle.
merge_group_retire: in-process groups of PA_CFG_GROUP_RETIRE members through a small churn (v2 over three shards, v1 over two):
retirement with the group-wide last_use, re-registration into freed slots, compaction, and v1 store references as handles,
checked against one PA_CFG_RETIRE_STACKS aggregator."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import oracle_py  # noqa: E402
from parca_agent_b200 import abi, lib, sharded, synth  # noqa: E402


def lz4_gpu():
    from test_ipc_lz4_gpu import check_stream
    base = synth.edge_workload(seed=3, n=3000, hash_mode=abi.PA_HASH_XXH64X2)
    for kw in ({}, {"frame_id_bytes": 4}):
        a = lib.from_workload(base, chunk_samples=450, ipc_compression=abi.PA_IPC_LZ4_FRAME_GPU, **kw)
        for n in (3000, 1200):
            w = base.head(n)
            lib.load(a, w)
            check_stream(a.flush().ipc_bytes(), oracle_py.run(w)[0])
        a.close()
    w = synth.config2(n=3000, u=800, p=1024)
    w.schema = abi.PA_SCHEMA_V1
    o = oracle_py.Oracle(w)
    o.ingest(w.hdrs, w.frame_ids)
    want, _ = o.flush()
    a = lib.from_workload(w, ipc_compression=abi.PA_IPC_LZ4_FRAME_GPU)
    lib.load(a, w)
    r = a.flush()
    check_stream(r.ipc_bytes(), want)
    ids = a.last_stack_ids(r.n_unique_stacks).tobytes()
    check_stream(a.stacktraces(ids).ipc_bytes(), o.stacktraces(ids)[0])
    a.close(); o.close()
    print("sanitize_small lz4_gpu ok")


def merge_lz4_gpu():
    from test_ipc_lz4_gpu import check_buffers
    lz4 = abi.PA_IPC_LZ4_FRAME_GPU
    w = synth.config1().head(24_000)
    cuts = [0, 8191, 8191, 8200, 16384, 24_000]
    idx = [np.arange(cuts[i], cuts[i + 1]) for i in range(len(cuts) - 1)]
    parts = [w.rows(ix) for ix in idx]
    aggs = [lib.from_workload(p, ipc_compression=lz4) for p in parts]
    g = lib.MergeGroup.local(aggs)
    for _ in range(2):
        for a, p in zip(aggs, parts):
            lib.load(a, p)
        got = g.flush().ipc_bytes()
        assert got == lib.run(w, ipc_compression=lz4)[0]
        check_buffers(got, oracle_py.run(w)[0])
    g.close()
    for a in aggs:
        a.close()
    print("sanitize_small merge_lz4_gpu ok")


def merge_v1():
    from test_merge_v1 import lru_scenario
    lru_scenario(oracle_py, lib, 3, intervals=6).close()
    lru_scenario(oracle_py, lib, 2, lz4=True, intervals=4).close()
    print("sanitize_small merge_v1 ok")


def registered():
    """PA_CFG_REGISTERED_STACKS: both hash modes, narrow ids, small chunks, v1, a row naming an unregistered stack"""
    for mode in (abi.PA_HASH_PROVIDED, abi.PA_HASH_XXH64X2):
        w = synth.edge_workload(seed=3, n=3000, hash_mode=mode, external=False)
        for kw in ({}, {"frame_id_bytes": 4, "chunk_samples": 700}):
            got, _ = lib.run(w, registered_stacks=True, **kw)
            assert got == oracle_py.run(w)[0]
        w.schema = abi.PA_SCHEMA_V1
        got, _ = lib.run(w, registered_stacks=True)
        assert got == oracle_py.run(w)[0]
    w = synth.ragged(n=3000, u=300, p=1024)
    a = lib.from_workload(w, registered_stacks=True)
    hv, _, _ = a.acquire(2, 0)
    hv[:] = w.hdrs[:2]
    hv["frame_off"] = [0, 1 << 40]
    a.commit(2)
    try:
        a.flush()
        raise AssertionError("an unregistered stack id must fail the flush")
    except lib.PaError:
        pass
    lib.load(a, w)
    assert a.flush().ipc_bytes() == oracle_py.run(w)[0]
    a.close()
    print("sanitize_small registered ok")


def merge_group_stacks():
    from test_merge_group_stacks import lru_quad, one_interval
    w = synth.edge_workload(seed=5, n=2000, hash_mode=abi.PA_HASH_PROVIDED, external=False)
    idx = sharded.shard_rows(w, 2)
    one_interval(oracle_py, lib, w, [idx[0], np.zeros(0, np.int64), idx[1]])
    lru_quad(oracle_py, lib, 3, intervals=4).close()
    print("sanitize_small merge_group_stacks ok")


def merge_group_retire():
    from test_merge_group_retire import GroupChurn
    from test_stack_retirement import windows
    for world, schema in ((3, abi.PA_SCHEMA_V2), (2, abi.PA_SCHEMA_V1)):
        w = synth.ragged(n=3000, u=600, p=1024, max_depth=40, hash_mode=abi.PA_HASH_XXH64X2)
        w.schema = schema
        c = GroupChurn(w, world, max_frames=200_000, max_samples=600, stack_cache_entries=150 if schema == abi.PA_SCHEMA_V1 else 0)
        ws = windows(len(c.sf.hashes), 200, 60, 7)
        for k in range(6):
            hdrs, stacks = c.rows(ws[k], 500)
            r, r1 = c.flush(hdrs, stacks, k)
            assert r.ipc_bytes() == r1.ipc_bytes()
            if schema == abi.PA_SCHEMA_V1:
                ids = c.single.last_stack_ids(r1.n_unique_stacks).tobytes()
                assert c.g.stacktraces(ids).ipc_bytes() == c.single.stacktraces(ids).ipc_bytes()
            c.retire(1)
            c.check_counters()
        c.close()
    print("sanitize_small merge_group_retire ok")


def main():
    oracle_py.build()
    if sys.argv[1:] == ["merge_group_retire"]:
        return merge_group_retire()
    if sys.argv[1:] == ["merge_group_stacks"]:
        return merge_group_stacks()
    if sys.argv[1:] == ["registered"]:
        return registered()
    if sys.argv[1:] == ["lz4_gpu"]:
        return lz4_gpu()
    if sys.argv[1:] == ["merge_lz4_gpu"]:
        return merge_lz4_gpu()
    if sys.argv[1:] == ["merge_v1"]:
        return merge_v1()
    # early copy-out: several intervals through one aggregator, 7 chunks each
    base = synth.edge_workload(seed=3, n=3000, hash_mode=abi.PA_HASH_XXH64X2, external=False)
    for kw in ({}, {"frame_id_bytes": 4}):
        a = lib.from_workload(base, chunk_samples=450, **kw)
        for n in (3000, 3000, 1200, 2999):
            w = base.head(n)
            lib.load(a, w)
            assert a.flush().ipc_bytes() == oracle_py.run(w)[0]
        a.close()
    # hash kernel variants (each reads PA_HASH_VARIANT at create)
    rag = synth.ragged(n=3000, u=300, p=1024)
    for v in ("wide", "widepf", "tma", "tma24x2", "tma13x2r", "tmag13x2"):
        os.environ["PA_HASH_VARIANT"] = v
        for w in (base, rag):
            got, _ = lib.run(w, chunk_samples=700)
            assert got == oracle_py.run(w)[0], v
    os.environ.pop("PA_HASH_VARIANT")
    # v1 LRU store
    big = synth.config2(n=3000, u=800, p=1024)
    big.schema = abi.PA_SCHEMA_V1
    o = oracle_py.Oracle(big, stack_cache_entries=100)
    a = lib.from_workload(big, max_samples=3000, max_frames=3000 * 64, stack_cache_entries=100)
    rng = np.random.Generator(np.random.PCG64(1))
    seen = []
    for k in range(14):
        part = big.rows(np.sort(rng.choice(big.n, 300 if k == 5 else 70, replace=False)))
        part.schema = abi.PA_SCHEMA_V1
        o.ingest(part.hdrs, part.frame_ids)
        want, _ = o.flush()
        lib.load(a, part)
        r = a.flush()
        assert r.ipc_bytes() == want
        ids = [bytes(x) for x in a.last_stack_ids(r.n_unique_stacks)]
        seen += [i for i in ids if i not in set(seen)]
        probe = b"".join(seen[:: max(1, len(seen) // 60)])
        assert a.stacktraces(probe).ipc_bytes() == o.stacktraces(probe)[0]
    assert a.kernel_ms("store_compactions")[1] >= 1
    a.close(); o.close()
    # merged record from 3 shards on one device
    w = synth.edge_workload(seed=4, n=2500, hash_mode=abi.PA_HASH_XXH64X2, external=False)
    idx = sharded.shard_rows(w, 3)
    parts = [w.rows(ix) for ix in idx]
    aggs = [lib.from_workload(p) for p in parts]
    g = lib.MergeGroup.local(aggs)
    for x, p in zip(aggs, parts):
        lib.load(x, p)
    assert g.flush().ipc_bytes() == oracle_py.run(w.rows(np.concatenate(idx)))[0]
    g.close()
    for x in aggs:
        x.close()
    print("sanitize_small ok")


if __name__ == "__main__":
    main()
