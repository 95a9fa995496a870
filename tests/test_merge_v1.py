"""Merge groups of PA_SCHEMA_V1 members. A group must behave, interval by interval, like ONE v1 aggregator fed
[shard 0's rows, shard 1's rows, ...] and driven through the same calls: the sample record, the stacktrace records, the
merged stacktrace_id dictionary (pa_agg_last_stack_ids on every member) and the store counters, byte for byte, through
evictions, revivals, compactions and batches with more unique stacks than the store holds. That single aggregator is itself
pinned to the oracle (oracle_py.Oracle with the same stack cache). Multi-process groups run tests/dist_merge_v1_check.py under
torchrun."""
import os
import subprocess
import sys

import numpy as np
import pyarrow as pa
import pytest

from parca_agent_b200 import abi, sharded, synth
from test_ipc_lz4_gpu import check_buffers

V1 = abi.PA_SCHEMA_V1
LZ4 = abi.PA_IPC_LZ4_FRAME_GPU
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COUNTERS = ("store_evictions", "store_compactions")


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from parca_agent_b200 import lib
    lib.lib()
    return lib


def missing_ids(k):
    return [bytes([0xEE, i]) * 8 for i in range(k)]


class Trio:
    """The oracle, one v1 aggregator and a local merge group of `world` v1 members over the same workload's registrations, fed
    the same intervals and requests. `lz4`: the aggregator and the members use PA_IPC_LZ4_FRAME_GPU (the oracle stays plain)."""

    def __init__(self, oracle, gpu, w, world, cap=0, frames=0, lz4=False, **kw):
        w.schema = V1
        self.w, self.gpu, self.lz4 = w, gpu, lz4
        opts = dict(max_samples=max(w.n, 1), max_frames=max(w.n_frame_ids, 1), stack_cache_entries=cap, stack_cache_frames=frames,
                    ipc_compression=LZ4 if lz4 else abi.PA_IPC_PLAIN, **kw)
        self.o = oracle.Oracle(w, stack_cache_entries=cap)
        self.single = gpu.from_workload(w, **opts)
        self.members = [gpu.from_workload(w, **opts) for _ in range(world)]
        self.g = gpu.MergeGroup.local(self.members)
        self.seen = []

    def same(self, got, single, plain, what):
        assert got == single, "%s: merged bytes differ from the single aggregator's (%d vs %d)" % (what, len(got), len(single))
        if not self.lz4:
            assert single == plain, "%s: the single aggregator differs from the oracle" % what
        elif plain:
            check_buffers(single, plain, python_decoder=len(plain) < (1 << 20))

    def interval(self, idx_lists):
        """one interval: member k gets rows idx_lists[k]; returns the merged dictionary (== the ids of this interval)"""
        parts = [self.w.rows(np.asarray(ix, dtype=np.int64)) for ix in idx_lists]
        ref = self.w.rows(np.concatenate([np.asarray(ix, dtype=np.int64) for ix in idx_lists]))
        for p in parts + [ref]:
            p.schema = V1
        self.o.ingest(ref.hdrs, ref.frame_ids)
        plain, _ = self.o.flush()
        self.gpu.load(self.single, ref)
        r1 = self.single.flush()
        single = r1.ipc_bytes()
        for a, p in zip(self.members, parts):
            self.gpu.load(a, p)
        rg = self.g.flush()
        assert (rg.n_rows, rg.n_unique_stacks) == (r1.n_rows, r1.n_unique_stacks)
        self.same(rg.ipc_bytes(), single, plain, "sample record")
        n = r1.n_unique_stacks
        ids = [bytes(x) for x in self.single.last_stack_ids(n)]
        if plain:
            col = pa.ipc.open_stream(plain).read_all().column("stacktrace_id").chunk(0)
            assert ids == [bytes(x) for x in col.values.dictionary.to_pylist()]
        for a in self.members:
            assert [bytes(x) for x in a.last_stack_ids(n)] == ids
        self.check_counters()
        self.seen += [i for i in ids if i not in set(self.seen)]
        return ids

    def check_counters(self):
        for name in COUNTERS:
            want = self.single.kernel_ms(name)[1]
            assert [a.kernel_ms(name)[1] for a in self.members] == [want] * len(self.members), name

    def request(self, ids):
        blob = b"".join(ids)
        plain, nloc = self.o.stacktraces(blob)
        r1 = self.single.stacktraces(blob)
        rg = self.g.stacktraces(blob)
        assert (rg.n_rows, rg.n_locations) == (r1.n_rows, r1.n_locations) == (len(ids), nloc)
        self.same(rg.ipc_bytes(), r1.ipc_bytes(), plain, "stacktrace record")

    def close(self):
        self.g.close()
        for a in self.members + [self.single]:
            a.close()
        self.o.close()


def one_interval(oracle, gpu, w, idx, **kw):
    t = Trio(oracle, gpu, w, len(idx), **kw)
    ids = t.interval(idx)
    mixed = list(ids)
    for i, m in enumerate(missing_ids(3)):
        mixed.insert((7 * i) % (len(mixed) + 1), m)
    t.request(mixed + ids[:2])
    t.request(list(reversed(ids)))
    t.close()
    return ids


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("mode", [abi.PA_HASH_PROVIDED, abi.PA_HASH_XXH64X2])
def test_config1_and_edge_workloads(oracle, gpu, world, mode):
    w = synth.config1(hash_mode=mode).head(30_000)
    one_interval(oracle, gpu, w, sharded.shard_rows(w, world))
    e = synth.edge_workload(seed=3 + world, n=3000, hash_mode=mode, external=False)
    one_interval(oracle, gpu, e, sharded.shard_rows(e, world))


@pytest.mark.gpu
def test_narrow_ring_members(oracle, gpu):
    w = synth.edge_workload(seed=14, n=4000, hash_mode=abi.PA_HASH_XXH64X2, external=False)
    one_interval(oracle, gpu, w, sharded.shard_rows(w, 3), frame_id_bytes=4)


@pytest.mark.gpu
def test_cuts_inside_stack_and_timestamp_runs(oracle, gpu):
    """every row repeated 7 times in a row: runs of one stacktrace_id and of one timestamp, cut by the shard borders"""
    e = synth.edge_workload(seed=17, n=600, external=False)
    w = e.rows(np.repeat(np.arange(e.n), 7))
    cuts = [0, 7 * 10 + 3, 7 * 11 + 1, 7 * 40 + 6, w.n]
    idx = [np.arange(cuts[i], cuts[i + 1]) for i in range(len(cuts) - 1)]
    for c in cuts[1:-1]:  # the same stack and the same timestamp on both sides of every cut
        assert w.hdrs["hash_hi"][c - 1] == w.hdrs["hash_hi"][c] and w.hdrs["timestamp_ns"][c - 1] == w.hdrs["timestamp_ns"][c]
    one_interval(oracle, gpu, w, idx)


@pytest.mark.gpu
def test_empty_shards_and_all_empty_group(oracle, gpu):
    w = synth.config1().head(5000)
    idx = sharded.shard_rows(w, 2)
    empty = np.zeros(0, np.int64)
    one_interval(oracle, gpu, w, [idx[0], empty, empty, idx[1]])
    t = Trio(oracle, gpu, w, 3)
    assert t.interval([empty] * 3) == []
    ids = t.interval([idx[0], empty, idx[1]])
    assert t.interval([empty] * 3) == []  # an empty interval changes nothing
    t.request(ids + missing_ids(1))
    t.close()


@pytest.mark.gpu
def test_one_provided_id_for_different_stacks_on_different_shards(oracle, gpu):
    """the store keeps the frames of the id's GLOBAL first occurrence, whichever shard holds it"""
    w = synth.edge_workload(seed=23, n=2000, hash_mode=abi.PA_HASH_PROVIDED, external=False)
    nf = w.hdrs["nframes"]
    a = next(i for i in range(w.n) if nf[i] > 0)
    b = next(j for j in range(w.n - 1, w.n // 2, -1) if nf[j] != nf[a])  # a different stack: its depth differs
    for f in ("hash_hi", "hash_lo"):
        w.hdrs[f][b] = w.hdrs[f][a]
    cut = w.n // 2
    # shard 0 holds the first occurrence; then the shard order is swapped, so the later shard's stack comes first globally
    for idx in ([np.arange(0, cut), np.arange(cut, w.n)], [np.arange(cut, w.n), np.arange(0, cut)]):
        one_interval(oracle, gpu, w, idx)


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [0, 5])
def test_external_label_and_label_flags(oracle, gpu, flags):
    w = synth.edge_workload(seed=8, n=1500, label_flags=flags, external=False)
    w.strings = list(w.strings) + [b"cluster", b"prod"]
    w.external_labels = [(len(w.strings) - 2, len(w.strings) - 1)]
    one_interval(oracle, gpu, w, sharded.shard_rows(w, 3))


def lru_scenario(oracle, gpu, world, lz4=False, intervals=8):
    """many small intervals against a small store: evictions every interval, revivals, compactions, one interval with more
    unique stacks than the store holds; requests in between mix live, evicted and never-seen ids"""
    w = synth.config2(n=9000, u=2500, p=4096)
    t = Trio(oracle, gpu, w, world, cap=300, lz4=lz4)
    rng = np.random.Generator(np.random.PCG64(11))
    for k in range(intervals):
        rows = np.sort(rng.choice(w.n, 900 if k == 3 else 220, replace=False))  # interval 3 alone holds more stacks than the store
        cuts = np.sort(rng.choice(len(rows) + 1, world - 1, replace=True))
        t.interval(np.split(rows, cuts))
        probe = [t.seen[int(j)] for j in rng.choice(len(t.seen), min(len(t.seen), 120), replace=False)]
        t.request(probe + missing_ids(1) + probe[:5])
    t.request(t.seen)
    return t


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_store_through_evictions_revivals_and_compactions(oracle, gpu, world):
    t = lru_scenario(oracle, gpu, world, intervals=18 if world == 3 else 8)
    assert t.single.kernel_ms("store_evictions")[1] >= 6
    if world == 3:
        assert t.single.kernel_ms("store_compactions")[1] >= 1
    frames_sent = [a.kernel_ms("store_frames")[1] for a in t.members]
    assert all(x >= 0 for x in frames_sent)
    # a member on its own after merged intervals continues from the group's store: compare with the single aggregator fed
    # those rows next
    part = t.w.rows(np.arange(4000, 4300))
    part.schema = V1
    t.o.ingest(part.hdrs, part.frame_ids)
    plain, _ = t.o.flush()
    gpu.load(t.single, part)
    want = t.single.flush().ipc_bytes()
    m = t.members[world - 1]
    gpu.load(m, part)
    assert m.flush().ipc_bytes() == want == plain
    probe = t.seen[::5] + missing_ids(2)
    blob = b"".join(probe)
    assert m.stacktraces(blob).ipc_bytes() == t.single.stacktraces(blob).ipc_bytes() == t.o.stacktraces(blob)[0]
    for name in COUNTERS:
        assert m.kernel_ms(name)[1] == t.single.kernel_ms(name)[1]
    t.close()


@pytest.mark.gpu
def test_steady_state_exchanges_no_frames(oracle, gpu):
    """a repeated interval: every stack is already in the store, so no frames cross between the shards"""
    w = synth.config1().head(20_000)
    idx = sharded.shard_rows(w, 3)
    t = Trio(oracle, gpu, w, 3)
    t.interval(idx)
    assert sum(a.kernel_ms("store_frames")[1] for a in t.members) > 0
    t.interval([np.zeros(0, np.int64)] * 3)  # an empty interval sends nothing
    assert [a.kernel_ms("store_frames")[1] for a in t.members] == [0, 0, 0]
    ids = t.interval(idx)
    assert [a.kernel_ms("store_frames")[1] for a in t.members] == [0, 0, 0]
    arr = t.members[1].last_stack_ids(len(ids))  # a request straight from pa_agg_last_stack_ids' numpy array
    assert t.g.stacktraces(arr).ipc_bytes() == t.single.stacktraces(arr.tobytes()).ipc_bytes()
    t.close()


@pytest.mark.gpu
def test_unregistered_frame_id_fails_like_one_aggregator(gpu):
    """a frame id beyond the registered frames, in stacks whose first occurrence is on the last shard only: the group fails the
    interval with PA_EINVAL, as one v1 aggregator does (the multi-process form is in dist_merge_v1_check.py)"""
    import dataclasses
    w = synth.edge_workload(seed=46, n=2000, hash_mode=abi.PA_HASH_XXH64X2, external=False)
    w.schema = V1
    fids = np.asarray(w.frame_ids)
    off, nf = w.hdrs["frame_off"].astype(np.int64), w.hdrs["nframes"].astype(np.int64)
    top = int(fids.max())
    first = next(i for i in range(w.n) if nf[i] and int(fids[off[i]:off[i] + nf[i]].max()) == top)
    registered = dataclasses.replace(w, frames=w.frames[:top])
    opts = dict(max_samples=w.n, max_frames=w.n_frame_ids)
    single = gpu.from_workload(registered, **opts)
    gpu.load(single, w)
    with pytest.raises(gpu.PaError) as e:
        single.flush()
    assert e.value.code == -22 and "unregistered frame id" in str(e.value)
    members = [gpu.from_workload(registered, **opts) for _ in range(3)]
    g = gpu.MergeGroup.local(members)
    for a, ix in zip(members, (np.arange(first // 2), np.arange(first // 2, first), np.arange(first, w.n))):
        gpu.load(a, w.rows(ix))
    with pytest.raises(gpu.PaError) as e:
        g.flush()
    assert e.value.code == -22 and "unregistered frame id" in str(e.value)
    g.close()
    for a in members + [single]:
        a.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 3, 5])
def test_lz4_gpu_members(oracle, gpu, world):
    w = synth.config1().head(40_000)
    t = Trio(oracle, gpu, w, world, lz4=True)
    ids = t.interval(sharded.shard_rows(w, world))
    t.request(ids + missing_ids(2))
    t.close()
    e = synth.edge_workload(seed=31 + world, n=3000, hash_mode=abi.PA_HASH_XXH64X2, external=False)
    t = Trio(oracle, gpu, e, world, lz4=True)
    t.interval(sharded.shard_rows(e, world))
    t.close()


@pytest.mark.gpu
def test_lz4_gpu_members_through_evictions(oracle, gpu):
    lru_scenario(oracle, gpu, 3, lz4=True, intervals=6).close()


@pytest.mark.gpu
def test_refusals(gpu):
    w = synth.edge_workload(seed=4, n=200, hash_mode=abi.PA_HASH_XXH64X2, external=False)
    v2 = gpu.from_workload(w)
    w.schema = V1
    v1a = gpu.from_workload(w, stack_cache_entries=1000)
    v1b = gpu.from_workload(w, stack_cache_entries=2000)
    v1c = gpu.from_workload(w, stack_cache_entries=1000, stack_cache_frames=4096)
    for pair, text in (([v1a, v2], b"PA_SCHEMA_V1 and PA_SCHEMA_V2"), ([v2, v1a], b"PA_SCHEMA_V1 and PA_SCHEMA_V2"),
                       ([v1a, v1b], b"stack_cache_entries"), ([v1a, v1c], b"stack_cache_frames")):
        with pytest.raises(gpu.PaError) as e:
            gpu.MergeGroup.local(pair)
        assert e.value.code == -22
        for a in pair:
            assert text in gpu.lib().pa_agg_last_error(a.h)
    # pa_merge_stacktraces needs a v1 group
    g = gpu.MergeGroup.local([v2, gpu.from_workload(synth.edge_workload(seed=4, n=200, hash_mode=abi.PA_HASH_XXH64X2, external=False))])
    with pytest.raises(gpu.PaError) as e:
        g.stacktraces(b"\x01" * 16)
    assert e.value.code == -22 and "PA_SCHEMA_V1" in str(e.value)
    g.close()
    for a in (v2, v1a, v1b, v1c):
        a.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world,transport,mailbox", [(2, "gloo", 0), (3, "gloo", 0), (2, "shm", 4096), (3, "shm", 8192)])
def test_multi_process_groups(world, transport, mailbox):
    """one shard per process on this one GPU; small mailboxes make the store exchange take many rounds; the last case of the
    script mixes schemas and must fail pa_merge_process on every rank"""
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", PA_ONE_GPU="1", PA_MERGE_TRANSPORT=transport, PA_SHM_MAILBOX=str(mailbox))
    port = 29611 + world + (10 if transport == "shm" else 0)
    p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
                        "--master-port", str(port), os.path.join(ROOT, "tests", "dist_merge_v1_check.py")], capture_output=True, text=True, env=env, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    assert "merge-v1 ok world=%d transport=%s" % (world, transport) in p.stdout
