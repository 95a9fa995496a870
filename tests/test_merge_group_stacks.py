"""Merge groups of PA_CFG_GROUP_STACKS members: registered stacks with group-wide ids. Every member registers the same
group_stack_form and its rows name those stacks; the merged stream must be byte for byte the one a single aggregator returns
for [shard 0's rows, shard 1's rows, ...]. Each case compares the group with the oracle on the concatenated rows, with a ring
group fed the same rows and with one group-stacks aggregator on the concatenated rows. Multi-process groups run
tests/dist_merge_group_stacks_check.py under torchrun."""
import dataclasses
import os
import subprocess
import sys

import numpy as np
import pytest

from parca_agent_b200 import abi, sharded, synth
from test_scale_edges import merge_batch

V1 = abi.PA_SCHEMA_V1
LZ4 = abi.PA_IPC_LZ4_FRAME_GPU
EINVAL = -22
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
COUNTERS = ("store_evictions", "store_compactions")


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from parca_agent_b200 import lib
    lib.lib()
    return lib


def sub_form(gpu, form, s0, s1):
    """stacks [s0, s1) of a StackForm, as one register_stacks call takes them"""
    o = form.offsets
    return gpu.StackForm(form.hashes[s0:s1], form.frames[int(o[s0]):int(o[s1])], o[s0:s1 + 1] - o[s0], None)


def register(a, w, form):
    a.register_stacks(form.frames, form.offsets, form.hashes if w.hash_mode == abi.PA_HASH_PROVIDED else None)


class Quad:
    """The oracle, one group-stacks aggregator, a ring group and a group-stacks group of `world` members, all over the same
    workload's registrations and fed the same intervals. `form` is registered on every group-stacks aggregator."""

    def __init__(self, oracle, gpu, w, world, form, cap=0, lz4=False, arena=0, **kw):
        self.w, self.gpu, self.lz4, self.v1 = w, gpu, lz4, w.schema == V1
        opts = dict(max_samples=max(w.n, 1), stack_cache_entries=cap, ipc_compression=LZ4 if lz4 else abi.PA_IPC_PLAIN, **kw)
        nf = max(w.n_frame_ids, 1)
        nreg = max(len(form.frames), arena, 1)  # (arena: the frames of the stacks add_stacks registers later too)
        self.o = oracle.Oracle(w, stack_cache_entries=cap)
        self.single = gpu.from_workload(w, group_form=form, max_frames=nreg, **opts)
        self.ring = [gpu.from_workload(w, max_frames=nf, **opts) for _ in range(world)]
        self.members = [gpu.from_workload(w, group_form=form, max_frames=nreg, **opts) for _ in range(world)]
        self.g_ring = gpu.MergeGroup.local(self.ring)
        self.g = gpu.MergeGroup.local(self.members)

    def add_stacks(self, form):
        for a in self.members + [self.single]:
            register(a, self.w, form)

    def interval(self, idx, sor):
        """member k gets rows idx[k], naming the registered stacks sor[k]; returns the merged dictionary (v1) or None"""
        parts = [self.w.rows(np.asarray(ix, dtype=np.int64)) for ix in idx]
        ref = self.w.rows(np.concatenate([np.asarray(ix, dtype=np.int64) for ix in idx]))
        self.o.ingest(ref.hdrs, ref.frame_ids)
        plain, _ = self.o.flush()
        self.gpu.load(self.single, ref, stack_of_row=np.concatenate([np.asarray(s, dtype=np.uint64) for s in sor]))
        r1 = self.single.flush()
        single = r1.ipc_bytes()
        for a, p in zip(self.ring, parts):
            self.gpu.load(a, p)
        ring = self.g_ring.flush().ipc_bytes()
        for a, p, s in zip(self.members, parts, sor):
            self.gpu.load(a, p, stack_of_row=s)
        rg = self.g.flush()
        assert (rg.n_rows, rg.n_unique_stacks) == (r1.n_rows, r1.n_unique_stacks)
        got = rg.ipc_bytes()
        assert got == single, "merged bytes differ from the single group-stacks aggregator's (%d vs %d)" % (len(got), len(single))
        assert got == ring, "merged bytes differ from the ring group's"
        if not self.lz4:
            assert single == plain, "the single aggregator differs from the oracle"
        if not self.v1:
            return None
        ids = [bytes(x) for x in self.single.last_stack_ids(r1.n_unique_stacks)]
        for a in self.members + self.ring:
            assert [bytes(x) for x in a.last_stack_ids(len(ids))] == ids
        for name in COUNTERS:
            want = self.single.kernel_ms(name)[1]
            assert [a.kernel_ms(name)[1] for a in self.members] == [want] * len(self.members), name
        return ids

    def refs(self):
        return [a.kernel_ms("store_refs")[1] for a in self.members], [a.kernel_ms("store_frames")[1] for a in self.members]

    def request(self, ids):
        blob = b"".join(ids)
        plain, _ = self.o.stacktraces(blob)
        want = self.single.stacktraces(blob).ipc_bytes()
        assert self.g.stacktraces(blob).ipc_bytes() == want == self.g_ring.stacktraces(blob).ipc_bytes()
        if not self.lz4:
            assert want == plain

    def close(self):
        self.g.close()
        self.g_ring.close()
        for a in self.members + self.ring + [self.single]:
            a.close()
        self.o.close()


def one_interval(oracle, gpu, w, idx, **kw):
    """the shards' stacks through group_stack_form, one interval"""
    form, sor = gpu.group_stack_form([w.rows(np.asarray(ix, dtype=np.int64)) for ix in idx])
    q = Quad(oracle, gpu, w, len(idx), form, **kw)
    ids = q.interval(idx, sor)
    if ids:
        q.request(ids + [b"\xEE\x01" * 8])
    q.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 8])
def test_config1_pid_sharded(oracle, gpu, world):
    w = synth.config1().head(30_000)
    one_interval(oracle, gpu, w, sharded.shard_rows(w, world))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [abi.PA_HASH_PROVIDED, abi.PA_HASH_XXH64X2])
def test_edge_workload(oracle, gpu, mode):
    e = synth.edge_workload(seed=61, n=3000, hash_mode=mode, external=False)
    one_interval(oracle, gpu, e, sharded.shard_rows(e, 3))


@pytest.mark.gpu
@pytest.mark.parametrize("schema", [abi.PA_SCHEMA_V2, V1])
def test_provided_id_on_different_stacks_on_different_shards(oracle, gpu, schema):
    """two registered stacks share one provided id: the frames of the id's GLOBAL first occurrence win, whichever shard holds it
    (v2: in the location-index stream; v1: in every member's store, which only the reference exchange fills)"""
    w = synth.edge_workload(seed=23, n=2000, hash_mode=abi.PA_HASH_PROVIDED, external=False)
    w.schema = schema
    nf = w.hdrs["nframes"]
    a = next(i for i in range(w.n) if nf[i] > 0)
    b = next(j for j in range(w.n - 1, w.n // 2, -1) if nf[j] != nf[a])
    for f in ("hash_hi", "hash_lo"):
        w.hdrs[f][b] = w.hdrs[f][a]
    cid = int(w.hdrs["hash_hi"][a]).to_bytes(8, "big") + int(w.hdrs["hash_lo"][a]).to_bytes(8, "big")  # its stacktrace_id
    cut = w.n // 2
    # shard 0 holds the first occurrence (row a); then the shard order is swapped, so row b's stack comes first globally
    for idx in ([np.arange(0, cut), np.arange(cut, w.n)], [np.arange(cut, w.n), np.arange(0, cut)]):
        form, sor = gpu.group_stack_form([w.rows(ix) for ix in idx])
        assert len({(int(h[0]), int(h[1])) for h in form.hashes}) < len(form.hashes)  # the id names two registered stacks
        q = Quad(oracle, gpu, w, len(idx), form)
        ids = q.interval(idx, sor)
        if schema == V1:
            assert cid in ids
            q.request([cid])  # the store's frames for the id, against the single aggregator, the ring group and the oracle
            q.request(ids)
        q.close()


@pytest.mark.gpu
def test_all_zero_id(oracle, gpu):
    w = synth.edge_workload(seed=62, n=1500, hash_mode=abi.PA_HASH_PROVIDED, external=False)
    zero = np.arange(w.n) % 7 == 3
    w.hdrs["hash_hi"][zero] = 0
    w.hdrs["hash_lo"][zero] = 0
    one_interval(oracle, gpu, w, sharded.shard_rows(w, 3))


@pytest.mark.gpu
def test_empty_and_tiny_shards(oracle, gpu):
    w = synth.config1().head(5000)
    e = np.zeros(0, np.int64)
    idx = sharded.shard_rows(w, 2)
    one_interval(oracle, gpu, w, [idx[0][:1], e, idx[0][1:], e, idx[1][:2], idx[1][2:], e])
    one_interval(oracle, gpu, w, [e, np.arange(3), e])


@pytest.mark.gpu
def test_narrow_ids(oracle, gpu):
    w = synth.edge_workload(seed=14, n=4000, hash_mode=abi.PA_HASH_XXH64X2, external=False)
    one_interval(oracle, gpu, w, sharded.shard_rows(w, 3), frame_id_bytes=4)


@pytest.mark.gpu
def test_external_labels(oracle, gpu):
    w = synth.edge_workload(seed=8, n=1500, external=False)
    w.strings = list(w.strings) + [b"cluster", b"prod"]
    w.external_labels = [(len(w.strings) - 2, len(w.strings) - 1)]
    one_interval(oracle, gpu, w, sharded.shard_rows(w, 3))


@pytest.mark.gpu
@pytest.mark.parametrize("schema", [abi.PA_SCHEMA_V2, V1])
def test_repeated_intervals_and_stacks_registered_between_them(oracle, gpu, schema):
    """intervals 0 and 1 name the first half of the stacks only; the rest is registered on every member before interval 2"""
    w = synth.edge_workload(seed=63, n=3000, hash_mode=abi.PA_HASH_PROVIDED, external=False)
    w.schema = schema
    half = np.arange(w.n // 2)
    form, _ = gpu.group_stack_form([w.rows(half), w.rows(np.arange(w.n // 2, w.n))])
    k = int(form.stack_of_row[:w.n // 2].max()) + 1
    q = Quad(oracle, gpu, w, 3, sub_form(gpu, form, 0, k), arena=len(form.frames))
    cuts = [np.arange(0, 500), np.arange(500, 900), np.arange(900, w.n // 2)]
    sor = [form.stack_of_row[c] for c in cuts]
    q.interval(cuts, sor)
    q.interval(cuts, sor)
    q.add_stacks(sub_form(gpu, form, k, len(form.hashes)))
    cuts = [np.arange(w.n // 2 - 300, w.n - 700), np.arange(w.n - 700, w.n), np.arange(0, 100)]
    q.interval(cuts, [form.stack_of_row[c] for c in cuts])
    q.close()


@pytest.mark.gpu
def test_tile_border_batches_three_shards(oracle, gpu):
    """the adversarial three-shard batch of test_scale_edges (more than 0.5 M rows): run-end warp and tile borders at and
    around the shard borders"""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for mode in (abi.PA_HASH_XXH64X2, abi.PA_HASH_PROVIDED):
        w = dataclasses.replace(merge_batch(sms), hash_mode=mode)
        assert w.n >= 500_000
        idx = [np.arange(p0, p1) for p0, p1 in w.meta["parts"]]
        one_interval(oracle, gpu, w, idx, chunk_samples=w.n)


# ---- v1 and LZ4 ---------------------------------------------------------------------------------------------------------
def lru_quad(oracle, gpu, world, lz4=False, intervals=8):
    """small intervals against a small store: evictions, revivals, compactions, one interval with more stacks than the store"""
    w = synth.config2(n=9000, u=2500, p=4096)
    w.schema = V1
    form, _ = gpu.group_stack_form([w])
    q = Quad(oracle, gpu, w, world, form, cap=300, lz4=lz4)
    rng = np.random.Generator(np.random.PCG64(12))
    seen = []
    for k in range(intervals):
        rows = np.sort(rng.choice(w.n, 900 if k == 3 else 220, replace=False))
        idx = np.split(rows, np.sort(rng.choice(len(rows) + 1, world - 1, replace=True)))
        ids = q.interval(idx, [form.stack_of_row[ix] for ix in idx])
        seen += [i for i in ids if i not in set(seen)]
        probe = [seen[int(j)] for j in rng.choice(len(seen), min(len(seen), 100), replace=False)]
        q.request(probe + [b"\xEE\x02" * 8])
    q.request(seen)
    return q


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_v1_store_through_evictions(oracle, gpu, world):
    q = lru_quad(oracle, gpu, world, intervals=12 if world == 3 else 8)
    assert q.single.kernel_ms("store_evictions")[1] >= 5
    q.close()


@pytest.mark.gpu
def test_v1_cold_interval_sends_references_and_steady_state_nothing(oracle, gpu):
    w = synth.config1().head(20_000)
    w.schema = V1
    idx = sharded.shard_rows(w, 3)
    form, sor = gpu.group_stack_form([w.rows(ix) for ix in idx])
    q = Quad(oracle, gpu, w, 3, form)
    ids = q.interval(idx, sor)
    refs, frames = q.refs()
    assert sum(refs) == len(ids) and frames == [0, 0, 0]  # one reference per stack (config 1 has no stack of depth 0)
    q.interval(idx, sor)
    assert q.refs() == ([0, 0, 0], [0, 0, 0])
    q.request(ids[::3])
    q.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 3])
def test_lz4_gpu_members(oracle, gpu, world):
    w = synth.config1().head(40_000)
    one_interval(oracle, gpu, w, sharded.shard_rows(w, world), lz4=True)
    e = synth.edge_workload(seed=31 + world, n=3000, hash_mode=abi.PA_HASH_XXH64X2, external=False)
    e.schema = V1
    one_interval(oracle, gpu, e, sharded.shard_rows(e, world), lz4=True)


@pytest.mark.gpu
def test_lz4_gpu_v1_through_evictions(oracle, gpu):
    lru_quad(oracle, gpu, 3, lz4=True, intervals=5).close()


# ---- refusals -----------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_flag_needs_registered_stacks(gpu):
    w = synth.edge_workload(seed=4, n=200, external=False)
    with pytest.raises(gpu.PaError) as e:
        gpu.from_workload(w, flags=abi.PA_CFG_GROUP_STACKS)
    assert e.value.code == EINVAL


@pytest.mark.gpu
def test_mixed_groups_are_refused(gpu):
    w = synth.edge_workload(seed=4, n=200, hash_mode=abi.PA_HASH_XXH64X2, external=False)
    form, _ = gpu.group_stack_form([w])
    L = gpu.lib()
    for kinds in (("grp", "ring"), ("ring", "grp", "grp"), ("grp", "plain"), ("plain", "grp", "ring")):
        make = {"grp": lambda: gpu.from_workload(w, group_form=form), "ring": lambda: gpu.from_workload(w),
                "plain": lambda: gpu.from_workload(w, registered_stacks=True)}
        members = [make[k]() for k in kinds]  # fresh members: every last error below comes from this refusal
        with pytest.raises(gpu.PaError) as e:
            gpu.MergeGroup.local(members)
        assert e.value.code == EINVAL
        for k, a in zip(kinds, members):
            assert (b"merge groups do not support PA_CFG_REGISTERED_STACKS" if k == "plain" else b"mixes PA_CFG_GROUP_STACKS") in L.pa_agg_last_error(a.h)
        for a in members:  # every member still flushes alone
            gpu.load(a, w)
            assert a.flush().n_rows == w.n
            a.close()


@pytest.mark.gpu
@pytest.mark.parametrize("change", ["count", "frame"])
def test_differing_registries_fail_every_member(oracle, gpu, change):
    w = synth.edge_workload(seed=64, n=1200, hash_mode=abi.PA_HASH_XXH64X2, external=False)
    idx = sharded.shard_rows(w, 3)
    form, sor = gpu.group_stack_form([w.rows(ix) for ix in idx])
    other = form
    if change == "count":  # one more stack on the last member
        other = gpu.StackForm(np.concatenate([form.hashes, form.hashes[:1]]), np.concatenate([form.frames, form.frames[:2]]),
                              np.concatenate([form.offsets, form.offsets[-1:] + 2]), None)
    else:  # the same count and arena length, one frame id changed
        fr = np.array(form.frames, copy=True)
        fr[len(fr) // 2] = (int(fr[len(fr) // 2]) + 1) % len(w.frames)
        other = gpu.StackForm(form.hashes, fr, form.offsets, None)
    members = [gpu.from_workload(w, group_form=form if k < 2 else other) for k in range(3)]
    g = gpu.MergeGroup.local(members)
    for a, p, s in zip(members, idx, sor):
        gpu.load(a, w.rows(p), stack_of_row=s)
    with pytest.raises(gpu.PaError) as e:
        g.flush()
    assert e.value.code == EINVAL and "identical stacks" in str(e.value)
    for a in members:
        assert b"identical stacks" in gpu.lib().pa_agg_last_error(a.h)
    g.close()
    want, _ = oracle.run(w.rows(idx[0]))
    for k, (a, p, s) in enumerate(zip(members, idx, sor)):  # every member still flushes alone
        gpu.load(a, w.rows(p), stack_of_row=s)
        got = a.flush().ipc_bytes()
        if k == 0:
            assert got == want
    for a in members:
        a.close()


# ---- across processes ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("world,transport,mailbox", [(2, "gloo", 0), (3, "gloo", 0), (2, "shm", 0), (3, "shm", 8192)])
def test_multi_process_groups(world, transport, mailbox):
    """one shard per process on this one GPU: v2, v1 and GPU-LZ4 groups, then a rank with a differing registry, which must
    fail pa_merge_process on every rank"""
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", PA_ONE_GPU="1", PA_MERGE_TRANSPORT=transport, PA_SHM_MAILBOX=str(mailbox))
    port = 29641 + world + (10 if transport == "shm" else 0) + (20 if mailbox else 0)
    p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
                        "--master-port", str(port), os.path.join(ROOT, "tests", "dist_merge_group_stacks_check.py")],
                       capture_output=True, text=True, env=env, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    assert "merge-group-stacks ok world=%d transport=%s" % (world, transport) in p.stdout
