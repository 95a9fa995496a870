"""Group-wide stack retirement (PA_CFG_GROUP_RETIRE): the members of a merge group register the same stacks by handle and retire
them together through pa_merge_retire_stacks. Interval after interval, a group fed shards [0..W) must give the stream, the
retired handles and the registry counters of ONE PA_CFG_RETIRE_STACKS aggregator fed the same registrations, the concatenated
rows and the same retire calls; on the plain schema also the oracle's (through the ring-mode stream), and the handles of
test_stack_retirement's model of the contract."""
import os
import subprocess
import sys

import numpy as np
import pytest

from parca_agent_b200 import abi, lib, synth
from test_scale_edges import merge_batch
from test_stack_retirement import Model, pack, ring_workload, same_record, windows

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EINVAL = -22
REG, GSTACKS, RETIRE, GRETIRE = abi.PA_CFG_REGISTERED_STACKS, abi.PA_CFG_GROUP_STACKS, abi.PA_CFG_RETIRE_STACKS, abi.PA_CFG_GROUP_RETIRE
GROUP = REG | GSTACKS | GRETIRE


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    lib.lib()
    return lib


class GroupChurn:
    """A group of `world` PA_CFG_GROUP_RETIRE members, one PA_CFG_RETIRE_STACKS aggregator and the model, driven through the same
    registrations, rows and retire calls. The caller's lookup (stack -> handle) is the one map every shard shares."""

    def __init__(self, w, world, max_frames, max_samples, **kw_agg):
        self.w, self.world, self.sf = w, world, lib.stack_form(w)
        self.depth = np.diff(self.sf.offsets.astype(np.int64))
        mk = lambda flags: lib.from_workload(w.head(0), max_samples=max_samples, max_frames=max_frames, flags=flags, **kw_agg)
        self.members = [mk(GROUP) for _ in range(world)]
        self.single = mk(REG | RETIRE)
        self.g = lib.MergeGroup.local(self.members)
        self.m = Model(max_frames)
        self.lookup, self.rng = {}, np.random.Generator(np.random.PCG64(11 + world))

    def register(self, stacks):
        """on every member, the single aggregator and the model: the same handles everywhere"""
        if not len(stacks):
            return
        fr, o, hs = pack(self.sf, stacks)
        hs = hs if self.w.hash_mode == abi.PA_HASH_PROVIDED else None
        got = [[int(x) for x in a.register_stack_handles(fr, o, hs)] for a in self.members + [self.single]]
        assert all(h == got[0] for h in got), "members handed out different handles"
        assert got[0] == self.m.register([int(self.depth[s]) for s in stacks])
        self.lookup.update(zip((int(s) for s in stacks), got[0]))

    def rows(self, window, n):
        self.register([s for s in dict.fromkeys(int(x) for x in window) if s not in self.lookup])
        idx = np.sort(self.rng.choice(self.w.n, n, replace=n > self.w.n))
        return np.array(self.w.hdrs[idx], copy=True), self.rng.choice(window, n)

    def cuts(self, n, k):
        """uneven shard borders; some intervals have empty and one-row shards"""
        c = np.sort(self.rng.choice(n + 1, self.world - 1, replace=True))
        if self.world > 2 and k % 4 == 1:
            c[0] = c[1] = c[0]  # an empty shard
        if self.world > 2 and k % 4 == 2 and n > 2:
            c[0], c[1] = 0, 1  # an empty first shard and a one-row shard
        return c

    def load(self, a, hdrs, handles):
        hv, _, _ = a.acquire(len(hdrs), 0)
        hv[:] = hdrs
        hv["frame_off"] = handles
        a.commit(len(hdrs))

    def flush(self, hdrs, stacks, k=0, cuts=None):
        """(group result, single result): the group's shards and the single aggregator take the same rows"""
        handles = np.array([self.lookup[int(s)] for s in stacks], dtype=np.uint64)
        cuts = self.cuts(len(hdrs), k) if cuts is None else cuts
        for a, hp, sp in zip(self.members, np.split(hdrs, cuts), np.split(handles, cuts)):
            self.load(a, hp, sp)
        self.load(self.single, hdrs, handles)
        self.m.stage()
        assert self.m.batch([int(h) for h in handles])
        r = self.g.flush()
        return r, self.single.flush()

    def retire(self, idle, cap=None):
        got = [int(x) for x in self.g.retire_stacks(idle, cap)]
        assert got == [int(x) for x in self.single.retire_stacks(idle, cap)] == self.m.retire(idle, cap)
        gone = set(got)
        self.lookup = {s: h for s, h in self.lookup.items() if h not in gone}
        return got

    def check_counters(self):
        want = self.single.stack_counters()
        assert {k: want[k] for k in self.m.counters()} == self.m.counters()
        for a in self.members:
            assert a.stack_counters() == want
        return want

    def close(self):
        self.g.close()
        for a in self.members + [self.single]:
            a.close()


CHURN = [  # (world, hash mode, frame id bytes, output)
    (1, abi.PA_HASH_PROVIDED, 8, "v2"),
    (2, abi.PA_HASH_XXH64X2, 4, "v1"),
    (2, abi.PA_HASH_PROVIDED, 4, "v2"),
    (3, abi.PA_HASH_PROVIDED, 8, "lz4"),
    (3, abi.PA_HASH_XXH64X2, 8, "v2"),
    (8, abi.PA_HASH_XXH64X2, 8, "v1"),
    (8, abi.PA_HASH_PROVIDED, 8, "lz4"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("world,mode,idb,out", CHURN)
def test_churn_matches_one_retiring_aggregator(oracle, gpu, world, mode, idb, out):
    """20 intervals over a window that shifts every interval, retire(1..3) after each, re-registration into freed slots"""
    w = synth.ragged(n=20_000, u=3_000, p=8_192, max_depth=90, hash_mode=mode)
    w.schema = abi.PA_SCHEMA_V1 if out == "v1" else abi.PA_SCHEMA_V2
    comp = abi.PA_IPC_LZ4_FRAME_GPU if out == "lz4" else abi.PA_IPC_PLAIN
    c = GroupChurn(w, world, max_frames=4_000_000, max_samples=4_000, frame_id_bytes=idb, ipc_compression=comp,
                   stack_cache_entries=700 if out == "v1" else 0)
    ws = windows(len(c.sf.hashes), 900, 140, 21)
    seen, retired = [], 0
    for k in range(20):
        hdrs, stacks = c.rows(ws[k], 2500 if k != 6 else 3900)
        r, r1 = c.flush(hdrs, stacks, k)
        want = r1.ipc_bytes()
        assert r.ipc_bytes() == want, "interval %d differs from the single retiring aggregator" % k
        assert (r.n_rows, r.n_unique_stacks) == (r1.n_rows, r1.n_unique_stacks)
        if out == "v2":
            assert want == oracle.run(ring_workload(w, c.sf, hdrs, stacks))[0]
        elif out == "lz4":
            same_record(want, oracle.run(ring_workload(w, c.sf, hdrs, stacks))[0])
        else:
            ids = [bytes(x) for x in c.single.last_stack_ids(r1.n_unique_stacks)]
            seen += [i for i in ids if i not in set(seen)]
            probe = b"".join([seen[int(j)] for j in c.rng.choice(len(seen), min(len(seen), 150), replace=False)] + [b"\xee" * 16])
            assert c.g.stacktraces(probe).ipc_bytes() == c.single.stacktraces(probe).ipc_bytes()
        retired += len(c.retire(1 + k % 3))
        c.check_counters()
    assert retired > 1000 and c.single.stack_counters()["stack_compactions"] >= 1
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_one_shard_keeps_a_stack_alive(gpu, world):
    """a stack named only by the last member's rows is not idle, although every other member's own last_use says it is"""
    w = synth.edge_workload(seed=31, n=400, hash_mode=abi.PA_HASH_XXH64X2, external=False)
    c = GroupChurn(w, world, max_frames=100_000, max_samples=w.n)
    c.register(list(range(10)))
    hdrs = np.array(w.hdrs[:40], copy=True)
    stacks = [i % 5 for i in range(39)] + [7]  # stack 7: the last row only, on the last shard
    c.flush(hdrs, stacks, cuts=np.full(world - 1, 39))
    assert c.retire(1) == [5, 6, 8, 9]
    c.check_counters()
    c.close()


@pytest.mark.gpu
def test_registration_concurrent_with_the_retire_call(gpu):
    """a producer registers on member 0 before the retire call and on the other members after it: the members' registry digests
    must still agree, so the next interval works"""
    w = synth.edge_workload(seed=33, n=400, hash_mode=abi.PA_HASH_PROVIDED, external=False)
    c = GroupChurn(w, 3, max_frames=100_000, max_samples=w.n)
    c.register(list(range(10)))
    hdrs = np.array(w.hdrs[:60], copy=True)
    c.flush(hdrs, [i % 4 for i in range(60)])
    fr, o, hs = pack(c.sf, [20, 21])
    early = [int(x) for x in c.members[0].register_stack_handles(fr, o, hs)]
    assert [int(x) for x in c.single.register_stack_handles(fr, o, hs)] == early == c.m.register([int(c.depth[20]), int(c.depth[21])])
    assert c.retire(1) == list(range(4, 10))
    for a in c.members[1:]:
        assert [int(x) for x in a.register_stack_handles(fr, o, hs)] == early
    c.lookup.update({20: early[0], 21: early[1]})
    st = [[0, 1, 20, 21][i % 4] for i in range(60)]
    for _ in range(2):  # the grace batch, then the batch after the stage that frees the retired stacks
        r, r1 = c.flush(hdrs, st)
        assert r.ipc_bytes() == r1.ipc_bytes()
    c.check_counters()
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [abi.PA_HASH_PROVIDED, abi.PA_HASH_XXH64X2])
def test_grace_batch_then_refusal_then_reuse(oracle, gpu, mode):
    w = synth.edge_workload(seed=21, n=400, hash_mode=mode, external=False)
    c = GroupChurn(w, 3, max_frames=100_000, max_samples=w.n)
    n_st = len(c.sf.hashes)
    c.register(list(range(n_st)))
    hdrs = np.array(w.hdrs[:60], copy=True)
    thirds = np.array([20, 40])
    c.flush(hdrs, [i % 2 for i in range(60)], cuts=thirds)
    old = dict(c.lookup)
    assert c.retire(1) == [old[s] for s in range(2, n_st)]
    # the grace batch: rows of shard 1 still name retired stacks and come out exactly right
    st = [i % 2 if not 20 <= i < 40 else 2 + i % (n_st - 2) for i in range(60)]
    c.lookup = old
    r, r1 = c.flush(hdrs, st, cuts=thirds)
    assert r.ipc_bytes() == r1.ipc_bytes() == oracle.run(ring_workload(w, c.sf, hdrs, st))[0]
    # one batch later a retired handle on shard 2 fails the group, on every member, and the single aggregator alike
    bad = np.array([old[0]] * 59 + [old[3]], dtype=np.uint64)
    for a, hp, sp in zip(c.members, np.split(hdrs, thirds), np.split(bad, thirds)):
        c.load(a, hp, sp)
    c.load(c.single, hdrs, bad)
    c.m.stage()
    assert not c.m.batch([int(h) for h in bad])
    with pytest.raises(lib.PaError) as e:
        c.g.flush()
    assert e.value.code == EINVAL and "unregistered stack id" in str(e.value)
    with pytest.raises(lib.PaError) as e:
        c.single.flush()
    assert e.value.code == EINVAL
    # the next interval works; a new registration reuses the lowest freed slot under the next generation on every member
    c.lookup = {0: old[0], 1: old[1]}
    new = [n_st - 1, 5]
    c.register(new)
    assert [c.lookup[s] for s in new] == [1 << 32 | 2, 1 << 32 | 3]
    st = [new[i % 2] if i >= 30 else i % 2 for i in range(60)]
    r, r1 = c.flush(hdrs, st, cuts=thirds)
    assert r.ipc_bytes() == r1.ipc_bytes() == oracle.run(ring_workload(w, c.sf, hdrs, st))[0]
    c.check_counters()
    c.close()


@pytest.mark.gpu
def test_v1_store_reads_each_members_own_arena_layout(gpu):
    """Two members whose arenas hold the same stacks at different offsets. R1 takes a freed low slot; member 0 uploads it at its
    stage, member 1 only at pa_merge_process, where a 65535-id R2 makes both grow (and compact) the arena: member 0's compaction
    moves R1 into slot order, member 1 appends it after the compacted stacks. A cold v1 interval whose store needs R1 must still
    give the single aggregator's stacktrace records, which arena offsets as store references would not."""
    w = synth.config2(n=4000, u=400, p=4096)
    w.schema = abi.PA_SCHEMA_V1
    c = GroupChurn(w, 2, max_frames=1_000_000, max_samples=w.n, stack_cache_entries=2000)
    c.register(list(range(60)))
    hdrs = np.array(w.hdrs[:200], copy=True)
    named = [s for s in range(60) if s != 3]
    c.flush(hdrs, [named[i % len(named)] for i in range(200)])
    assert c.retire(1) == [3]
    c.flush(hdrs, [named[i % len(named)] for i in range(200)])  # the grace batch
    c.flush(hdrs, [named[i % len(named)] for i in range(200)])  # its stage frees slot 3
    r1_stack, r2 = 100, np.arange(65535, dtype=np.uint64) % np.uint64(len(w.frames))
    fr, o, hs = pack(c.sf, [r1_stack])
    hs = hs if w.hash_mode == abi.PA_HASH_PROVIDED else None
    r2_hash = np.array([[0x5EED, 0x65535]], dtype=np.uint64) if hs is not None else None
    # member 0: R1 before its stage
    h1 = int(c.members[0].register_stack_handles(fr, o, hs)[0])
    assert h1 == 1 << 32 | 3
    st = np.array([c.lookup[named[i % len(named)]] for i in range(100)] + [h1] * 100, dtype=np.uint64)
    before = [a.stack_counters() for a in c.members]
    for a, hp, sp in zip(c.members, np.split(hdrs, [100]), np.split(st, [100])):
        c.load(a, hp, sp)
        a.stage()
    mid = [a.stack_counters() for a in c.members]
    # member 0: R2; member 1: R1 and R2, all between the stage and pa_merge_process
    assert int(c.members[0].register_stack_handles(r2, [0, 65535], r2_hash)[0]) == 60
    assert int(c.members[1].register_stack_handles(fr, o, hs)[0]) == h1
    assert int(c.members[1].register_stack_handles(r2, [0, 65535], r2_hash)[0]) == 60
    c.g.process()
    c.g.plan()
    r = c.g.collect()
    after = [a.stack_counters() for a in c.members]
    for b, m, f in zip(before, mid, after):
        assert m["stack_compactions"] == b["stack_compactions"] and m["stack_frames_dead"] > 0  # no compaction at the stage
        assert f["stack_compactions"] == b["stack_compactions"] + 1 and f["stack_frames_dead"] == 0  # one at the process
    assert c.members[1].kernel_ms("store_refs")[1] + c.members[0].kernel_ms("store_refs")[1] > 0
    # the single aggregator: the same registrations, the concatenated rows
    assert int(c.single.register_stack_handles(fr, o, hs)[0]) == h1
    assert int(c.single.register_stack_handles(r2, [0, 65535], r2_hash)[0]) == 60
    c.load(c.single, hdrs, st)
    r1 = c.single.flush()
    assert r.ipc_bytes() == r1.ipc_bytes()
    ids = c.single.last_stack_ids(r1.n_unique_stacks).tobytes()
    assert c.g.stacktraces(ids).ipc_bytes() == c.single.stacktraces(ids).ipc_bytes()
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [abi.PA_HASH_PROVIDED, abi.PA_HASH_XXH64X2])
def test_compaction_and_regrowth_in_a_group(oracle, gpu, mode):
    """a 65535-id stack registered and retired at a moving offset: dead frames outweigh live ones (compaction at a stage) and
    pending frames overflow the arena (regrowth)"""
    w = synth.edge_workload(seed=23, n=400, hash_mode=mode, external=False)
    c = GroupChurn(w, 3, max_frames=1_000_000, max_samples=w.n)
    n_st = len(c.sf.hashes)
    big = np.arange(65535, dtype=np.uint64) % np.uint64(len(w.frames))
    hdrs = np.array(w.hdrs[:90], copy=True)
    for k in range(6):
        c.register([s for s in (k % n_st, (k + 1) % n_st) if s not in c.lookup])
        hs = np.array([[0xB16 + k, 0xF00D]], dtype=np.uint64) if mode == abi.PA_HASH_PROVIDED else None
        got = [int(a.register_stack_handles(big, [0, 65535], hs)[0]) for a in c.members + [c.single]]
        assert len(set(got)) == 1 and got[0] == c.m.register([65535])[0]
        stacks = [k % n_st, (k + 1) % n_st] * 45
        handles = [c.lookup[s] for s in stacks[:-1]] + [got[0]]
        cuts = np.array([30, 60])
        for a, hp, sp in zip(c.members, np.split(hdrs, cuts), np.split(np.array(handles, np.uint64), cuts)):
            c.load(a, hp, sp)
        c.load(c.single, hdrs, np.array(handles, np.uint64))
        c.m.stage()
        assert c.m.batch(handles)
        r = c.g.flush()
        assert r.ipc_bytes() == c.single.flush().ipc_bytes()
        c.retire(1)
        c.check_counters()
    assert c.single.stack_counters()["stack_compactions"] >= 2
    c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [abi.PA_HASH_XXH64X2, abi.PA_HASH_PROVIDED])
def test_tile_border_batch_three_shards(gpu, mode):
    """test_scale_edges' adversarial three-shard batch (more than 0.5 M rows), its rows naming handles"""
    import dataclasses

    import torch
    w = dataclasses.replace(merge_batch(torch.cuda.get_device_properties(0).multi_processor_count), hash_mode=mode)
    assert w.n >= 500_000
    sf = lib.stack_form(w)
    c = GroupChurn(w, 3, max_frames=len(sf.frames) + 1, max_samples=w.n, chunk_samples=w.n)
    c.register(list(range(len(sf.hashes))))
    cuts = np.array([p1 for _, p1 in w.meta["parts"]][:-1])
    r, r1 = c.flush(np.array(w.hdrs, copy=True), sf.stack_of_row, cuts=cuts)
    assert r.ipc_bytes() == r1.ipc_bytes()
    c.close()


@pytest.mark.gpu
def test_refusals(gpu):
    import ctypes as C
    L = lib.lib()
    for flags in (GRETIRE, REG | GRETIRE, GSTACKS | GRETIRE, GROUP | RETIRE, REG | RETIRE | GRETIRE):
        with pytest.raises(lib.PaError) as e:
            lib.Aggregator(flags=flags)
        assert e.value.code == EINVAL
    w = synth.edge_workload(seed=41, n=300, hash_mode=abi.PA_HASH_XXH64X2, external=False)
    c = GroupChurn(w, 2, max_frames=100_000, max_samples=w.n)
    c.register(list(range(8)))
    c.flush(np.array(w.hdrs[:20], copy=True), [0] * 20)
    with pytest.raises(lib.PaError) as e:  # members retire only with their group
        c.members[0].retire_stacks(1)
    assert e.value.code == EINVAL and "pa_merge_retire_stacks" in str(e.value)
    with pytest.raises(lib.PaError) as e:
        c.g.retire_stacks(0)
    assert e.value.code == EINVAL
    # a staged batch that has not been collected
    for a in c.members:
        c.load(a, w.hdrs[:1], [c.lookup[0]])
        a.stage()
    c.g.process()
    with pytest.raises(lib.PaError) as e:
        c.g.retire_stacks(1)
    assert e.value.code == EINVAL and "collected" in str(e.value)
    c.g.plan()
    c.g.collect()
    assert c.members[0].stack_counters()["stacks_retired"] == 0
    # the refusals retired nothing: stacks 1..7 are still idle and live
    assert [int(x) for x in c.g.retire_stacks(1)] == list(range(1, 8))
    # a member flushed on its own has left the group's lockstep: the next group flush fails on every member
    c.load(c.members[1], w.hdrs[:1], [c.lookup[0]])
    c.members[1].flush()
    for a in c.members:
        c.load(a, w.hdrs[:1], [c.lookup[0]])
    with pytest.raises(lib.PaError) as e:
        c.g.flush()
    assert e.value.code == EINVAL and "left the group" in str(e.value)
    for a in c.members:
        assert b"left the group" in L.pa_agg_last_error(a.h)
    c.close()
    # mixed groups are refused at creation: with plain group-stacks members, ring members and plain retiring aggregators
    form, _ = lib.group_stack_form([w])
    for other in (lambda: lib.from_workload(w, group_form=form), lambda: lib.from_workload(w)):
        members = [lib.from_workload(w, group_form=form, group_retire=True), other()]
        with pytest.raises(lib.PaError) as e:
            lib.MergeGroup.local(members)
        assert e.value.code == EINVAL
        assert b"mixes PA_CFG_GROUP_RETIRE" in L.pa_agg_last_error(members[0].h) or b"mixes PA_CFG_GROUP_STACKS" in L.pa_agg_last_error(members[0].h)
        for a in members:
            a.close()
    retiring = lib.from_workload(w, registered_stacks=True, flags=RETIRE)
    h = C.c_void_p()
    assert L.pa_merge_create_local((C.c_void_p * 1)(retiring.h), 1, C.byref(h)) == EINVAL
    retiring.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world,transport", [(2, "gloo"), (3, "gloo"), (2, "shm"), (3, "shm")])
def test_multi_process_groups(world, transport):
    """one shard per process on this one GPU: a churn sequence with every rank getting the same handles and rank 0's stream equal
    to one retiring aggregator's; then refusals that must reach every rank (a stale handle on the last rank, different idle / cap,
    a mixed group)"""
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", PA_ONE_GPU="1", PA_MERGE_TRANSPORT=transport)
    port = 29741 + world + (10 if transport == "shm" else 0)
    p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
                        "--master-port", str(port), os.path.join(ROOT, "tests", "dist_merge_group_retire_check.py")],
                       capture_output=True, text=True, env=env, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    assert "merge-group-retire ok world=%d transport=%s" % (world, transport) in p.stdout
