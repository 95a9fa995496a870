"""Stack retirement (PA_CFG_RETIRE_STACKS): registered stacks that no batch has named for a while are retired, their slots are
reused under a new generation, and the device frame arena is compacted, so a long-running registry stays bounded. Every batch's
stream must stay byte for byte the ring-mode stream of the same rows (and the oracle's).

CPU tests: a plain-Python model of the contract (idle window, grace batch, slot reuse with generations, cap) on hand-worked
sequences. GPU tests: the library against the model and the oracle through churning intervals, grace, reuse, compaction, a
bounded registry that the plain registered mode cannot keep, provided-id collisions, and the refusals."""
import heapq
import threading

import numpy as np
import pytest

from parca_agent_b200 import abi, lib, synth

EINVAL, ENOSPC = -22, -28
REG, RETIRE = abi.PA_CFG_REGISTERED_STACKS, abi.PA_CFG_RETIRE_STACKS
LIVE, RETIRING, FREE = 0, 1, 2


class Model:
    """The registry as pa_agg_register_stack_handles / pa_agg_retire_stacks / the stages define it. A handle is gen << 32 | slot;
    `last` is the sequence number of the last batch that named the slot, or the stage count when it was registered."""

    def __init__(self, max_frames=None):
        self.state, self.depth, self.gen, self.last = [], [], [], []
        self.free, self.retiring = [], []  # min-heap of free slots; (slot, stage count at which it is freed)
        self.stages, self.frames_live, self.max_frames, self.retired = 0, 0, max_frames, 0

    def register(self, depths):
        """Handles of new stacks, or None (PA_ENOSPC: the live frames would exceed max_frames; nothing is registered)."""
        if self.max_frames is not None and self.frames_live + sum(depths) > self.max_frames:
            return None
        out = []
        for d in depths:
            if self.free:
                s = heapq.heappop(self.free)
            else:
                s = len(self.state)
                self.state.append(FREE); self.depth.append(0); self.gen.append(0); self.last.append(0)
            self.state[s], self.depth[s], self.last[s] = LIVE, d, self.stages
            self.frames_live += d
            out.append(self.gen[s] << 32 | s)
        return out

    def stage(self):
        self.stages += 1
        keep = []
        for s, at in self.retiring:
            if at > self.stages:
                keep.append((s, at))
                continue
            self.state[s] = FREE
            self.gen[s] += 1
            self.frames_live -= self.depth[s]
            heapq.heappush(self.free, s)
        self.retiring = keep

    def valid(self, h):
        s, g = h & 0xFFFFFFFF, h >> 32
        return s < len(self.state) and self.state[s] != FREE and self.gen[s] == g

    def batch(self, handles):
        """The staged batch names `handles`; returns whether its flush succeeds."""
        ok = True
        for h in handles:
            if self.valid(h):
                self.last[h & 0xFFFFFFFF] = self.stages
            else:
                ok = False
        return ok

    def retire(self, idle, cap=None):
        assert idle >= 1
        if self.stages < idle:
            return []
        bound = self.stages - idle
        out = [s for s in range(len(self.state)) if self.state[s] == LIVE and self.last[s] <= bound]
        out = out if cap is None else out[:cap]
        for s in out:
            self.state[s] = RETIRING
            self.retiring.append((s, self.stages + 2))
        self.retired += len(out)
        return [self.gen[s] << 32 | s for s in out]

    def counters(self):
        live = sum(1 for x in self.state if x != FREE)
        return {"stacks_live": live, "stacks_free": len(self.state) - live, "stack_frames_live": self.frames_live,
                "stacks_retired": self.retired}


# ---- CPU: the model on hand-worked sequences ---------------------------------------------------------------------------
def test_model_idle_window_and_grace():
    m = Model()
    assert m.register([2, 3, 4]) == [0, 1, 2]
    assert m.retire(1) == []  # no batch yet: nothing can have been idle for one
    m.stage()
    assert m.batch([0])
    assert m.retire(2) == []  # one batch so far
    assert m.retire(1) == [1, 2]  # registered before batch 1 and not named by it
    assert m.retire(1) == []  # already retiring
    m.stage()  # batch 2 is the grace batch: 1 and 2 still name their stacks
    assert m.batch([1, 2, 0])
    assert m.retire(1) == []  # 0 was named by batch 2
    assert m.retire(2) == []
    m.stage()  # batch 3: 1 and 2 are freed
    assert not m.batch([1])
    assert m.state[1] == FREE and m.gen[1] == 1 and m.free == [1, 2]
    assert m.retire(2) == []  # 0 was named by batch 2
    assert m.retire(1) == [0]  # but not by batch 3, which failed and still counts


def test_model_reuse_with_generations():
    m = Model()
    m.register([1, 1, 1])
    m.stage()
    assert m.retire(1) == [0, 1, 2]
    m.stage()
    assert m.register([5]) == [3]  # no slot is free before the stage after the grace batch
    m.stage()
    assert m.register([7, 8]) == [1 << 32 | 0, 1 << 32 | 1]  # the lowest free slots, next generation
    assert not m.valid(0) and m.valid(1 << 32 | 0) and not m.valid(2 << 32 | 0)
    assert m.counters() == {"stacks_live": 3, "stacks_free": 1, "stack_frames_live": 20, "stacks_retired": 3}
    m.stage()
    m.stage()
    assert m.retire(2) == [1 << 32 | 0, 1 << 32 | 1, 3]  # ascending slot order
    # a stack registered after a batch was staged is not idle for that batch
    m2 = Model()
    m2.stage()
    m2.register([1])
    assert m2.retire(1) == []
    m2.stage()
    assert m2.retire(1) == [0]


def test_model_cap_and_max_frames():
    m = Model(max_frames=10)
    assert m.register([4, 4]) == [0, 1]
    assert m.register([3]) is None  # 11 > 10
    m.stage()
    assert m.retire(1, cap=1) == [0]  # the lowest slot; slot 1 stays live
    assert m.retire(1, cap=5) == [1]  # and a later call finds it
    assert m.register([3]) is None  # frames of stacks in their grace batch still count
    m.stage()
    m.stage()
    assert m.frames_live == 0 and m.register([10]) == [1 << 32 | 0]


# ---- GPU ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    lib.lib()
    return lib


def ring_workload(w, sf, hdrs, stacks):
    """Rows `hdrs` naming the stacks `stacks` of `sf`, as a ring-mode workload (frame ids in the stream)."""
    hd, fr = lib.expand_stack_form(hdrs, lib.StackForm(sf.hashes, sf.frames, sf.offsets, np.asarray(stacks, np.uint64)))
    return synth.Workload(w.name + "[ring]", w.strings, w.frames, w.labelsets, hd, _frame_ids=fr, hash_mode=w.hash_mode,
                          label_flags=w.label_flags, samples_per_second=w.samples_per_second, external_labels=list(w.external_labels),
                          meta=dict(w.meta), schema=w.schema)


def same_record(packed, plain):
    """A PA_IPC_LZ4_FRAME_GPU stream decodes (pyarrow's LZ4) to the same record as the plain stream of the same rows: both,
    written again by pyarrow's own uncompressed writer, give the same bytes (Table.equals can stall on run-end encoded columns)."""
    import pyarrow as pa

    def rewritten(t):
        sink = pa.BufferOutputStream()
        with pa.ipc.new_stream(sink, t.schema) as w:
            w.write_table(t)
        return sink.getvalue().to_pybytes()

    a, b = pa.ipc.open_stream(plain).read_all(), pa.ipc.open_stream(packed).read_all()
    assert a.schema.equals(b.schema, check_metadata=True) and a.num_rows == b.num_rows and rewritten(a) == rewritten(b)


def pack(sf, stacks):
    offs = sf.offsets.astype(np.int64)
    parts = [sf.frames[offs[s]:offs[s + 1]] for s in stacks]
    o = np.zeros(len(stacks) + 1, dtype=np.uint64)
    o[1:] = np.cumsum([len(p) for p in parts])
    fr = np.concatenate(parts).astype(np.uint64) if parts else np.zeros(0, np.uint64)
    return fr, o, sf.hashes[list(stacks)] if len(stacks) else np.zeros((0, 2), np.uint64)


class Churn:
    """One PA_CFG_RETIRE_STACKS aggregator (and its model) fed intervals of rows that name a rotating stack population. The
    caller's lookup (stack -> handle) drops retired handles before the next flush, as a reporter does."""

    def __init__(self, w, max_frames, max_samples, **kw_agg):
        self.w, self.sf = w, lib.stack_form(w)
        self.depth = np.diff(self.sf.offsets.astype(np.int64))
        self.a = lib.from_workload(w.head(0), max_samples=max_samples, max_frames=max_frames, flags=REG | RETIRE, **kw_agg)
        self.m = Model(max_frames)
        self.lookup, self.rng = {}, np.random.Generator(np.random.PCG64(5))

    def register(self, stacks):
        if not len(stacks):
            return
        fr, o, hs = pack(self.sf, stacks)
        h = self.a.register_stack_handles(fr, o, hs if self.w.hash_mode == abi.PA_HASH_PROVIDED else None)
        assert [int(x) for x in h] == self.m.register([int(self.depth[s]) for s in stacks])
        self.lookup.update(zip(stacks, (int(x) for x in h)))

    def rows(self, window, n):
        missing = [s for s in window if s not in self.lookup]
        self.register(missing)
        idx = np.sort(self.rng.choice(self.w.n, n, replace=n > self.w.n))
        stacks = self.rng.choice(window, n)
        hdrs = np.array(self.w.hdrs[idx], copy=True)
        return hdrs, stacks

    def flush(self, hdrs, stacks, during=()):
        """Ingest, then stage; while process + collect run, register `during` (stacks of the next interval)."""
        handles = [self.lookup[int(s)] for s in stacks]
        hv, _, _ = self.a.acquire(len(hdrs), 0)
        hv[:] = hdrs
        hv["frame_off"] = handles
        self.a.commit(len(hdrs))
        self.a.stage()
        self.m.stage()
        assert self.m.batch(handles)
        fresh = [s for s in dict.fromkeys(int(x) for x in during) if s not in self.lookup]
        t = threading.Thread(target=self.register, args=(fresh,))
        t.start()
        try:
            self.a.process()
            r = self.a.collect()
        finally:
            t.join()
        return r

    def retire(self, idle, cap=None):
        got = [int(x) for x in self.a.retire_stacks(idle, cap)]
        assert got == self.m.retire(idle, cap)
        gone = set(got)
        self.lookup = {s: h for s, h in self.lookup.items() if h not in gone}
        return got

    def check_counters(self):
        c = self.a.stack_counters()
        assert {k: c[k] for k in self.m.counters()} == self.m.counters()
        return c


def windows(u, size, step, k):
    return [np.arange(i * step, i * step + size) % u for i in range(k)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [abi.PA_HASH_PROVIDED, abi.PA_HASH_XXH64X2])
@pytest.mark.parametrize("idb", [8, 4])
@pytest.mark.parametrize("out", ["v1", "lz4"])
def test_churn_matches_the_ring_and_the_model(oracle, gpu, mode, idb, out):
    w = synth.ragged(n=20_000, u=3_000, p=8_192, max_depth=90, hash_mode=mode)
    w.schema = abi.PA_SCHEMA_V1 if out == "v1" else abi.PA_SCHEMA_V2
    comp = abi.PA_IPC_LZ4_FRAME_GPU if out == "lz4" else abi.PA_IPC_PLAIN
    kw_agg = dict(frame_id_bytes=idb, ipc_compression=comp, stack_cache_entries=700 if out == "v1" else 0)
    c = Churn(w, max_frames=4_000_000, max_samples=4_000, **kw_agg)
    ring = lib.from_workload(w.head(0), max_samples=4_000, max_frames=4_000 * 128, **kw_agg)
    o = oracle.Oracle(w, stack_cache_entries=700) if out == "v1" else None
    ws = windows(len(c.sf.hashes), 900, 260, 13)
    seen, retired = [], 0
    for k in range(12):
        hdrs, stacks = c.rows(ws[k], 2500 if k != 4 else 3900)
        rw = ring_workload(w, c.sf, hdrs, stacks)
        r = c.flush(hdrs, stacks, during=ws[k + 1][::3])
        lib.load(ring, rw)
        want = ring.flush().ipc_bytes()
        assert r.ipc_bytes() == want, "interval %d differs from the ring mode" % k
        if o is not None:
            o.ingest(rw.hdrs, rw.frame_ids)
            assert o.flush()[0] == want
            ids = [bytes(x) for x in c.a.last_stack_ids(r.n_unique_stacks)]
            seen += [i for i in ids if i not in set(seen)]
            probe = [seen[int(j)] for j in c.rng.choice(len(seen), min(len(seen), 150), replace=False)] + [b"\xee" * 16]
            assert c.a.stacktraces(b"".join(probe)).ipc_bytes() == o.stacktraces(b"".join(probe))[0]
        else:
            same_record(r.ipc_bytes(), oracle.run(rw)[0])
        retired += len(c.retire(1 + k % 3))
        c.check_counters()
    if o is not None:
        for name in ("store_compactions", "store_evictions"):
            assert c.a.kernel_ms(name) == ring.kernel_ms(name)
        o.close()
    assert retired > 1000 and c.a.stack_counters()["stack_compactions"] >= 1
    c.a.close(); ring.close()


def one_batch(c, hdrs, handles):
    hv, _, _ = c.a.acquire(len(hdrs), 0)
    hv[:] = hdrs
    hv["frame_off"] = handles
    c.a.commit(len(hdrs))
    return c.a.flush().ipc_bytes()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [abi.PA_HASH_PROVIDED, abi.PA_HASH_XXH64X2])
def test_grace_batch_then_refusal_then_reuse(oracle, gpu, mode):
    w = synth.edge_workload(seed=21, n=400, hash_mode=mode, external=False)
    c = Churn(w, max_frames=100_000, max_samples=w.n)
    n_st = len(c.sf.hashes)
    c.register(list(range(n_st)))
    hdrs = w.hdrs[:40]
    keep = [0, 1]
    c.flush(hdrs, [keep[i % 2] for i in range(40)])
    gone = c.retire(1)
    assert len(gone) == n_st - 2 and c.a.stack_counters()["stacks_retired"] == n_st - 2
    # the grace batch: rows that still name retired stacks come out exactly right
    old = {s: c.m.gen[s] << 32 | s for s in range(n_st)}
    st = [2 + i % (n_st - 2) for i in range(40)]
    want = oracle.run(ring_workload(w, c.sf, hdrs, st))[0]
    c.m.stage(); c.m.batch([old[s] for s in st])
    assert one_batch(c, hdrs, [old[s] for s in st]) == want
    # one batch later the handles are refused; the next flush is exact
    c.m.stage()
    with pytest.raises(lib.PaError) as e:
        one_batch(c, hdrs, [old[2]] + [old[0]] * 39)
    assert e.value.code == EINVAL and "stack" in str(e.value)
    st = [0, 1] * 20
    c.m.stage(); c.m.batch([old[s] for s in st])
    assert one_batch(c, hdrs, [old[s] for s in st]) == oracle.run(ring_workload(w, c.sf, hdrs, st))[0]
    # reuse: the freed slots go to new stacks with the next generation; their frames, not the old ones, come out
    c.lookup = {0: old[0], 1: old[1]}
    new = [n_st - 1, n_st - 2, 5]  # stacks of the form, registered again into reused slots
    c.register(new)
    assert [c.lookup[s] for s in new] == [1 << 32 | 2, 1 << 32 | 3, 1 << 32 | 4]
    st = [new[i % 3] for i in range(40)]
    c.m.stage(); c.m.batch([c.lookup[s] for s in st])
    assert one_batch(c, hdrs, [c.lookup[s] for s in st]) == oracle.run(ring_workload(w, c.sf, hdrs, st))[0]
    c.m.stage()
    with pytest.raises(lib.PaError) as e:
        one_batch(c, hdrs[:1], [old[2]])  # slot 2 now holds another stack: the old handle is refused
    assert e.value.code == EINVAL
    c.check_counters()
    c.a.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [abi.PA_HASH_PROVIDED, abi.PA_HASH_XXH64X2])
def test_compaction_regrowth_and_a_65535_id_stack(oracle, gpu, mode):
    base = synth.ragged(n=6_000, u=2_000, p=4_096, max_depth=60, hash_mode=mode)
    sf = lib.stack_form(base)
    u0 = len(sf.hashes)
    rng = np.random.Generator(np.random.PCG64(2))
    n_extra, d_extra = 8_000, 60  # stacks no row names, registered while a batch is staged: the arena must regrow before its pass
    deep = rng.integers(0, len(base.frames), 65535).astype(np.uint64)
    extra = rng.integers(0, len(base.frames), n_extra * d_extra).astype(np.uint64)
    hashes = np.vstack([sf.hashes, [[0xDEE9, 0x5]], rng.integers(1, 1 << 62, (n_extra, 2))]).astype(np.uint64)
    offsets = np.concatenate([sf.offsets, sf.offsets[-1] + np.uint64(65535) + np.arange(n_extra + 1, dtype=np.uint64) * np.uint64(d_extra)])
    sf = lib.StackForm(hashes, np.concatenate([sf.frames, deep, extra]), offsets, sf.stack_of_row)
    c = Churn(base, max_frames=2_000_000, max_samples=3_000)
    c.sf, c.depth = sf, np.diff(sf.offsets.astype(np.int64))
    ws = windows(u0, 300, 300, 14)  # disjoint windows: each interval retires the last one's stacks
    c.register(list(ws[0]))
    c.register([u0])  # the deep stack goes after them: every compaction moves it to a new, non-zero offset
    assert c.lookup[u0] == 300
    grew = False
    for k, win in enumerate(ws):
        hdrs, stacks = c.rows(win, 1500)
        stacks[::50] = u0
        if k == 7:  # regrowth while a batch is staged: the pass must read the moved arena
            handles = [c.lookup[int(s)] for s in stacks]
            hv, _, _ = c.a.acquire(len(hdrs), 0)
            hv[:] = hdrs
            hv["frame_off"] = handles
            c.a.commit(len(hdrs))
            c.a.stage(); c.m.stage(); c.m.batch(handles)
            n0 = c.a.stack_counters()["stack_compactions"]
            c.register(list(range(u0 + 1, u0 + 1 + n_extra)))
            c.a.process()
            r = c.a.collect()
            grew = c.a.stack_counters()["stack_compactions"] > n0
        else:
            r = c.flush(hdrs, stacks)
        assert r.ipc_bytes() == oracle.run(ring_workload(base, sf, hdrs, stacks))[0], "interval %d" % k
        c.retire(1)
        cnt = c.check_counters()
    assert grew and cnt["stack_compactions"] >= 2 and cnt["stack_frames_live"] == c.m.frames_live
    ms, launches = c.a.kernel_ms("stack_compact")
    assert ms > 0 and launches == 4
    c.a.close()


@pytest.mark.gpu
def test_bounded_registry_never_runs_out(oracle, gpu):
    """max_frames just above the working set plus the grace batch: 50 churn intervals with reporter-style re-registration (every
    fifth interval the lookup is cleared, as ReportExecutable clears the stack cache) never hit PA_ENOSPC; a plain registered
    aggregator fed the same registrations does."""
    w = synth.config2(n=20_000, u=4_000, p=8_192, hash_mode=abi.PA_HASH_XXH64X2)
    sf = lib.stack_form(w)
    size, step = 400, 100
    max_frames = 64 * (2 * size + 2 * step) + 64 * size  # working set, stacks still in grace, duplicates of a cleared lookup
    c = Churn(w, max_frames=max_frames, max_samples=2_000)
    plain = lib.from_workload(w.head(0), max_samples=2_000, max_frames=max_frames, flags=REG)
    plain_enospc = None
    for k, win in enumerate(windows(len(sf.hashes), size, step, 50)):
        if k % 5 == 4:
            c.lookup = {}  # the duplicates registered now leave the old copies idle: they are retired
        before = set(c.lookup)
        hdrs, stacks = c.rows(win, 1500)
        fresh = [s for s in win if s not in before]
        if plain_enospc is None and fresh:
            fr, o, _ = pack(sf, fresh)
            try:
                plain.register_stacks(fr, o)
            except lib.PaError as e:
                assert e.code == ENOSPC
                plain_enospc = k
        r = c.flush(hdrs, stacks)
        if k % 10 == 0:
            assert r.ipc_bytes() == oracle.run(ring_workload(w, sf, hdrs, stacks))[0]
        c.retire(1)
        assert c.check_counters()["stack_frames_live"] <= max_frames
    assert plain_enospc is not None and plain_enospc < 50
    c.a.close(); plain.close()


@pytest.mark.gpu
def test_provided_id_collisions_first_occurrence_wins(oracle, gpu):
    """Two slots share a provided id (different frames); one is retired while rows still name the other."""
    base = synth.edge_workload(seed=14, n=60, hash_mode=abi.PA_HASH_PROVIDED, external=False)
    A, B, C = [1, 2, 3], [4, 5], [6, 7, 8, 9]
    frames = np.asarray(A + B + C, np.uint64)
    sf = lib.StackForm(np.asarray([(0x11, 0x22), (0x11, 0x22), (0, 0)], np.uint64), frames, np.asarray([0, 3, 5, 9], np.uint64), None)
    c = Churn(base, max_frames=1_000, max_samples=base.n)
    c.sf, c.depth = sf, np.diff(sf.offsets.astype(np.int64))
    c.register([0, 1, 2])
    hdrs = base.hdrs[:30]
    st = [0, 1, 2] * 10
    assert c.flush(hdrs, st).ipc_bytes() == oracle.run(ring_workload(base, sf, hdrs, st))[0]
    st = [1, 2] * 15
    assert c.flush(hdrs, st).ipc_bytes() == oracle.run(ring_workload(base, sf, hdrs, st))[0]
    h_a = c.lookup[0]
    assert c.retire(1) == [h_a]  # A is idle; B, which shares its id, is not
    c.lookup[0] = h_a  # rows committed before the handle was dropped
    st = [0, 1, 2, 1] * 7 + [0, 1]  # the grace batch names both: A's frames win as the first occurrence
    assert c.flush(hdrs, st).ipc_bytes() == oracle.run(ring_workload(base, sf, hdrs, st))[0]
    del c.lookup[0]
    st = [1, 2] * 15
    assert c.flush(hdrs, st).ipc_bytes() == oracle.run(ring_workload(base, sf, hdrs, st))[0]
    c.a.close()


@pytest.mark.gpu
def test_cap_and_refusals(gpu):
    import ctypes as C
    w = synth.edge_workload(seed=2, n=200)
    c = Churn(w, max_frames=100_000, max_samples=w.n)
    n_st = len(c.sf.hashes)
    c.register(list(range(n_st)))
    c.flush(w.hdrs[:10], [0] * 10)
    assert c.retire(1, cap=3) == [1, 2, 3]  # slot 0 was named
    assert c.retire(1, cap=0) == []
    assert len(c.retire(1)) == n_st - 4  # the rest, found by a later call
    with pytest.raises(lib.PaError) as e:
        c.a.retire_stacks(0)
    assert e.value.code == EINVAL
    hv, _, _ = c.a.acquire(1, 0)
    hv[:] = w.hdrs[:1]
    hv["frame_off"] = [0]
    c.a.commit(1)
    c.a.stage()
    with pytest.raises(lib.PaError) as e:
        c.a.retire_stacks(1)  # a staged batch has not been collected
    assert e.value.code == EINVAL
    c.a.process()
    c.a.collect()
    with pytest.raises(lib.PaError) as e:
        c.a.register_stacks([0], [0, 1], np.zeros((1, 2), np.uint64))
    assert e.value.code == EINVAL
    plain = lib.from_workload(w, registered_stacks=True, max_frames=100_000)
    with pytest.raises(lib.PaError) as e:
        plain.retire_stacks(1, cap=4)
    assert e.value.code == EINVAL
    assert list(plain.register_stack_handles([0, 1], [0, 1, 2], np.zeros((2, 2), np.uint64))) == [n_st, n_st + 1]
    for flags in (RETIRE, RETIRE | abi.PA_CFG_GROUP_STACKS | REG, RETIRE | abi.PA_CFG_GROUP_STACKS):
        with pytest.raises(lib.PaError) as e:
            lib.Aggregator(flags=flags)
        assert e.value.code == EINVAL
    for name in ("stacks_live", "stack_compact"):  # the registry's counters exist on retiring aggregators only
        with pytest.raises(lib.PaError) as e:
            plain.kernel_ms(name)
        assert e.value.code == EINVAL
    L, h = lib.lib(), C.c_void_p()
    assert L.pa_merge_create_local((C.c_void_p * 2)(c.a.h, plain.h), 2, C.byref(h)) == EINVAL
    assert L.pa_merge_create_host(c.a.h, None, 0, 2, C.byref(h)) == EINVAL
    c.a.close(); plain.close()
