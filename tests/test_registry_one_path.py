"""Every PA_CFG_REGISTERED_STACKS aggregator keeps its stacks in one slot registry. One that cannot retire never frees a slot,
so each new stack takes the next slot with generation 0 and its handle is its consecutive id. These tests pin what that
relies on: a plain registered aggregator and a PA_CFG_RETIRE_STACKS one that never retires hand out the same handles and
return the same streams, and PA_CFG_GROUP_STACKS groups, which send handles in their v1 store exchange, still give one
registered aggregator's stream."""
import threading

import numpy as np
import pytest

from parca_agent_b200 import abi, lib, synth

V1, V2 = abi.PA_SCHEMA_V1, abi.PA_SCHEMA_V2
PROVIDED = abi.PA_HASH_PROVIDED


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    lib.lib()
    return lib


def random_stacks(rng, w, n, max_depth):
    """n stacks that no row names: (frames, offsets, hashes or None)"""
    d = rng.integers(0, max_depth + 1, n)
    off = np.zeros(n + 1, dtype=np.uint64)
    off[1:] = np.cumsum(d)
    fr = rng.integers(0, len(w.frames), int(off[-1])).astype(np.uint64)
    return fr, off, rng.integers(1, 1 << 62, (n, 2)).astype(np.uint64) if w.hash_mode == PROVIDED else None


def chunk(w, sf, s0, s1):
    """stacks [s0, s1) of a StackForm as one registration call takes them"""
    o = sf.offsets
    return sf.frames[int(o[s0]):int(o[s1])], o[s0:s1 + 1] - o[s0], sf.hashes[s0:s1] if w.hash_mode == PROVIDED else None


@pytest.mark.gpu
@pytest.mark.parametrize("schema", [V2, V1])
@pytest.mark.parametrize("idb", [4, 8])
@pytest.mark.parametrize("mode", [PROVIDED, abi.PA_HASH_XXH64X2])
def test_plain_registry_is_a_registry_that_never_retires(oracle, gpu, schema, idb, mode):
    """The same registrations on both: each interval's stacks between intervals, a second thread's stacks during each flush,
    and one burst that outgrows the arena. Handles, ids and streams agree, and every stream is the oracle's."""
    w = synth.edge_workload(seed=71, n=4000, hash_mode=mode, external=False)
    w.schema = schema
    sf = lib.stack_form(w)
    n_st = len(sf.hashes)
    opts = dict(max_samples=w.n, max_frames=4_000_000, frame_id_bytes=idb)
    plain = lib.from_workload(w.head(0), registered_stacks=True, **opts)
    retiring = lib.from_workload(w.head(0), registered_stacks=True, flags=abi.PA_CFG_RETIRE_STACKS, **opts)
    o = oracle.Oracle(w)
    rng = np.random.Generator(np.random.PCG64(idb + 2 * mode))
    ids = np.zeros(n_st, dtype=np.uint64)

    def flush_while_registering(a, batches, out, errors):
        """flushes `a` while a second thread registers `batches`; the thread's handles go to `out`"""
        def registrar():
            try:
                for fr, off, hs in batches:
                    out.append(a.register_stack_handles(fr, off, hs))
            except Exception as e:  # noqa: BLE001
                errors.append(repr(e))
        t = threading.Thread(target=registrar)
        t.start()
        try:
            return a.flush().ipc_bytes()
        finally:
            t.join()

    for k in range(8):
        lo, hi = (k * n_st) // 8, ((k + 1) * n_st) // 8
        if k == 4:  # a burst several times the arena
            fr, off, hs = random_stacks(rng, w, 100_000, 8)
            first = plain.register_stacks(fr, off, hs)
            assert np.array_equal(retiring.register_stack_handles(fr, off, hs), first + np.arange(100_000, dtype=np.uint64))
        fr, off, hs = chunk(w, sf, lo, hi)
        first = plain.register_stacks(fr, off, hs)
        h = retiring.register_stack_handles(fr, off, hs)
        assert np.array_equal(h, first + np.arange(hi - lo, dtype=np.uint64))
        ids[lo:hi] = h
        mine = np.nonzero(sf.stack_of_row < hi)[0]
        part = w.rows(mine)
        o.ingest(part.hdrs, part.frame_ids)
        want, _ = o.flush()
        batches = [random_stacks(rng, w, 64, 11) for _ in range(300)]
        got, thread_handles = [], []
        for a in (plain, retiring):
            lib.load(a, part, stack_of_row=ids[sf.stack_of_row[mine].astype(np.int64)])
            handles, errors = [], []
            got.append(flush_while_registering(a, batches, handles, errors))
            assert not errors, errors
            thread_handles.append(np.concatenate(handles))
        assert got[0] == got[1] == want, "interval %d" % k
        assert np.array_equal(thread_handles[0], thread_handles[1])
        assert np.array_equal(thread_handles[0], thread_handles[0][0] + np.arange(300 * 64, dtype=np.uint64))
    c = retiring.stack_counters()
    assert c["stacks_free"] == 0 and c["stack_frames_dead"] == 0 and c["stacks_retired"] == 0
    assert c["stack_compactions"] >= 3  # every regrow of a non-empty arena is one
    assert c["stacks_live"] == int(plain.register_stacks([], [0]))
    plain.close(); retiring.close(); o.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_group_stacks_send_handles_across_an_arena_regrow(oracle, gpu, world):
    """v1 PA_CFG_GROUP_STACKS groups: every interval, member 0 registers new stacks (and enough unnamed ones to regrow the
    arena at the next upload) before its stage, the other members between their stage and pa_merge_process. The stream is one
    registered aggregator's for the concatenated rows, and the store exchange sends one handle per stack the store lacked."""
    w = synth.config2(n=9000, u=2500, p=4096)
    w.schema = V1
    form, _ = gpu.group_stack_form([w])
    n_st = len(form.hashes)
    cap = 1500
    opts = dict(max_samples=w.n, max_frames=2_000_000, stack_cache_entries=cap)
    k0 = 400
    init = gpu.StackForm(form.hashes[:k0], form.frames[:int(form.offsets[k0])], form.offsets[:k0 + 1], None)
    members = [gpu.from_workload(w, group_form=init, **opts) for _ in range(world)]
    g = gpu.MergeGroup.local(members)
    single = gpu.from_workload(w.head(0), registered_stacks=True, **opts)
    base = single.register_stacks(*chunk(w, form, 0, k0))  # (the members' stack i is the single aggregator's base + i)
    o = oracle.Oracle(w, stack_cache_entries=cap)
    rng = np.random.Generator(np.random.PCG64(world))
    ids = np.full(n_st, -1, dtype=np.int64)
    ids[:k0] = np.arange(k0)
    seen = set()
    before = int(form.offsets[k0])  # frames registered on every member
    for k in range(4):
        s0, s1 = k0 + 150 * k, k0 + 150 * (k + 1)
        # More pending frames than registered ones: the arena holds at most twice the frames registered at its last grow, so
        # the next upload regrows it (on member 0 at its stage, on the others at pa_merge_process).
        nf = before // 4000 + 1
        filler = (rng.integers(0, len(w.frames), nf * 4000).astype(np.uint64), np.arange(nf + 1, dtype=np.uint64) * np.uint64(4000),
                  rng.integers(1, 1 << 62, (nf, 2)).astype(np.uint64) if w.hash_mode == PROVIDED else None)
        new = chunk(w, form, s0, s1)
        assert nf * 4000 > before
        before += nf * 4000 + int(new[1][-1])
        first = single.register_stacks(*filler) - base
        assert single.register_stacks(*new) == base + first + nf
        ids[s0:s1] = first + nf + np.arange(s1 - s0)
        named = np.nonzero(ids[form.stack_of_row.astype(np.int64)] >= 0)[0]
        rows = np.sort(rng.choice(named, 600, replace=False))
        idx = np.array_split(rows, np.sort(rng.choice(len(rows) + 1, world - 1)))
        sor = [ids[form.stack_of_row[ix].astype(np.int64)].astype(np.uint64) for ix in idx]

        def register(a):
            assert int(a.register_stack_handles(*filler)[0]) == first
            assert int(a.register_stack_handles(*new)[0]) == first + nf
        register(members[0])
        for a, ix, s in zip(members, idx, sor):
            gpu.load(a, w.rows(ix), stack_of_row=s)
            a.stage()
        for a in members[1:]:
            register(a)
        g.process()
        g.plan()
        got = g.collect().ipc_bytes()
        ref = w.rows(rows)
        gpu.load(single, ref, stack_of_row=np.concatenate(sor) + np.uint64(base))
        r1 = single.flush()
        o.ingest(ref.hdrs, ref.frame_ids)
        want, _ = o.flush()
        assert got == r1.ipc_bytes() == want, "interval %d" % k
        uniq = [bytes(x) for x in single.last_stack_ids(r1.n_unique_stacks)]
        lacked = [u for u in uniq if u not in seen]
        seen.update(uniq)
        assert sum(a.kernel_ms("store_refs")[1] for a in members) == len(lacked) > 0
        assert [a.kernel_ms("store_frames")[1] for a in members] == [0] * world
    assert single.kernel_ms("store_evictions")[1] == 0  # (so the store lacked exactly the stacks not seen before)
    assert min(int(form.offsets[s + 1] - form.offsets[s]) for s in range(n_st)) > 0  # (and every one of them crosses)
    g.close()
    for a in members + [single]:
        a.close()
    o.close()
