"""Registered stacks (PA_CFG_REGISTERED_STACKS): stacks are registered once and every sample row names its stack in frame_off,
so the ring holds 64-byte headers only. Every record must be byte for byte the one the ring-mode aggregator builds from the
same rows expanded to frame ids, and the oracle's. CPU tests: the expansion helper and the C++ reporter's registered mode."""
import hashlib
import os
import subprocess
import threading

import numpy as np
import pytest

import kat_workloads as kw
from parca_agent_b200 import abi, lib, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EINVAL, ENOSPC, ERANGE = -22, -28, -34


def ring_form(w):
    """The workload's rows expanded from its registered-stacks form back to frame ids (an explicit-stream workload)."""
    hd, fr = lib.expand_stack_form(w.hdrs, lib.stack_form(w))
    return synth.Workload(w.name + "[ring]", w.strings, w.frames, w.labelsets, hd, _frame_ids=fr, hash_mode=w.hash_mode,
                          label_flags=w.label_flags, samples_per_second=w.samples_per_second, external_labels=list(w.external_labels),
                          meta=dict(w.meta), schema=w.schema)


def from_stack_form(w, sf):
    """A workload whose rows are given in registered-stacks form (sf.stack_of_row), in ring form."""
    hd, fr = lib.expand_stack_form(w.hdrs[:len(sf.stack_of_row)], sf)
    return synth.Workload(w.name + "[sf]", w.strings, w.frames, w.labelsets, hd, _frame_ids=fr, hash_mode=w.hash_mode,
                          label_flags=w.label_flags, samples_per_second=w.samples_per_second, external_labels=list(w.external_labels),
                          meta=dict(w.meta), schema=w.schema)


# ---- CPU ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("make", [
    synth.config1, lambda: synth.config1(hash_mode=abi.PA_HASH_PROVIDED).head(3000), lambda: synth.config2(n=20_000, u=2_000, p=4_096),
    lambda: synth.config3(n=20_000, u=3_000, p=4_096, npids=50, lsets=3), lambda: synth.ragged(n=20_000, u=2_000),
    lambda: synth.edge_workload(seed=3), lambda: synth.edge_workload(seed=4, hash_mode=abi.PA_HASH_XXH64X2),
    lambda: synth.config1().rows(np.arange(2999, -1, -3)), lambda: synth.edge_workload(seed=5, n=300).rows(np.arange(299, -1, -1)),
    kw.stack_dedup, kw.writer_basic, kw.multiple_frame_types, kw.func_dedup_in_stack, kw.null_lines])
def test_stack_form_expands_to_the_workload(make):
    w = make()
    sf = lib.stack_form(w)
    assert len(sf.offsets) == len(sf.hashes) + 1 and len(sf.stack_of_row) == w.n
    assert int(sf.stack_of_row.max(initial=0)) < max(1, len(sf.hashes))
    hd, fr = lib.expand_stack_form(w.hdrs, sf)
    assert hd.tobytes() == w.hdrs.tobytes()
    assert fr.dtype == np.uint64 and np.array_equal(fr, w.frame_ids)


def test_stack_form_registers_each_distinct_stack_once():
    w = synth.edge_workload(seed=6, n=2000)
    sf = lib.stack_form(w)
    keys = {(int(h[0]), int(h[1]), sf.frames[int(a):int(b)].tobytes()) for h, a, b in zip(sf.hashes, sf.offsets[:-1], sf.offsets[1:])}
    assert len(keys) == len(sf.hashes) <= 40  # the workload draws from a pool of 40 stacks
    w = synth.config1()
    assert len(lib.stack_form(w).hashes) == w.meta["U"]  # the stack table itself


def build_bin(name):
    exe = os.path.join(ROOT, "tests", "cpp", "_build", name)
    src = os.path.join(ROOT, "tests", "cpp", name + ".cpp")
    so = os.path.join(ROOT, "parca_agent_b200", "libparcaagg.so")
    os.makedirs(os.path.dirname(exe), exist_ok=True)
    if not os.path.exists(exe) or os.path.getmtime(exe) < max(os.path.getmtime(src), os.path.getmtime(so)):
        subprocess.run(["g++", "-O1", "-std=c++17", "-o", exe, src, "-L" + os.path.join(ROOT, "parca_agent_b200"), "-lparcaagg",
                        "-Wl,-rpath," + os.path.join(ROOT, "parca_agent_b200"), "-lpthread"], check=True)
    return exe


def test_reporter_registers_stacks():
    out = subprocess.run([build_bin("test_reporter_stacks")], capture_output=True, text=True)
    assert out.returncode == 0, out.stderr
    assert out.stdout.strip() == "ok"


# ---- GPU ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    lib.lib()
    return lib


def check(oracle, w, **kw_run):
    """Registered-mode stream == ring-mode stream on the expanded rows == the oracle's; returns the registered Result."""
    wr = ring_form(w)
    want, st = oracle.run(wr)
    ring, _ = lib.run(wr, **kw_run)
    got, r = lib.run(w, registered_stacks=True, **kw_run)
    assert ring == want, "ring mode differs from the oracle"
    assert got == ring, "registered stacks differ from the ring (len %d vs %d)" % (len(got), len(ring))
    assert r.n_rows == st["rows"] and r.n_unique_stacks == st["unique_stacks"]
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["stack_dedup", "writer_basic", "multiple_frame_types", "func_dedup_in_stack", "null_lines"])
def test_reference_unit_test_inputs(oracle, gpu, name):
    check(oracle, getattr(kw, name)())


@pytest.mark.gpu
@pytest.mark.parametrize("seed", [1, 2, 3, 4])
@pytest.mark.parametrize("mode", [abi.PA_HASH_PROVIDED, abi.PA_HASH_XXH64X2])
@pytest.mark.parametrize("external", [False, True])
def test_edge_batches(oracle, gpu, seed, mode, external):
    check(oracle, synth.edge_workload(seed=seed, hash_mode=mode, external=external))


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [1, 2, 4, 7, 3])
def test_edge_label_flags(oracle, gpu, flags):
    check(oracle, synth.edge_workload(seed=11, label_flags=flags, external=True))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [abi.PA_HASH_PROVIDED, abi.PA_HASH_XXH64X2])
def test_config1_full(oracle, gpu, mode):
    r = check(oracle, synth.config1(hash_mode=mode))
    assert r.n_unique_stacks == 1000


@pytest.mark.gpu
def test_config2_and_config3_scaled(oracle, gpu):
    check(oracle, synth.config2(n=400_000, u=20_000, p=32_768), chunk_samples=65536)
    check(oracle, synth.config3(n=300_000, u=30_000, p=16_384, npids=500, lsets=10))
    check(oracle, synth.config2(n=200_000, u=10_000, p=16_384, hash_mode=abi.PA_HASH_PROVIDED))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [abi.PA_HASH_XXH64X2, abi.PA_HASH_PROVIDED])
def test_config2_full_matches_the_ring(gpu, mode):
    """Config 2 at its full size (10M rows x 64 frames, 100k stacks): the same stream as the ring mode."""
    w = synth.config2(hash_mode=mode)
    ring, _ = lib.run(w, chunk_samples=1 << 20)
    want = hashlib.sha256(ring).hexdigest()
    del ring
    got, r = lib.run(w, chunk_samples=1 << 20, registered_stacks=True)
    assert r.n_rows == 10_000_000 and r.n_unique_stacks == 100_000
    assert hashlib.sha256(got).hexdigest() == want


def with_empty_stacks(w, every=7):
    """The workload with every `every`-th stack of its registered form emptied (depth 0)."""
    sf = lib.stack_form(w)
    depth = np.diff(sf.offsets.astype(np.int64))
    depth[::every] = 0
    offsets = np.zeros(len(depth) + 1, dtype=np.uint64)
    offsets[1:] = np.cumsum(depth)
    frames = np.concatenate([sf.frames[int(a):int(a) + int(d)] for a, d in zip(sf.offsets[:-1], depth)])
    return from_stack_form(w, lib.StackForm(sf.hashes, frames, offsets, sf.stack_of_row))


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [abi.PA_HASH_PROVIDED, abi.PA_HASH_XXH64X2])
def test_ragged_depths_and_the_deepest_stack(oracle, gpu, mode):
    w = with_empty_stacks(synth.ragged(n=200_000, u=6_000, max_depth=127, hash_mode=mode))  # depths 0..127
    assert int(w.hdrs["nframes"].min()) == 0 and int(w.hdrs["nframes"].max()) == 127
    check(oracle, w)
    base = synth.edge_workload(seed=8, n=60, hash_mode=mode)
    sf = lib.stack_form(base)
    deep = np.random.Generator(np.random.PCG64(1)).integers(0, len(base.frames), 65535).astype(np.uint64)
    rows = sf.stack_of_row.copy()
    rows[[5, 33, 59]] = len(sf.hashes)
    sf = lib.StackForm(np.vstack([sf.hashes, [[0xABCD, 0x1234]]]).astype(np.uint64), np.concatenate([sf.frames, deep]),
                       np.append(sf.offsets, sf.offsets[-1] + np.uint64(65535)), rows)
    w = from_stack_form(base, sf)
    assert int(w.hdrs["nframes"].max()) == 65535
    check(oracle, w)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [abi.PA_HASH_PROVIDED, abi.PA_HASH_XXH64X2])
def test_narrow_ids_small_chunks_and_single_ring(oracle, gpu, mode):
    for w in (synth.edge_workload(seed=51, n=6000, hash_mode=mode), synth.config1(hash_mode=mode).head(50_000)):
        check(oracle, w, frame_id_bytes=4)
        check(oracle, w, frame_id_bytes=4, chunk_samples=777)
        check(oracle, w, chunk_samples=777)
        check(oracle, w, flags=abi.PA_CFG_SINGLE_RING)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [abi.PA_HASH_PROVIDED, abi.PA_HASH_XXH64X2])
def test_lz4_frame_gpu(gpu, mode):
    for w in (synth.edge_workload(seed=12, n=5000, hash_mode=mode), synth.config1(hash_mode=mode)):
        for v1 in (False, True):
            w.schema = abi.PA_SCHEMA_V1 if v1 else abi.PA_SCHEMA_V2
            wr = ring_form(w)
            ring, _ = lib.run(wr, ipc_compression=abi.PA_IPC_LZ4_FRAME_GPU)
            got, _ = lib.run(w, registered_stacks=True, ipc_compression=abi.PA_IPC_LZ4_FRAME_GPU)
            assert got == ring


def missing_ids(k):
    return [bytes([0xEE, i]) * 8 for i in range(k)]


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [abi.PA_HASH_PROVIDED, abi.PA_HASH_XXH64X2])
def test_v1_intervals_with_a_small_store(oracle, gpu, mode):
    """v1: sample records, pa_agg_last_stack_ids, pa_agg_stacktraces and the store counters over many intervals against a
    small store, registered vs a ring-mode v1 aggregator driven identically (and the sample records vs the oracle)."""
    w = synth.config2(n=9000, u=2500, p=4096, hash_mode=mode)
    w.schema = abi.PA_SCHEMA_V1
    kw_agg = dict(max_samples=4000, max_frames=400_000, stack_cache_entries=300)
    ring = lib.from_workload(w.head(0), **kw_agg)
    reg = lib.from_workload(w, registered_stacks=True, **kw_agg)  # registers the whole stack table up front
    o = oracle.Oracle(w, stack_cache_entries=300)
    rng = np.random.Generator(np.random.PCG64(9))
    seen = []
    for k in range(14):
        part = w.rows(np.sort(rng.choice(w.n, 900 if k == 5 else 220, replace=False)))
        o.ingest(part.hdrs, part.frame_ids)
        want, _ = o.flush()
        lib.load(ring, part)
        lib.load(reg, part, stack_of_row=part.stack_choice)
        a, b = ring.flush(), reg.flush()
        assert a.ipc_bytes() == want and b.ipc_bytes() == want
        ids = [bytes(x) for x in reg.last_stack_ids(b.n_unique_stacks)]
        assert ids == [bytes(x) for x in ring.last_stack_ids(a.n_unique_stacks)]
        seen += [i for i in ids if i not in set(seen)]
        probe = [seen[int(j)] for j in rng.choice(len(seen), min(len(seen), 100), replace=False)] + missing_ids(1)
        assert reg.stacktraces(b"".join(probe)).ipc_bytes() == ring.stacktraces(b"".join(probe)).ipc_bytes()
    assert reg.stacktraces(b"".join(seen)).ipc_bytes() == ring.stacktraces(b"".join(seen)).ipc_bytes()
    for name in ("store_compactions", "store_evictions"):
        assert reg.kernel_ms(name) == ring.kernel_ms(name)
    assert ring.kernel_ms("store_evictions")[1] >= 5
    ring.close(); reg.close(); o.close()


def collision_workload(order):
    """Provided ids: stacks A and B share one id with different frames, C and D share the all-zero id. `order` is the row
    order of the first occurrences; the registration order is the reverse of the first occurrences in half the cases."""
    base = synth.edge_workload(seed=14, n=40, hash_mode=abi.PA_HASH_PROVIDED)
    A, B, C, D = [1, 2, 3], [4, 5], [6, 7, 8, 9], [10]
    stacks = {"A": A, "B": B, "C": C, "D": D}
    ids = {"A": (0x1111, 0x2222), "B": (0x1111, 0x2222), "C": (0, 0), "D": (0, 0)}
    names = list(order)
    frames = np.concatenate([np.asarray(stacks[n], np.uint64) for n in names])
    offsets = np.zeros(len(names) + 1, dtype=np.uint64)
    offsets[1:] = np.cumsum([len(stacks[n]) for n in names])
    hashes = np.asarray([ids[n] for n in names], dtype=np.uint64)
    rows = np.asarray([k % len(names) for k in range(base.n)], dtype=np.uint64)
    return base, lib.StackForm(hashes, frames, offsets, rows)


def run_registered(w, sf, register_order=None, **kw_agg):
    """One flush of rows given in registered form, the stacks registered explicitly (in register_order, default as given)."""
    a = lib.from_workload(w.head(0), registered_stacks=True, max_samples=max(1, len(sf.stack_of_row)), max_frames=len(sf.frames) + 1, **kw_agg)
    n = len(sf.hashes)
    order = list(range(n)) if register_order is None else list(register_order)
    remap = np.zeros(n, dtype=np.uint64)
    for pos, s in enumerate(order):
        lo, hi = int(sf.offsets[s]), int(sf.offsets[s + 1])
        first = a.register_stacks(sf.frames[lo:hi], [0, hi - lo], sf.hashes[s:s + 1] if w.hash_mode == abi.PA_HASH_PROVIDED else None)
        assert first == pos
        remap[s] = pos
    hv, _, _ = a.acquire(len(sf.stack_of_row), 0)
    hv[:] = w.hdrs[:len(sf.stack_of_row)]
    hv["frame_off"] = remap[sf.stack_of_row.astype(np.int64)]
    a.commit(len(sf.stack_of_row))
    out = a.flush().ipc_bytes()
    a.close()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("order", ["ABCD", "BADC"])
def test_provided_id_collisions_first_occurrence_wins(oracle, gpu, order):
    base, sf = collision_workload(order)
    wr = from_stack_form(base, sf)
    want, _ = oracle.run(wr)
    assert lib.run(wr)[0] == want
    assert run_registered(base, sf) == want
    assert run_registered(base, sf, register_order=range(len(sf.hashes) - 1, -1, -1)) == want
    v1 = from_stack_form(base, sf)
    v1.schema = abi.PA_SCHEMA_V1
    base.schema = abi.PA_SCHEMA_V1
    assert run_registered(base, sf) == oracle.run(v1)[0]


@pytest.mark.gpu
def test_stack_ids_equal_the_ring_xxh64_ids(gpu):
    """The library's registration hash (host) against the hash kernel (device) on the same rows."""
    w = synth.ragged(n=30_000, u=3_000, hash_mode=abi.PA_HASH_XXH64X2)
    w = with_empty_stacks(w, every=11)
    out = []
    for registered in (False, True):
        a = lib.from_workload(w if registered else ring_form(w), registered_stacks=registered)
        lib.load(a, w if registered else ring_form(w))
        a.stage()
        a.process()
        out.append(a.debug_stack_ids(w.n).copy())
        if registered:
            assert a.kernel_ms("hash")[1] == 0  # no hash kernel: the ids come from the registered records
        a.collect()
        a.close()
    assert np.array_equal(out[0], out[1])


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [abi.PA_HASH_PROVIDED, abi.PA_HASH_XXH64X2])
def test_registration_between_intervals_and_during_flushes(oracle, gpu, mode):
    """Stacks registered between intervals are used by the next; a second thread keeps registering (stacks no row names)
    while the flushes run, which also regrows the device mirrors many times over."""
    w = synth.edge_workload(seed=61, n=4000, hash_mode=mode, external=False)
    sf = lib.stack_form(w)
    n_st = len(sf.hashes)
    a = lib.from_workload(w.head(0), registered_stacks=True, max_samples=w.n, max_frames=8_000_000)
    stop, errors = threading.Event(), []

    def registrar():
        rng = np.random.Generator(np.random.PCG64(3))
        try:
            for _ in range(5000):  # at most ~1.8M frames: max_frames is never reached
                if stop.is_set():
                    break
                d = rng.integers(0, 12, 64)
                off = np.zeros(65, dtype=np.uint64)
                off[1:] = np.cumsum(d)
                fr = rng.integers(0, len(w.frames), int(off[-1])).astype(np.uint64)
                a.register_stacks(fr, off, rng.integers(1, 1 << 62, (64, 2)).astype(np.uint64) if mode == abi.PA_HASH_PROVIDED else None)
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))

    first_ids = {}
    t = threading.Thread(target=registrar)
    t.start()
    try:
        for k in range(12):
            lo, hi = (k * n_st) // 12, ((k + 1) * n_st) // 12
            if k == 6:  # far more stacks than the device mirrors hold: they are regrown before the next pass
                d = np.arange(50_000) % 9
                off = np.zeros(len(d) + 1, dtype=np.uint64)
                off[1:] = np.cumsum(d)
                a.register_stacks(np.arange(int(off[-1])) % len(w.frames), off,
                                  np.ones((len(d), 2), np.uint64) if mode == abi.PA_HASH_PROVIDED else None)
            for s in range(lo, hi):  # this interval's new stacks, interleaved with the other thread's registrations
                a0, a1 = int(sf.offsets[s]), int(sf.offsets[s + 1])
                first_ids[s] = a.register_stacks(sf.frames[a0:a1], [0, a1 - a0], sf.hashes[s:s + 1] if mode == abi.PA_HASH_PROVIDED else None)
            mine = np.nonzero(sf.stack_of_row < hi)[0]
            part = w.rows(mine)
            want, _ = oracle.run(part)
            hv, _, _ = a.acquire(part.n, 0)
            hv[:] = part.hdrs
            hv["frame_off"] = [first_ids[int(s)] for s in sf.stack_of_row[mine]]
            a.commit(part.n)
            assert a.flush().ipc_bytes() == want
    finally:
        stop.set()
        t.join()
    a.close()
    assert not errors, errors
    assert max(first_ids.values()) > 50_000 + n_st


def registered_agg(w=None, **kw_agg):
    w = w or synth.edge_workload(seed=2, n=200)
    return w, lib.from_workload(w, registered_stacks=True, **kw_agg)


@pytest.mark.gpu
def test_errors(gpu):
    w, a = registered_agg(max_frames=100_000)
    sf = a.stack_form
    # a row naming an unregistered stack fails the flush; the next flush works
    hv, _, _ = a.acquire(3, 0)
    hv[:] = w.hdrs[:3]
    hv["frame_off"] = [0, len(sf.hashes), 1]
    a.commit(3)
    with pytest.raises(lib.PaError) as e:
        a.flush()
    assert e.value.code == EINVAL and "stack id" in str(e.value)
    lib.load(a, w)
    assert a.flush().n_rows == w.n
    # acquire with frames
    with pytest.raises(lib.PaError) as e:
        a.acquire(1, 1)
    assert e.value.code == EINVAL
    # an unknown frame id, a stack deeper than 65535, wrong hashes for the mode: nothing is registered
    n0 = a.register_stacks([], [0])
    with pytest.raises(lib.PaError) as e:
        a.register_stacks([0, len(w.frames)], [0, 2], np.zeros((1, 2), np.uint64))
    assert e.value.code == EINVAL
    with pytest.raises(lib.PaError) as e:
        a.register_stacks(np.zeros(65536, np.uint64), [0, 65536], np.zeros((1, 2), np.uint64))
    assert e.value.code == ERANGE
    with pytest.raises(lib.PaError) as e:
        a.register_stacks([0], [0, 1])  # PA_HASH_PROVIDED needs the ids
    assert e.value.code == EINVAL
    assert a.register_stacks(np.zeros(65535, np.uint64), [0, 65535], np.zeros((1, 2), np.uint64)) == n0
    a.close()
    wx, b = registered_agg(synth.edge_workload(seed=2, n=200, hash_mode=abi.PA_HASH_XXH64X2))
    with pytest.raises(lib.PaError) as e:
        b.register_stacks([0], [0, 1], np.zeros((1, 2), np.uint64))  # XXH64 mode computes them
    assert e.value.code == EINVAL
    b.close()
    # the registered frames are bounded by max_frames
    w, c = registered_agg(max_frames=10_000)
    left = 10_000 - len(c.stack_form.frames)
    c.register_stacks(np.zeros(left, np.uint64), [0, left], np.zeros((1, 2), np.uint64))
    with pytest.raises(lib.PaError) as e:
        c.register_stacks([0], [0, 1], np.zeros((1, 2), np.uint64))
    assert e.value.code == ENOSPC
    c.close()
    # register_stacks on a ring-mode aggregator
    r = lib.from_workload(w)
    with pytest.raises(lib.PaError) as e:
        r.register_stacks([0], [0, 1], np.zeros((1, 2), np.uint64))
    assert e.value.code == EINVAL
    r.close()


@pytest.mark.gpu
def test_merge_and_shard_entry_points_are_refused(gpu):
    import ctypes as C
    w, a = registered_agg()
    ring = lib.from_workload(w)
    L = lib.lib()

    def refused(rc):
        assert rc == EINVAL
        assert b"REGISTERED_STACKS" in L.pa_agg_last_error(a.h)

    h = C.c_void_p()
    refused(L.pa_merge_create_local((C.c_void_p * 2)(a.h, ring.h), 2, C.byref(h)))
    refused(L.pa_merge_create_host(a.h, None, 0, 2, C.byref(h)))
    refused(L.pa_merge_create_shm(a.h, b"/pa_registered_refused", 0, 2, 0, C.byref(h)))
    refused(L.pa_merge_create_nccl(a.h, bytes(128), 0, 2, C.byref(h)))
    lib.load(a, w)
    a.stage()
    a.process()
    refused(L.pa_agg_shard_export(a.h, 0, None, None))
    a.collect()
    refused(L.pa_agg_stage_device(a.h, None, 0, None, 0))
    refused(L.pa_agg_stage_device_parts(a.h, None, 0, 0))
    lib.load(a, w)
    assert a.flush().n_rows == w.n  # nothing was left behind
    a.close(); ring.close()
