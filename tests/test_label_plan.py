"""The label column plan of each batch: predicted from the previous batch, checked on the GPU, redone on a miss.

An agent relabels every pod label into a label name (`labelmap: __meta_kubernetes_pod_label_(.+)`), so over days the
registered labelsets name far more than the 246 label columns one record can hold, while each interval's rows name a few
dozen. The plan of a batch is the names the previous batch's rows used plus every name registered since (on a cold start:
every name, when they fit); `k_ls_plan` checks it against what the batch's labelsets name and the pass is redone with exactly
the used names when the prediction missed one. PlanModel below is that rule in plain Python; the GPU tests check that the
aggregator follows it ("label_columns", "label_replans") and that every stream stays byte-identical to the oracle fed the
same registrations and flushes.
"""
import dataclasses
import os
import subprocess
import sys
import threading

import numpy as np
import pyarrow as pa
import pytest

import pyref
from parca_agent_b200 import abi, synth

V1, V2 = abi.PA_SCHEMA_V1, abi.PA_SCHEMA_V2
XXH, PROVIDED = abi.PA_HASH_XXH64X2, abi.PA_HASH_PROVIDED
LABEL_COLS = 246   # label columns one batch can hold (kernel-parameter tables: 256 minus the kind-derived and v1 columns)
WINDOW = 34        # pod-label names each interval of the churn brings
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---- the prediction, in plain Python -----------------------------------------------------------------------------------
class PlanModel:
    """One aggregator's label column plan. flush() takes the names registered when the batch is flushed and the name ordinals
    its rows use (None: an empty interval, which leaves the prediction as it is); it returns (planned ordinals, missed) or
    raises OverflowError when the rows use more names than fit (the flush fails; the next plan starts cold)."""

    def __init__(self, sample_cols=3):
        self.sample_cols = sample_cols  # cpu / thread_id / thread_name columns of the config
        self.used_prev, self.names_planned, self.failed, self.replans = [], 0, False, 0

    def fits(self, k):
        return k + self.sample_cols <= LABEL_COLS

    def predict(self, n_names):
        if self.failed:
            self.used_prev, self.names_planned = [], 0
        pred = self.used_prev + list(range(self.names_planned, n_names))
        if not self.fits(len(pred)):
            pred = list(self.used_prev) if self.fits(len(self.used_prev)) else []
        return pred

    def flush(self, n_names, used):
        if used is None:
            return None, False
        pred, used = self.predict(n_names), sorted(set(used))
        miss = not set(used) <= set(pred)
        self.failed = True
        if miss:
            self.replans += 1
            if not self.fits(len(used)):
                raise OverflowError("too many distinct label names in one batch")
        self.used_prev, self.names_planned, self.failed = used, n_names, False
        return (used if miss else pred), miss


def test_model_cold_start_plans_every_name():
    m = PlanModel()
    assert m.flush(5, [1, 3]) == ([0, 1, 2, 3, 4], False)


def test_model_cold_start_with_too_many_names_plans_none():
    m = PlanModel()
    assert m.flush(300, [7, 250]) == ([7, 250], True) and m.replans == 1
    assert m.flush(300, [7]) == ([7, 250], False)  # the used names of the last batch


def test_model_a_new_name_is_predicted():
    m = PlanModel()
    m.flush(5, [1, 3])
    assert m.flush(7, [1, 6]) == ([1, 3, 5, 6], False)


def test_model_an_old_name_coming_back_misses():
    m = PlanModel()
    m.flush(5, [1, 3])
    m.flush(7, [1, 6])
    assert m.flush(7, [0, 1]) == ([0, 1], True) and m.replans == 1
    assert m.flush(7, [0]) == ([0, 1], False)


def test_model_an_empty_interval_keeps_the_prediction():
    m = PlanModel()
    m.flush(5, [1])
    assert m.flush(9, None) == (None, False)
    assert m.flush(9, [1, 7]) == ([1, 5, 6, 7, 8], False)  # the names registered before the empty interval are still new


def test_model_prediction_that_does_not_fit_keeps_the_used_names():
    m = PlanModel(sample_cols=0)
    m.flush(10, [2, 4])
    assert m.flush(400, [2]) == ([2, 4], False)
    assert m.flush(400, [2, 300]) == ([2, 300], True)


def test_model_a_failed_batch_restarts_cold():
    m = PlanModel(sample_cols=0)
    m.flush(3, [0])
    with pytest.raises(OverflowError):
        m.flush(300, list(range(247)))
    assert m.flush(300, [5]) == ([5], True)  # cold: 300 names do not fit, so nothing is predicted


# ---- pod-label churn ---------------------------------------------------------------------------------------------------
def name_ordinals(strings, labelsets, label_flags, ords):
    """Extend ords (name bytes -> ordinal) by the registration of labelsets, as the aggregator numbers label names."""
    off = {b"cpu": abi.PA_LABEL_DISABLE_CPU, b"thread_id": abi.PA_LABEL_DISABLE_THREAD_ID, b"thread_name": abi.PA_LABEL_DISABLE_THREAD_COMM}
    for s in labelsets:
        for n, v in s:
            name = as_bytes(strings[n])
            if not as_bytes(strings[v]) or (name in off and not label_flags & off[name]):
                continue
            ords.setdefault(name, len(ords))
    return ords


def as_bytes(s):
    return s if isinstance(s, bytes) else s.encode()


@dataclasses.dataclass
class Interval:
    new_labelsets: list
    w: synth.Workload       # this interval's rows (base rows with their labelset ids replaced)
    used: list              # name ordinals the rows use (None for an empty interval)
    n_names: int            # names registered when the interval is flushed


def churn(seed=3, n_intervals=30, rows=3000, hash_mode=XXH, label_flags=0, schema=V2, world=1, empty_at=(12,), sample_names=False,
          external_name=None):
    """A lifetime of pod-label churn: each interval registers six labelsets over the WINDOW names no earlier interval had (a
    small one with two of them first), and its rows name the edge workload's labelsets and some of the new ones. Every
    seventh interval from the fourth on also names the small labelset of three intervals before (old names coming back,
    a miss); every fifth from the fifth on names the edge labelsets only. With world > 1 the small labelset of the interval
    is named only by the first shard's rows, and an old one only by the last shard's. sample_names: one more labelset in the
    first interval carries cpu / thread_id / thread_name, and every fourth interval names it again."""
    base = synth.edge_workload(seed=seed, n=rows, hash_mode=hash_mode, label_flags=label_flags, external=False)
    st = synth.StringTable()
    st.strings, st.index = list(base.strings), {s: i for i, s in enumerate(base.strings)}
    names = [st.sid("pod_label_%04d" % k) for k in range(WINDOW * n_intervals)]
    vals = [st.sid("pv%d" % k) for k in range(12)]
    sample_ls = [(st.sid("thread_id"), vals[0]), (st.sid("cpu"), vals[1]), (st.sid("thread_name"), vals[2]), (names[5], vals[3])]
    ext = [(st.sid(external_name), st.sid("ext-value"))] if external_name else []
    w0 = dataclasses.replace(base, strings=st.strings, external_labels=ext)
    if schema == V1:
        w0.schema = V1
    rng = np.random.Generator(np.random.PCG64(seed))
    ords = name_ordinals(st.strings, w0.labelsets, label_flags, {})
    n_ls = len(w0.labelsets)
    small_of = []
    cut = [rows * i // world for i in range(world + 1)]
    ivs = []
    for i in range(n_intervals):
        win = names[WINDOW * i:WINDOW * (i + 1)]
        new = [[(win[0], vals[int(rng.integers(0, 12))]), (win[1], vals[int(rng.integers(0, 12))])]]
        for part in np.array_split(np.arange(2, WINDOW), 5):  # together the five name every name of the window
            extra = rng.choice(np.arange(2, WINDOW), size=int(rng.integers(0, 6)), replace=False)
            chosen = sorted(set(part.tolist()) | set(extra.tolist()))
            new.append([(win[c], vals[int(rng.integers(0, 12))]) for c in chosen])
        if sample_names and i == 0:
            new.append(sample_ls)
            sample_id = n_ls + len(new) - 1
        first = n_ls
        n_ls += len(new)
        ords = name_ordinals(st.strings, new, label_flags, ords)
        small_of.append(first)
        if i in empty_at:
            ivs.append(Interval(new, w0.rows(np.zeros(0, np.int64)), None, len(ords)))
            continue
        hd = w0.hdrs.copy()
        base_ids = np.arange(len(w0.labelsets))
        pool = base_ids if i % 5 == 4 else np.concatenate([base_ids, np.arange(first + 1, first + 6)])
        ls = pool[np.repeat(rng.integers(0, len(pool), rows // 25 + 1), 25)[:rows]]
        if i % 5 != 4:  # the small labelset, on the first shard's rows
            ls[rng.integers(0, cut[1], 3)] = first
        if i % 7 == 3 and i >= 3:  # an old labelset, on the last shard's rows
            ls[rng.integers(cut[world - 1], rows, 3)] = small_of[i - 3]
        if sample_names and i % 4 == 0:
            ls[rng.integers(0, rows, 5)] = sample_id
        hd["labelset_id"] = ls
        w = dataclasses.replace(w0, hdrs=hd, name="churn_%d" % i)
        all_ls = list(w0.labelsets) + [s for iv in ivs for s in iv.new_labelsets] + new
        on = {as_bytes(st.strings[n]) for k in np.unique(ls) for n, _ in all_ls[k]}
        used = sorted(ords[x] for x in on if x in ords)
        ivs.append(Interval(new, w, used, len(ords)))
    w0.meta = dict(w0.meta, ords=ords)
    return w0, ivs


def test_churn_grows_past_the_old_limit_with_misses_and_hits():
    """The sequence crosses what the GPU tests rely on: >1000 names over the lifetime, at most 40 per interval, misses and hits."""
    w0, ivs = churn()
    assert ivs[-1].n_names > 1000
    assert max(len(iv.used) for iv in ivs if iv.used is not None) <= 40
    m = PlanModel()
    missed = [m.flush(iv.n_names, iv.used)[1] for iv in ivs if iv.used is not None]
    assert any(missed) and not all(missed)
    assert any(iv.used is None for iv in ivs)


# ---- the GPU side ------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from parca_agent_b200 import lib
    lib.lib()
    return lib


def oracle_register_labelsets(o, labelsets):
    from oracle import oracle_py
    if labelsets:
        pairs, offs = abi.pack_labelsets(labelsets)
        oracle_py.lib().orc_register_labelsets(o.h, pairs.ctypes.data, offs.ctypes.data, len(labelsets), None)


def oracle_flush(o, w):
    o.ingest(w.hdrs, w.frame_ids)
    return o.flush()[0]


def plan_counters(a):
    return a.kernel_ms("label_columns")[1], a.kernel_ms("label_replans")[1]


def same(want, got, schema=V2):
    if got != want:
        d = None
        if want and got:
            ex = pyref.extract_v1 if schema == V1 else pyref.extract
            d = pyref.diff(ex(pa.ipc.open_stream(want).read_all()), ex(pa.ipc.open_stream(got).read_all()))
        raise AssertionError("IPC bytes differ (len %d vs %d); first logical difference: %s" % (len(want), len(got), d))


MODES = {
    "v2_xxh": dict(hash_mode=XXH),
    "v2_provided": dict(hash_mode=PROVIDED),
    "narrow_ring": dict(hash_mode=XXH, agg=dict(frame_id_bytes=4)),
    "registered_stacks": dict(hash_mode=PROVIDED, agg=dict(registered_stacks=True)),
    "v1_requests": dict(hash_mode=XXH, schema=V1),
    "lz4_gpu": dict(hash_mode=XXH, agg=dict(ipc_compression=abi.PA_IPC_LZ4_FRAME_GPU)),
}


def run_lifetime(gpu, w0, ivs, agg=None, schema=V2, label_flags=0, expect_miss=True):
    """One aggregator and one oracle through the intervals; every stream and the plan counters checked after each flush."""
    from oracle import oracle_py
    from test_gpu_parity import assert_same_stacktraces
    from test_ipc_lz4_gpu import check_stream
    agg = dict(agg or {})
    lz4 = agg.get("ipc_compression") == abi.PA_IPC_LZ4_FRAME_GPU
    o = oracle_py.Oracle(w0)
    a = gpu.from_workload(w0, max_samples=max(iv.w.n for iv in ivs) or 1, **agg)
    sample_cols = 3 - bin(label_flags & 7).count("1")
    m = PlanModel(sample_cols)
    misses = hits = 0
    try:
        for iv in ivs:
            a.register_labelsets(iv.new_labelsets)
            oracle_register_labelsets(o, iv.new_labelsets)
            want = oracle_flush(o, iv.w)
            gpu.load(a, iv.w, stack_of_row=a.stack_form.stack_of_row[:iv.w.n] if a.registered else None)
            r = a.flush()
            got = r.ipc_bytes()
            if lz4:
                check_stream(got, want)
            else:
                same(want, got, schema)
            planned, missed = m.flush(iv.n_names, iv.used)
            if planned is not None:
                assert plan_counters(a) == (len(planned), m.replans), (iv.w.name, planned)
                misses, hits = misses + missed, hits + (not missed)
            if schema == V1 and r.n_unique_stacks:
                ids = a.last_stack_ids(r.n_unique_stacks)
                assert_same_stacktraces(o, a, [bytes(x) for x in ids[::3]])
    finally:
        a.close()
        o.close()
    if expect_miss:
        assert misses and hits
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
def test_lifetime_beyond_the_old_limit(gpu, mode):
    md = MODES[mode]
    w0, ivs = churn(hash_mode=md["hash_mode"], schema=md.get("schema", V2))
    assert ivs[-1].n_names > 1000
    run_lifetime(gpu, w0, ivs, agg=md.get("agg"), schema=md.get("schema", V2))


@pytest.mark.gpu
def test_miss_in_chunked_flush_with_early_copy_out(gpu, monkeypatch):
    monkeypatch.setenv("PA_EARLY_D2H_ALWAYS", "1")
    w0, ivs = churn(seed=8, n_intervals=12, rows=6000)
    m = run_lifetime(gpu, w0, ivs, agg=dict(chunk_samples=700))
    assert m.replans >= 1


@pytest.mark.gpu
@pytest.mark.parametrize("label_flags", range(8))
def test_label_disable_flags_with_sample_label_names_in_labelsets(gpu, label_flags):
    w0, ivs = churn(seed=11, n_intervals=9, label_flags=label_flags, sample_names=True, empty_at=())
    run_lifetime(gpu, w0, ivs, label_flags=label_flags)


@pytest.mark.gpu
def test_external_label_named_by_some_batches_only(gpu):
    # pod_label_0003 is in the first interval's window: some intervals' rows carry it, the rest get it from the external label
    w0, ivs = churn(seed=5, n_intervals=10, external_name="pod_label_0003", empty_at=())
    o3 = w0.meta["ords"][b"pod_label_0003"]
    carried = {iv.w.name for iv in ivs if iv.used is not None and o3 in iv.used}
    assert carried and len(carried) < len(ivs)
    run_lifetime(gpu, w0, ivs)


def wide(n_names, n_used, seed=2):
    """Labelsets over n_names names; the rows name only those over the first n_used (label flags 0: three more columns)."""
    base = synth.edge_workload(seed=seed, n=2000, hash_mode=XXH, external=False)
    st = synth.StringTable()
    st.strings, st.index = list(base.strings), {s: i for i, s in enumerate(base.strings)}
    nm = [st.sid("wide_%03d" % k) for k in range(n_names)]
    v = st.sid("v")
    rows_ls = [[(nm[k], v) for k in range(j, min(j + 50, n_used))] for j in range(0, n_used, 50)]
    rest = [[(nm[k], v) for k in range(j, min(j + 50, n_names))] for j in range(n_used, n_names, 50)]
    k = len(base.labelsets)
    w = dataclasses.replace(base, strings=st.strings, labelsets=list(base.labelsets) + rows_ls + rest)
    hd = w.hdrs.copy()
    hd["labelset_id"] = k + np.arange(len(hd)) % len(rows_ls)
    return dataclasses.replace(w, hdrs=hd, meta=dict(w.meta, first_wide=k))


@pytest.mark.gpu
def test_per_batch_limit(gpu):
    """Rows that use 247 names fail the flush with PA_ERANGE; the next flush, with fewer names, is byte-exact; a batch that fills
    the label columns exactly (243 names + cpu, thread_id, thread_name) works."""
    from oracle import oracle_py
    a = gpu.from_workload(wide(400, 247))
    gpu.load(a, wide(400, 247))
    with pytest.raises(gpu.PaError) as e:
        a.flush()
    assert e.value.code == -34 and "limit 246" in str(e.value)
    registered = list(wide(400, 247).labelsets)
    for n_used in (40, 243):
        w = wide(400, n_used)
        k = w.meta["first_wide"]
        a.register_labelsets(w.labelsets[k:])  # this batch's labelsets, registered after the failed batch's
        hd = w.hdrs.copy()
        hd["labelset_id"] += len(registered) - k
        registered += w.labelsets[k:]
        w = dataclasses.replace(w, labelsets=list(registered), hdrs=hd)
        gpu.load(a, w)
        same(oracle_py.run(w)[0], a.flush().ipc_bytes())
        assert plan_counters(a)[0] == n_used
    a.close()


@pytest.mark.gpu
def test_new_names_registered_during_flushes(gpu):
    """A producer thread registers labelsets with ever new label NAMES while the batch is flushed again and again: the pass uses
    the registrations it snapshotted, the prediction grows past what fits and falls back to the used names, and every record
    stays byte-exact."""
    from oracle import oracle_py
    w = synth.edge_workload(seed=61, n=4000, hash_mode=XXH, external=False)
    want, _ = oracle_py.run(w)
    a = gpu.from_workload(w)
    stop, errors = threading.Event(), []

    def registrar():
        i = 0
        try:
            while not stop.is_set():
                first = a.register_strings([("late-name-%d-%d" % (i, k)).encode() for k in range(6)])
                a.register_labelsets([[(first, first + 3)], [(first + 1, first + 4), (first + 2, first + 5)]])
                i += 1
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))

    t = threading.Thread(target=registrar)
    t.start()
    try:
        for _ in range(40):
            gpu.load(a, w)
            assert a.flush().ipc_bytes() == want
    finally:
        stop.set()
        t.join()
    a.close()
    assert not errors, errors


# ---- merge groups ------------------------------------------------------------------------------------------------------
def spans(n, world):
    cut = [n * i // world for i in range(world + 1)]
    return [np.arange(cut[i], cut[i + 1]) for i in range(world)]


@pytest.mark.gpu
@pytest.mark.parametrize("schema", [V2, V1])
def test_merge_group_names_on_one_shard_and_a_miss_on_one_shard(gpu, schema):
    """Three local members through a churn in which each interval's small labelset is named by the first shard's rows only and
    an old one (a miss) by the last shard's only: each merged stream equals that of one aggregator on the concatenated rows
    and the oracle's, and every member follows the group-wide plan."""
    from oracle import oracle_py
    W = 3
    w0, ivs = churn(seed=21, n_intervals=12, rows=3000, schema=schema, world=W)
    o = oracle_py.Oracle(w0)
    single = gpu.from_workload(w0)
    members = [gpu.from_workload(w0) for _ in range(W)]
    g = gpu.MergeGroup.local(members)
    m = PlanModel()
    try:
        for iv in ivs:
            for x in [single] + members:
                x.register_labelsets(iv.new_labelsets)
            oracle_register_labelsets(o, iv.new_labelsets)
            want = oracle_flush(o, iv.w)
            gpu.load(single, iv.w)
            one = single.flush().ipc_bytes()
            same(want, one, schema)
            for a, ix in zip(members, spans(iv.w.n, W)):
                gpu.load(a, iv.w.rows(ix))
            res = g.flush()
            same(want, res.ipc_bytes(), schema)
            planned, _ = m.flush(iv.n_names, iv.used)
            if planned is not None:
                for x in [single] + members:
                    assert plan_counters(x) == (len(planned), m.replans), iv.w.name
        assert m.replans >= 1
    finally:
        g.close()
        for x in [single] + members:
            x.close()
        o.close()


@pytest.mark.gpu
def test_merge_group_after_members_flushed_alone(gpu):
    """Each member of a local group flushes a batch of its own, so each predicts the next merged batch from different names.
    First the plans have the same size but different names: a name every member planned sits at different columns, and the
    merged batch names only it (no member misses). Then the plans differ in size. Every merged stream equals the oracle's."""
    from oracle import oracle_py
    base = synth.edge_workload(seed=31, n=1200, hash_mode=XXH, external=False)
    st = synth.StringTable()
    st.strings, st.index = list(base.strings), {s: i for i, s in enumerate(base.strings)}
    na, nc, nb, v = st.sid("solo_a"), st.sid("shared_c"), st.sid("solo_b"), st.sid("v")
    k = len(base.labelsets)  # k: {solo_a, shared_c}; k + 1: {shared_c, solo_b}; k + 2: {shared_c} (ordinals a < c < b)
    w = dataclasses.replace(base, strings=st.strings, labelsets=list(base.labelsets) + [[(na, v), (nc, v)], [(nc, v), (nb, v)], [(nc, v)]])

    def named(ls):
        hd = w.hdrs.copy()
        hd["labelset_id"] = ls
        return dataclasses.replace(w, hdrs=hd)

    members = [gpu.from_workload(w) for _ in range(3)]
    g = gpu.MergeGroup.local(members)

    def group_flush(x):
        for a, ix in zip(members, spans(x.n, 3)):
            gpu.load(a, x.rows(ix))
        same(oracle_py.run(x)[0], g.flush().ipc_bytes())

    try:
        group_flush(w)
        for solo in ([k, k + 1, k], [k, 2, k + 1]):
            for a, ls in zip(members, solo):
                x = named(np.full(w.n, ls, dtype=np.uint32))
                gpu.load(a, x)
                same(oracle_py.run(x)[0], a.flush().ipc_bytes())
            group_flush(named(np.full(w.n, k + 2, dtype=np.uint32)))
            group_flush(w)
        assert len({plan_counters(a)[0] for a in members}) == 1
    finally:
        g.close()
        for a in members:
            a.close()


@pytest.mark.gpu
@pytest.mark.parametrize("transport,mailbox", [("gloo", 0), ("shm", 4096)])
def test_multi_process_group(transport, mailbox):
    """Three processes, one member each, on this one GPU (tests/dist_label_plan_check.py): a churn with a name on one shard
    only and misses on one shard only, and members that flush alone in between, against the oracle"""
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", PA_ONE_GPU="1", PA_MERGE_TRANSPORT=transport, PA_SHM_MAILBOX=str(mailbox))
    port = 29751 + (10 if transport == "shm" else 0)
    p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "3", "--master-addr", "127.0.0.1",
                        "--master-port", str(port), os.path.join(ROOT, "tests", "dist_label_plan_check.py")], capture_output=True, text=True, env=env, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    assert "label-plan ok world=3 transport=%s" % transport in p.stdout
