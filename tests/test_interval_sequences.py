"""Long-lived aggregators and merge groups through one sequence of unlike intervals, each flush against the oracle.

An agent keeps one aggregator open for days, and every interval differs from the one before in size, stacks, thread ids,
registered label names and the order in which sample kinds first appear. Much state carries from one flush to the next:
the per-flush arena laid out again from each interval's sizes, table capacities predicted from the previous interval,
the v1 kind order and the `stacks` LRU, the early copy-out positions, the column plan, the registered-stack mirrors.
Repeating one batch cannot show a kernel that reads a stale word: the stale bytes are then the right ones. Here one
registry grows over the lifetime (every interval registers what it brings and is rewritten onto the union's ids), one
oracle lives through the same registrations, flushes and stacktrace requests, and every mode runs the same sequence on
one aggregator or group. A failing flush is replayed through a fresh aggregator to tell carried state from a bug in that
batch alone. The CPU-only self-checks assert, for 132 and 114 SMs, that the sequence crosses what it claims to cross.
"""
import collections
import ctypes as C
import dataclasses
import functools

import numpy as np
import pytest

import pyref
import test_scale_edges as se
from parca_agent_b200 import abi, synth
from test_gpu_parity import wide_label_workload
from test_ipc_lz4_gpu import check_buffers, check_stream

V1, V2 = abi.PA_SCHEMA_V1, abi.PA_SCHEMA_V2
XXH, PROVIDED = abi.PA_HASH_XXH64X2, abi.PA_HASH_PROVIDED
SPS = 19                  # samples_per_second: one setting for the whole lifetime
STORE_ENTRIES = 3500      # v1 stack_cache_entries: f alone holds more stacks; e, g, h and i push a full store over it
F_STACKS, F_TIDS = 650_000, 320_000
NAMES = "abcdefghij"
FRAME_SID_FIELDS = [n for n in abi.FRAME_DTYPE.names if n.endswith("_sid")]


# ---- the intervals ------------------------------------------------------------------------------------------------------
def first_kinds(hd):
    k = hd["kind"]
    u, first = np.unique(k, return_index=True)
    return tuple(int(x) for x in u[np.argsort(first)])


def with_new_name(w, row):
    """d: one row carries a labelset whose name no earlier interval registered (the column plan is rebuilt)"""
    st = synth.StringTable()
    st.strings, st.index = list(w.strings), {s: i for i, s in enumerate(w.strings)}
    ls = list(w.labelsets) + [[(st.sid("registered_just_before_d"), st.sid("d-value"))]]
    hd = w.hdrs.copy()
    hd["labelset_id"][row] = len(ls) - 1
    return dataclasses.replace(w, strings=st.strings, labelsets=ls, hdrs=hd)


def wide_interval(n=600_000, seed=9):
    """e: 200 label names in labelset runs, rows drawn from wide_label_workload's (mostly its 0-3-frame stacks), so the
    interval has few distinct stacks and thread ids and the tables of f are predicted small"""
    base = wide_label_workload(200, n=1500, seed=seed)
    rng = np.random.Generator(np.random.PCG64(seed))
    nf = base.hdrs["nframes"]
    shallow, deep = np.nonzero(nf <= 3)[0], np.nonzero(nf > 3)[0]
    idx = np.where(rng.random(n) < 0.97, shallow[rng.integers(0, len(shallow), n)], deep[rng.integers(0, len(deep), n)])
    w = base.rows(idx)
    # mostly the labelset with the most names: a row where a column is null is a run of its own, so nulls cost output
    dense = max(range(len(base.labelsets)), key=lambda i: len(base.labelsets[i]))
    p = np.full(len(base.labelsets), 0.1 / (len(base.labelsets) - 1))
    p[dense] = 0.9
    w.hdrs["labelset_id"] = se._runs(rng, n, 200, np.arange(len(base.labelsets)), p=p)
    w.hdrs["timestamp_ns"] = se.T0 + np.arange(n, dtype=np.int64) * 977
    return dataclasses.replace(w, name="wide_%d" % n, samples_per_second=SPS)


def many_stacks(n, n_stacks, n_tids, seed, kinds):
    """f / g: 3-frame stacks over config 1's frames; stack s has frames (s mod 4096, s div 4096, ...), so every stack has
    its own frame sequence (XXH64 ids stay distinct). Each stack and thread id occurs at least once."""
    base = synth.config1()
    rng = np.random.Generator(np.random.PCG64(seed))

    def draw(m):
        x = np.concatenate([np.arange(m), rng.integers(0, m, n - m)]) if m < n else rng.integers(0, m, n)
        return rng.permutation(x).astype(np.int64)

    s, t = draw(n_stacks), draw(n_tids)
    su = s.astype(np.uint64)
    fr = np.stack([su % np.uint64(4096), su // np.uint64(4096), (su * np.uint64(2654435761)) % np.uint64(4096)], axis=1)
    comms = np.unique(base.hdrs["comm_sid"])
    hd = np.zeros(n, dtype=abi.HDR_DTYPE)
    hd["hash_hi"] = synth.splitmix64(su + np.uint64(1 << 40))
    hd["hash_lo"] = synth.splitmix64(su ^ np.uint64(0x5DEECE66D))
    hd["timestamp_ns"] = se.T0 + np.arange(n, dtype=np.int64) * 1000
    hd["value"] = rng.integers(1, 1 << 30, n)
    hd["pid"] = 1000 + rng.integers(0, 64, n)
    hd["tid"] = 7 + t
    hd["comm_sid"] = se._runs(rng, n, 20, comms)
    hd["labelset_id"] = se._runs(rng, n, 30, np.arange(len(base.labelsets)))
    hd["cpu"] = rng.integers(0, 8, n)
    hd["kind"] = se._runs(rng, n, 5000, kinds)
    hd["nframes"] = 3
    hd["frame_off"] = np.arange(n, dtype=np.uint64) * np.uint64(3)
    return synth.Workload("stacks%d_tids%d" % (n_stacks, n_tids), base.strings, base.frames, base.labelsets, hd,
                          _frame_ids=fr.reshape(-1), hash_mode=PROVIDED, samples_per_second=SPS)


def kinds_first_in_a_new_order(w, earlier):
    """i: edge_workload's kinds relabelled so that their first-appearance order is one no earlier interval had"""
    order = first_kinds(w.hdrs)
    assert len(order) == 7
    for shift in range(7):
        target = tuple((6 - j + shift) % 7 for j in range(7))
        if target not in earlier:
            break
    perm = np.zeros(7, dtype=np.uint8)
    perm[list(order)] = target
    hd = w.hdrs.copy()
    hd["kind"] = perm[hd["kind"]]
    return dataclasses.replace(w, hdrs=hd)


def local_intervals(sms):
    empty = synth.edge_workload(seed=1, n=0, external=False)
    scale = se.scale_batch(se.n_for_per(160, sms), sms, seed=160)
    seq = [empty, synth.edge_workload(seed=2, n=1, external=False), scale,
           with_new_name(synth.edge_workload(seed=4, n=33, external=False), 17), wide_interval(),
           many_stacks(1_200_000, F_STACKS, F_TIDS, 6, [abi.PA_KIND_CPU, abi.PA_KIND_CUDA]),
           many_stacks(1_200_000, 10, 1, 7, [abi.PA_KIND_OFFCPU]), scale]
    earlier = {first_kinds(w.hdrs) for w in seq}
    seq.append(kinds_first_in_a_new_order(synth.edge_workload(seed=12, n=600, external=False), earlier))
    seq.append(empty)
    return seq


# ---- one registry for the lifetime ----------------------------------------------------------------------------------
@dataclasses.dataclass
class Interval:
    name: str
    w: synth.Workload        # rows on the union's ids; strings / frames / labelsets: the registry so far
    new_strings: list        # what this interval registers before its rows arrive
    new_frames: np.ndarray
    new_labelsets: list
    keys: np.ndarray         # per row: a 64-bit digest of the stack's frame ids (the stack, in XXH64 mode)
    last_order: list         # the interval's distinct keys by last occurrence
    reg_frames: np.ndarray   # registered stacks: this interval's new stacks (frames, offsets) and every row's stack id
    reg_offsets: np.ndarray
    stack_of_row: np.ndarray


def stack_keys(hd, stream):
    nf = hd["nframes"].astype(np.int64)
    off = hd["frame_off"].astype(np.int64)
    start = se._excl_cumsum(nf) if len(nf) else np.zeros(0, np.int64)
    total = int(nf.sum())
    pos = np.arange(total, dtype=np.int64) - np.repeat(start, nf)
    fid = np.asarray(stream, dtype=np.uint64)[np.repeat(off, nf) + pos]
    with np.errstate(over="ignore"):
        v = synth.splitmix64(fid * np.uint64(0x9E3779B97F4A7C15) + pos.astype(np.uint64))
        cs = np.zeros(total + 1, dtype=np.uint64)
        np.cumsum(v, out=cs[1:])
        return (cs[start + nf] - cs[start]) ^ synth.splitmix64(nf.astype(np.uint64) + np.uint64(12345))


class Registry:
    """The union of the intervals' strings, frames, labelsets and stacks; each registered once, when it first arrives."""

    def __init__(self):
        self.strings, self.sidx = [b""], {b"": 0}
        self.frames, self.fidx = [], {}
        self.labelsets, self.lidx = [], {}
        self.stacks = {}  # key -> registered stack id

    def _intern(self, table, index, item):
        i = index.get(item)
        if i is None:
            i = index[item] = len(table)
            table.append(item)
        return i

    def admit(self, name, w):
        ns, nf, nl = len(self.strings), len(self.frames), len(self.labelsets)
        smap = np.array([self._intern(self.strings, self.sidx, s) for s in w.strings], dtype=np.uint32)
        fr = np.array(w.frames, dtype=abi.FRAME_DTYPE, copy=True)
        for f in FRAME_SID_FIELDS:
            fr[f] = smap[fr[f]]
        fmap = np.array([self._intern(self.frames, self.fidx, fr[i:i + 1].tobytes()) for i in range(len(fr))] or [0], dtype=np.uint64)
        lmap = np.array([self._intern(self.labelsets, self.lidx, tuple((int(smap[k]), int(smap[v])) for k, v in s))
                         for s in w.labelsets] or [0], dtype=np.uint32)
        hd = w.hdrs.copy()
        hd["comm_sid"] = smap[hd["comm_sid"]]
        hd["labelset_id"] = lmap[hd["labelset_id"]]
        ids = fmap[np.asarray(w.frame_ids, dtype=np.int64)]
        frames = np.frombuffer(b"".join(self.frames), dtype=abi.FRAME_DTYPE).copy()
        gw = synth.Workload(w.name, list(self.strings), frames, [list(s) for s in self.labelsets], hd, _frame_ids=ids,
                            hash_mode=PROVIDED, samples_per_second=SPS, meta={})
        keys = stack_keys(hd, ids)
        uk, first, inv = np.unique(keys, return_index=True, return_inverse=True)
        last = np.full(len(uk), -1, dtype=np.int64)
        np.maximum.at(last, inv, np.arange(len(keys)))
        last_order = uk[np.argsort(last)].tolist()
        # registered stacks (XXH64 mode: a stack is its frame sequence)
        gid = np.zeros(len(uk), dtype=np.uint64)
        new = []
        for j, k in enumerate(uk.tolist()):
            s = self.stacks.get(k)
            if s is None:
                s = self.stacks[k] = len(self.stacks)
                new.append(j)
            gid[j] = s
        rows = first[np.asarray(new, dtype=np.int64)]
        depth = hd["nframes"][rows].astype(np.int64)
        offs = np.zeros(len(rows) + 1, dtype=np.uint64)
        offs[1:] = np.cumsum(depth)
        src = np.repeat(hd["frame_off"][rows].astype(np.int64), depth) + (np.arange(int(depth.sum())) - np.repeat(offs[:-1].astype(np.int64), depth))
        return Interval(name, gw, self.strings[ns:], np.frombuffer(b"".join(self.frames[nf:]), dtype=abi.FRAME_DTYPE).copy(),
                        [list(s) for s in self.labelsets[nl:]], keys, last_order, ids[src], offs, gid[inv])


@functools.lru_cache(maxsize=1)
def sequence(sms):
    reg = Registry()
    return [reg.admit(name, w) for name, w in zip(NAMES, local_intervals(sms))]


# ---- the v1 store, modelled as the reference's LRU ------------------------------------------------------------------
UNKNOWN = [("unknown", j) for j in range(3)]


def design_request(od, seen, prev_old):
    """Between intervals: the oldest live entries (refreshed here, so they must outlive the next eviction), the ones the
    previous request refreshed, a sample of evicted and of recent entries, never-seen ids, and repeats"""
    live = list(od)
    old = live[:min(256, len(live) // 4)]
    gone = [k for k in seen if k not in od]
    gone = gone[::max(1, len(gone) // 64)][:64]
    recent = live[-16:]
    return prev_old[:32] + old + gone[:32] + UNKNOWN[:2] + recent + gone[32:] + old[:3] + UNKNOWN[2:] + recent[:2]


def lru_walk(ivs, cap, requests=None):
    """Per interval: (distinct stacks U, live entries before, entries evicted, the request after it, the live set after the
    request). requests=None designs the requests and lets them refresh what they find; given requests do not refresh."""
    od, seen, seen_set, out, prev_old = collections.OrderedDict(), [], set(), [], []
    for k, iv in enumerate(ivs):
        live = len(od)
        for x in iv.last_order:
            od[x] = None
            od.move_to_end(x)
            if x not in seen_set:
                seen_set.add(x)
                seen.append(x)
        evicted = max(0, len(od) - cap)
        for _ in range(evicted):
            od.popitem(last=False)
        if requests is None:
            req = design_request(od, seen, prev_old)
            prev_old = list(od)[:min(256, len(od) // 4)]
            for x in req:
                if x in od:
                    od.move_to_end(x)
        else:
            req = requests[k]
        out.append(dict(U=len(iv.last_order), live=live, evicted=evicted, request=req, after=frozenset(od)))
    return out


# ---- CPU-tier self-checks --------------------------------------------------------------------------------------------
def pow2_at_least(x):
    return 1 << max(0, int(x - 1).bit_length())


def table_bound(n, prev, big, floor_):
    """agg.cu table_bound"""
    return n if n <= big else min(n, max(prev * 4 if prev else n // 16, floor_))


def predicted_caps(n, prev_unique, prev_tids):
    """agg.cu pass_plan: (stack table, thread-id table) capacities; a table overflows when more distinct keys arrive"""
    cap = max(pow2_at_least(2 * max(table_bound(n, prev_unique, 1 << 20, 1 << 18), 1)), 1024)
    tcap = max(pow2_at_least(2 * max(table_bound(n, prev_tids, 1 << 18, 1 << 16), 16)), 1024)
    return cap, tcap


def n_tids(w):
    return len(np.unique(w.hdrs["tid"]))


def check_table_predictions(ivs, sms):
    by = {iv.name: iv for iv in ivs}
    c, e, f, g = by["c"], by["e"], by["f"], by["g"]
    assert by["b"].w.n == 1 and len(by["b"].last_order) == 1
    assert c.w.n > 1 << 20 and g.w.n > 1 << 20 and f.w.n > 1 << 20
    assert np.array_equal(by["h"].w.hdrs, c.w.hdrs) and np.array_equal(by["h"].w.frame_ids, c.w.frame_ids)
    assert predicted_caps(c.w.n, 1, 1)[0] >= 2 * len(c.last_order)  # c: sized from b's single stack, and it fits
    cap, tcap = predicted_caps(f.w.n, len(e.last_order), n_tids(e.w))
    assert len(f.last_order) >= 600_000 and n_tids(f.w) >= 300_000
    assert len(f.last_order) > cap and n_tids(f.w) > tcap  # both tables overflow: the pass is redone with 4x larger ones
    cap_g, tcap_g = predicted_caps(g.w.n, len(f.last_order), n_tids(f.w))
    assert len(g.last_order) == 10 and n_tids(g.w) == 1 and cap_g >= 1 << 21 and tcap_g >= 1 << 20  # far too large
    assert 5_000_000 <= sum(iv.w.n for iv in ivs) <= 6_000_000
    assert by["a"].w.n == by["j"].w.n == 0


def check_label_columns(ivs, sms):
    e = next(iv for iv in ivs if iv.name == "e")
    assert se.ree_per(e.w.n, sms) >= 3 * se.REE_STEP
    names = {k for s in e.w.labelsets for k, _ in s}
    present = {k for ls in np.unique(e.w.hdrs["labelset_id"]) for k, _ in e.w.labelsets[ls]}
    assert len(present) >= 200 and len(names) >= 200
    d = next(iv for iv in ivs if iv.name == "d")
    (pair,) = d.new_labelsets[-1]
    assert d.w.strings[pair[0]] == b"registered_just_before_d" and pair[0] >= len(d.w.strings) - len(d.new_strings)
    assert np.sum(d.w.hdrs["labelset_id"] == len(d.w.labelsets) - 1) == 1 and d.w.n == 33


def check_kind_orders(ivs, sms):
    orders = [first_kinds(iv.w.hdrs) for iv in ivs]
    i = NAMES.index("i")
    assert sorted(orders[i]) == list(range(7))
    assert all(orders[i] != o for o in orders[:i])


def check_store_crossings(ivs, sms):
    walk = lru_walk(ivs, STORE_ENTRIES)
    C = STORE_ENTRIES
    assert any(s["U"] >= C for s in walk)                                      # one interval alone fills the store
    assert any(s["U"] < C < s["live"] + s["U"] and s["evicted"] for s in walk)  # a filled store evicts for a smaller one
    # the same requests without their refreshes: some later eviction removes other entries, and the next request asks for
    # one of them (a store whose request accesses are not newer than the batch before them fails there)
    stale = lru_walk(ivs, C, requests=[s["request"] for s in walk])
    hits = [k for k in range(1, len(ivs)) if walk[k]["evicted"] and walk[k - 1]["after"] == stale[k - 1]["after"]
            and any(x in (walk[k]["after"] ^ stale[k]["after"]) for x in walk[k]["request"])]
    assert hits, [(s["U"], s["live"], s["evicted"]) for s in walk]
    for s in walk:  # every request asks for never-seen ids and repeats the ones it asks for
        req = [x for x in s["request"] if not isinstance(x, tuple)]
        assert any(isinstance(x, tuple) for x in s["request"]) and (len(req) > len(set(req)) or not req)
    mixed = [s for s in walk if any(x in s["after"] for x in s["request"]) and any(not isinstance(x, tuple) and x not in s["after"] for x in s["request"])]
    assert len(mixed) >= 4  # live and evicted ids in one request



@pytest.fixture(scope="module", params=[132, 114])
def plan(request):
    return sequence(request.param), request.param


def test_tables_are_mispredicted_where_the_plan_says(plan):
    check_table_predictions(*plan)


def test_run_end_warps_take_three_substeps_in_the_wide_interval(plan):
    check_label_columns(*plan)


def test_kinds_first_appear_in_a_new_order_in_i(plan):
    check_kind_orders(*plan)


def test_store_crossings_and_a_request_that_decides_the_eviction(plan):
    check_store_crossings(*plan)


# ---- GPU: the lifetimes ------------------------------------------------------------------------------------------------
@dataclasses.dataclass(frozen=True)
class Mode:
    hash_mode: int = XXH
    schema: int = V2
    world: int = 1
    registered: bool = False
    env: tuple = ()
    opts: tuple = ()


MODES = {
    "xxh64": Mode(),
    "provided": Mode(hash_mode=PROVIDED),
    "narrow_ring": Mode(opts=(("frame_id_bytes", 4),)),
    "early_copy_chunks": Mode(env=(("PA_EARLY_D2H_ALWAYS", "1"),), opts=(("chunk_samples", 100_003),)),
    "registered_stacks": Mode(registered=True),
    "lz4_gpu": Mode(opts=(("ipc_compression", abi.PA_IPC_LZ4_FRAME_GPU),)),
    "v1": Mode(schema=V1),
    "merge_v2": Mode(world=3),
    "merge_v1": Mode(schema=V1, world=3),
}


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from parca_agent_b200 import lib
    lib.lib()
    return lib


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def spans(w, world):
    cut = [w.n * i // world for i in range(world + 1)]
    return list(zip(cut[:-1], cut[1:]))


def thirds(w):
    return [se.part_of(w, p0, p1) if p1 > p0 else w.head(0) for p0, p1 in spans(w, 3)]


def as_mode(w, m):
    return dataclasses.replace(w, hash_mode=m.hash_mode, schema=m.schema)


def stack_id(w, key_row):
    from oracle import oracle_py
    off, nf = int(w.hdrs["frame_off"][key_row]), int(w.hdrs["nframes"][key_row])
    data = np.asarray(w.frame_ids[off:off + nf], dtype="<u8").tobytes()
    return oracle_py.xxh64(data, 0).to_bytes(8, "big") + oracle_py.xxh64(data, abi.PA_XXH_SEED_LO).to_bytes(8, "big")


@functools.lru_cache(maxsize=1)
def request_blobs(sms):
    """the 16-byte ids of every designed request (XXH64 ids, computed from a row that carries the stack)"""
    ivs = sequence(sms)
    where = {}
    for iv in ivs:
        for k, r in zip(*np.unique(iv.keys, return_index=True)):
            where.setdefault(int(k), (iv.w, int(r)))
    out = []
    for s in lru_walk(ivs, STORE_ENTRIES):
        out.append(b"".join(bytes([0xEE, x[1]]) * 8 if isinstance(x, tuple) else stack_id(*where[x]) for x in s["request"]))
    return out


def oracle_register(o, iv):
    from oracle import oracle_py
    L = oracle_py.lib()
    if iv.new_strings:
        blob, offs = abi.pack_strings(iv.new_strings)
        L.orc_register_strings(o.h, blob, offs.ctypes.data, len(iv.new_strings), C.byref(C.c_uint32()))
    if len(iv.new_frames):
        L.orc_register_frames(o.h, iv.new_frames.ctypes.data, len(iv.new_frames), None)
    if iv.new_labelsets:
        pairs, offs = abi.pack_labelsets(iv.new_labelsets)
        L.orc_register_labelsets(o.h, pairs.ctypes.data, offs.ctypes.data, len(iv.new_labelsets), None)


@functools.lru_cache(maxsize=3)
def oracle_lifetime(sms, hash_mode, schema):
    """One oracle through the whole sequence: per interval (record bytes, stats, stacktrace record after it or None)"""
    from oracle import oracle_py
    ivs = sequence(sms)
    v1 = schema == V1
    o = oracle_py.Oracle(dataclasses.replace(ivs[0].w, strings=[b""], frames=np.zeros(0, abi.FRAME_DTYPE), labelsets=[],
                                             hash_mode=hash_mode, schema=schema), stack_cache_entries=STORE_ENTRIES if v1 else 0)
    out = []
    try:
        for k, iv in enumerate(ivs):
            oracle_register(o, iv)
            o.ingest(iv.w.hdrs, iv.w.frame_ids)
            rec, st = o.flush()
            out.append((rec, st, o.stacktraces(request_blobs(sms)[k])[0] if v1 else None))
    finally:
        o.close()
    return out


def agg_options(m, ivs, world):
    parts = [thirds(iv.w) if world > 1 else [iv.w] for iv in ivs]
    opts = dict(hash_mode=m.hash_mode, schema=m.schema, samples_per_second=SPS,
                max_samples=max(max(p.n for p in ps) for ps in parts) or 1,
                max_frames=max(max(p.n_frame_ids for p in ps) for ps in parts) or 1,
                stack_cache_entries=STORE_ENTRIES if m.schema == V1 else 0)
    if m.registered:
        opts.update(flags=abi.PA_CFG_REGISTERED_STACKS, max_frames=sum(len(iv.reg_frames) for iv in ivs))
    opts.update(dict(m.opts))
    return opts


def register(a, iv, m):
    if iv.new_strings:
        assert a.register_strings(iv.new_strings) == len(iv.w.strings) - len(iv.new_strings)
    if len(iv.new_frames):
        a.register_frames(iv.new_frames)
    if iv.new_labelsets:
        a.register_labelsets(iv.new_labelsets)
    if m.registered and len(iv.reg_offsets) > 1:
        a.register_stacks(iv.reg_frames, iv.reg_offsets)


def compare(m, want, got):
    """None if the flushed bytes are right, else the reason"""
    try:
        if dict(m.opts).get("ipc_compression") == abi.PA_IPC_LZ4_FRAME_GPU:
            if len(want) < (4 << 20):
                check_stream(got, want)
            else:
                check_buffers(got, want, python_decoder=False)
        elif got != want:
            return "bytes differ"
    except AssertionError as e:
        return "GPU-LZ4 stream differs from the plain one: %s" % e
    return None


def fresh_verdict(gpu, m, ivs, k, opts):
    """the interval through a fresh aggregator that registered the same registry at once"""
    from oracle import oracle_py
    iv = ivs[k]
    w = as_mode(iv.w, m)
    a = gpu.Aggregator(**dict(opts, max_samples=max(w.n, 1), max_frames=opts["max_frames"] if m.registered else max(w.n_frame_ids, 1)))
    try:
        for j in range(k + 1):
            register(a, ivs[j], m)
        gpu.load(a, w, stack_of_row=iv.stack_of_row if m.registered else None)
        bad = compare(m, oracle_py.run(w)[0], a.flush().ipc_bytes())
    finally:
        a.close()
    if bad:
        return "a fresh aggregator fed only this interval differs too: the bug is in this batch alone"
    return "a fresh aggregator fed only this interval matches the oracle: the difference is state carried from earlier intervals"


def run_lifetime(gpu, sms, m):
    ivs = sequence(sms)
    ref = oracle_lifetime(sms, m.hash_mode, m.schema)
    blobs = request_blobs(sms) if m.schema == V1 else None
    opts = agg_options(m, ivs, m.world)
    aggs = [gpu.Aggregator(**opts) for _ in range(m.world)]
    g = gpu.MergeGroup.local(aggs) if m.world > 1 else None
    records = {}
    try:
        for k, iv in enumerate(ivs):
            for a in aggs:
                register(a, iv, m)
            w = as_mode(iv.w, m)
            if g:
                for a, p in zip(aggs, thirds(w)):
                    gpu.load(a, p)
                res = g.flush()
            else:
                gpu.load(aggs[0], w, stack_of_row=iv.stack_of_row if m.registered else None)
                res = aggs[0].flush()
            got = res.ipc_bytes()
            want, st, want_req = ref[k]
            bad = compare(m, want, got)
            if bad:
                msg = "interval %s (%d rows): %s" % (iv.name, w.n, bad)
                if compare(Mode(), want, got):  # the plain streams: name the first differing column and row
                    msg += "; " + str(se.mismatch(w, want, got, sms, spans(w, m.world)))
                raise AssertionError(msg + "; " + fresh_verdict(gpu, m, ivs, k, opts))
            se.assert_counts(w, res, st)
            records[iv.name] = got
            if iv.name == "h" and ref[NAMES.index("c")][0] == want:
                assert got == records["c"], "interval h repeats c and the oracle's bytes agree, but the flushed bytes do not"
            if blobs is not None:
                r = g.stacktraces(blobs[k]) if g else aggs[0].stacktraces(blobs[k])
                got_req = r.ipc_bytes()
                if got_req != want_req:
                    d = pyref.diff(pyref.extract_stacktraces(want_req), pyref.extract_stacktraces(got_req)) if want_req and got_req else None
                    raise AssertionError("stacktrace request after interval %s (%d ids) differs: %s" % (iv.name, len(blobs[k]) // 16, d))
                assert r.n_rows == len(blobs[k]) // 16
    finally:
        if g:
            g.close()
        for a in aggs:
            a.close()


@pytest.mark.gpu
def test_plan_on_this_device(sms):
    """the self-checks above for the SM count of the device the lifetimes run on"""
    p = (sequence(sms), sms)
    check_table_predictions(*p)
    check_label_columns(*p)
    check_kind_orders(*p)
    check_store_crossings(*p)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", list(MODES))
def test_lifetime(gpu, sms, mode, monkeypatch):
    m = MODES[mode]
    for k, v in m.env:
        monkeypatch.setenv(k, v)
    run_lifetime(gpu, sms, m)
