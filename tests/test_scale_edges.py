"""Adversarial batches at the sizes where one warp of the run-end, header and hash passes handles several 32-row tiles.

The small edge batches (null label values, empty comm, every sample kind, provided-id collisions, 0-frame stacks) never
reach the multi-tile code of these passes, and the large batches are uniform. Here a plain-Python model of each pass's
row partition places every adversarial feature at a warp-range, iteration, sub-step or tile border of the default
kernels, and the GPU output must equal the oracle's byte for byte. The placement self-checks run without a GPU, for two
SM counts, so it is visible on any machine that the cases reach those borders.
"""
import dataclasses
import functools

import numpy as np
import pyarrow as pa
import pyarrow.compute as pc
import pytest

import pyref
from parca_agent_b200 import abi, synth

# ---- the partition model ---------------------------------------------------------------------------------------------
REE_BLOCKS_PER_SM = 8  # agg.cu pass_labels_count / pass_labels_emit: grid sms * ree_blocks (default 8) x column groups
WARPS_PER_BLOCK = 8    # kernels.cuh kWarps = kThreads / 32
REE_STEP = 32          # rows per sub-step of ree_single (four per iteration, kReeUnroll) and per step of ree_kinds
REE_ITER = 128         # rows per iteration of ree_single
HDR_BLOCKS_PER_SM = 8  # kernels.cuh kHdrBlocksPerSm (agg.cu launch_header)
HASH_WARPS = 24        # k_hash_insert_tma<24, 2, 8>, the default hash kernel (agg.cu launch_hash, tma_grid(24))
TILE = 32


def ree_warps(sms):
    return sms * REE_BLOCKS_PER_SM * WARPS_PER_BLOCK


def ree_per(n, sms):
    """warp_range (kernels.cuh): per = roundup32(ceil(n / warps))"""
    nw = ree_warps(sms)
    return (-(-n // nw) + 31) // 32 * 32


def ree_ranges(n, sms):
    """[begin, end) of every warp of k_ree_col (warp_range, kernels.cuh; grid agg.cu pass_labels_count)."""
    per = ree_per(n, sms)
    b = np.minimum(np.arange(ree_warps(sms), dtype=np.int64) * per, n)
    return b, np.minimum(b + per, n), per


def ree_place(row, n, sms):
    """(warp, iteration, sub-step) of a row in the run-end passes; ranges start on multiples of 32"""
    per = ree_per(n, sms)
    w, off = divmod(row, per)
    return w, off // REE_ITER, off % REE_ITER // REE_STEP


def header_warps(span, sms):
    """k_header grid (agg.cu launch_header): min(ceil(rows / 256), sms * 8) blocks of 8 warps"""
    return max(1, min(-(-span // (WARPS_PER_BLOCK * 32)), sms * HDR_BLOCKS_PER_SM)) * WARPS_PER_BLOCK


def hash_warps(span, sms):
    """k_hash_insert_tma<24, 2, 8> grid (agg.cu launch_hash): min(ceil(rows / 768), sms) blocks of 24 warps"""
    return max(1, min(-(-span // (HASH_WARPS * 32)), sms)) * HASH_WARPS


def tile_place(row, r0, nwarps):
    """(warp, index among the warp's tiles) of a row when tiles warp, warp + nwarps, ... of a launch over rows r0.. go to
    one warp (k_header, k_hash_insert_tma)"""
    t = (row - r0) // TILE
    return t % nwarps, t // nwarps


def locate(row, parts, sms):
    """Where the row falls in every pass, for failure messages (parts: the launch row spans, one per shard)."""
    for p0, p1 in parts:
        if p0 <= row < p1:
            m, r = p1 - p0, row - p0
            w, it, sub = ree_place(r, m, sms)
            hw, hk = tile_place(r, 0, header_warps(m, sms))
            xw, xk = tile_place(r, 0, hash_warps(m, sms))
            return ("shard rows %d..%d, local row %d: run-end warp %d (per %d) iteration %d sub-step %d; header warp %d tile %d; "
                    "hash warp %d tile %d" % (p0, p1, r, w, ree_per(m, sms), it, sub, hw, hk, xw, xk))
    return "row %d outside the batch" % row


def n_for_per(per, sms):
    """a batch size whose run-end ranges hold `per` rows, with a partial last range"""
    n = per * ree_warps(sms) - 13
    assert ree_per(n, sms) == per
    return n


# ---- the generator -----------------------------------------------------------------------------------------------------
DEEP_DEPTHS = [31, 32, 33, 63, 64, 65, 95, 96, 97, 255, 256, 257]  # around the 32-id (8-stripe) batch of the hash kernel
HUGE_DEPTH = 1500
N_BG, N_SHALLOW = 3000, 200
BORDER_OFFSETS = (-1, 0, 32, 64, 96, 128)  # from a range's first row; plus its last row
# job value per labelset: None, batch, None, None, None, x*300, None, batch, job-8 (labelsets 6 and 7 are first/last only)
LS_SEQ = [1, 0, 2, 5, 8, 1, 4, 3, 5, 0, 8]
KIND_SEQ = [0, 4, 1, 3, 6, 0, 5, 2, 4, 1, 6]
CPU_SEQ = [0, 65535, 1, 0, 65534, 65535, 2]
TID_SEQ = [0, 0xFFFFFFFF, 1, 0, 65536, 0xFFFFFFFF, 7]
T0 = 1_700_000_000_000_000_000
TS_SEQ = [T0, T0 + (1 << 32), -5, -5 + (1 << 40), T0 + (1 << 32), T0, -(1 << 62), T0 + (7 << 32)]
STACK_SEQ = [5, 0, 1, 2, 7, 9, 11, 53, 54]  # 0: all-zero id, 1: hi == 0, 2: lo == 0, 53 / 54: one provided id


def _runs(rng, n, mean, choices, p=None):
    start = rng.random(n) < 1.0 / mean
    start[0] = True
    rid = np.cumsum(start) - 1
    return np.asarray(choices)[rng.choice(len(choices), int(rid[-1]) + 1, p=p)][rid]


def _paint(col, starts, stop, vals):
    """col[starts[i]:starts[i + 1]] = vals[i % len(vals)], the last segment ending at stop"""
    starts = np.asarray(starts, dtype=np.int64)
    col[starts[0]:stop] = np.repeat(np.resize(np.asarray(vals, dtype=col.dtype), len(starts)), np.diff(np.append(starts, stop)))


def _excl_cumsum(x):
    out = np.zeros(len(x), dtype=np.int64)
    np.cumsum(x[:-1], out=out[1:])
    return out


def feature_groups(nwe, margin):
    """warps whose range borders carry the run-end features: the first, middle and last non-empty ranges (`margin` ranges
    in from the ends of a shard, whose borders carry the shard-border features)"""
    m = margin
    return [[m, m + 1, m + 2], [nwe // 2, nwe // 2 + 1, nwe // 2 + 2], [nwe - 3 - m, nwe - 2 - m, nwe - 1 - m]]


def scale_batch(n, sms, seed=1, parts=None, external=False):
    """An n-row batch with the frames, strings and labelsets of synth.edge_workload. `parts` are the row spans of the
    launches (one per shard of a merge group; default the whole batch); every feature is placed with the model of the
    span it falls in. Returned with provided-hash ids; use dataclasses.replace for the hash mode, schema and flags."""
    parts = parts or [(0, n)]
    margin = 3 if len(parts) > 1 else 0
    rng = np.random.Generator(np.random.PCG64(seed))
    base = synth.edge_workload(seed=seed, n=1, external=external)
    st = synth.StringTable()
    st.strings, st.index = list(base.strings), {s: i for i, s in enumerate(base.strings)}
    name = {k: st.sid(k) for k in ["comm", "node", "job", "zone", "first_only", "last_only"]}
    by_name = lambda pairs: sorted(pairs, key=lambda kv: st.strings[kv[0]])  # noqa: E731
    labelsets = list(base.labelsets) + [
        by_name([(name["first_only"], st.sid("row-zero")), (name["node"], st.sid("node-0"))]),
        by_name([(name["last_only"], st.sid("tail")), (name["job"], st.sid("batch"))]),
        by_name([(name["comm"], st.sid("svc-c")), (name["job"], st.sid("job-8")), (name["node"], st.sid("node-1")),
                 (name["zone"], st.sid("eu-west-1"))]),
    ]
    c_main, c_worker, c_gc = st.sid("main"), st.sid("worker"), st.sid("GC Thread#0")
    comm_seq = [c_main, 0, 0, c_worker, c_gc, 0, c_main, c_worker, 0]

    # stack pool: background 0..12 frames, shallow 0..3 frames (stack N_BG has none), deep around the batch border, one huge
    P = len(base.frames)
    depth = np.concatenate([rng.integers(0, 13, N_BG), rng.integers(0, 4, N_SHALLOW), np.repeat(DEEP_DEPTHS, 4), [HUGE_DEPTH]])
    depth[N_BG] = 0
    sh0, dp0, huge = N_BG, N_BG + N_SHALLOW, len(depth) - 1
    n_deep = 4 * len(DEEP_DEPTHS)
    pstart = _excl_cumsum(depth)
    pool = rng.integers(0, P, int(depth.sum()), dtype=np.uint64)
    ix = np.arange(len(depth), dtype=np.uint64)
    id_hi, id_lo = synth.splitmix64(ix + np.uint64(seed << 20)), synth.splitmix64(ix ^ np.uint64(0xD1B54A32D192ED03))
    id_hi[0] = id_lo[0] = 0
    id_hi[1] = 0
    id_lo[2] = 0
    coll = np.arange(3, N_BG - 1, 50)  # provided-id collisions: stack s carries the id of stack s + 1 (other frames)
    id_hi[coll], id_lo[coll] = id_hi[coll + 1], id_lo[coll + 1]

    ls = _runs(rng, n, 40, [0, 1, 2, 3, 4, 5, 8]).astype(np.uint32)
    comm = _runs(rng, n, 25, [c_main, c_worker, 0, c_gc]).astype(np.uint32)
    kind = _runs(rng, n, 3000, np.arange(7), p=[0.5, 0.1, 0.2, 0.05, 0.05, 0.05, 0.05]).astype(np.uint8)
    cpu = _runs(rng, n, 30, [0, 1, 2, 3, 65535]).astype(np.uint32)
    tid = _runs(rng, n, 30, [0, 1, 4242, 65536, 0xFFFFFFFF]).astype(np.uint32)
    ts = T0 + np.arange(n, dtype=np.int64) // 3 * 1000
    choice = _runs(rng, n, 3, np.arange(N_BG)).astype(np.int64)

    for p0, p1 in parts:
        m = p1 - p0
        b, e, per = ree_ranges(m, sms)
        b, e = b + p0, e + p0
        nw = int(np.sum(b < e))  # non-empty ranges
        for gi, g in enumerate(feature_groups(nw, margin)):
            q = {int(e[w]) - 1 for w in g} | {int(b[w]) + o for w in g for o in BORDER_OFFSETS if p0 <= b[w] + o < e[w]}
            q = sorted(q)
            stop = int(e[g[-1]])
            lead = q[0] > p0  # one row before the first border with the value that precedes the first one in the cycle
            for c, seq in ((ls, LS_SEQ), (comm, comm_seq), (kind, KIND_SEQ), (cpu, CPU_SEQ), (tid, TID_SEQ), (ts, TS_SEQ), (choice, STACK_SEQ)):
                seq = np.roll(seq, -3 * gi)
                _paint(c, [q[0] - 1] + q if lead else q, stop, np.roll(seq, 1) if lead else seq)
        w = nw // 4  # one labelset run over three whole ranges, one kind over four
        ls[b[w] - 5:e[w + 2] + 5] = 1
        kind[b[w] - 7:e[w + 3] + 7] = abi.PA_KIND_CPU
        ts[b[w] - 5:e[w + 2] + 5] = T0 - 1  # and one timestamp (v1: one int64 run over three ranges)
        choice[b[w + 1] - 2:b[w + 1] + 2] = 7
        r = int(e[nw // 3])  # nulls on both sides of a range border; kinds >= 3 (null temporality) over 100 rows
        ls[r - 20:r + 20] = 4
        comm[r - 20:r + 20] = 0
        kind[r - 50:r + 50] = abi.PA_KIND_MEM_ALLOC_OBJECTS
        # three sub-steps of 31, 31 and 32 run starts (alternating null / non-null): whatever the run index they start at,
        # the validity bits of one of them span two 32-bit words
        r = int(b[nw // 3 + 5])
        alt = np.arange(96) % 2 == 1
        alt[[5, 37]] = False
        comm[r - 1], ls[r - 1] = c_worker, 5
        comm[r:r + 96] = np.where(alt, 0, c_main)
        ls[r:r + 96] = np.where(alt, 4, 1)
        # hash kernel: tiles of 0..3-frame stacks (no whole 4-id stripe: the producer skips them) between deep tiles
        T, nwh = -(-m // TILE), hash_warps(m, sms)
        t = np.arange(T)
        hw, k = t % nwh, t // nwh
        M = (T - hw + nwh - 1) // nwh
        cls = hw % 16
        shallow = (((cls == 3) & (k % 2 == 1)) | ((cls == 7) & ((k == 0) | (k == M - 1) | (k % 3 == 2)))
                   | ((cls == 11) & np.isin(k % 4, (1, 2))))
        deep = np.isin(cls, (3, 7, 11)) & ~shallow
        tile_rows = lambda ts_, lanes: (p0 + ts_[:, None] * TILE + np.asarray(lanes)[None, :]).ravel()  # noqa: E731
        rows = tile_rows(t[shallow], np.arange(TILE))
        rows = rows[rows < p1]
        choice[rows] = sh0 + rng.integers(0, N_SHALLOW, len(rows))
        rows = tile_rows(t[deep], [0, 17])
        rows = rows[rows < p1]
        choice[rows] = dp0 + np.arange(len(rows)) % n_deep
        ht = t[(cls == 13) & (k == M // 2) & ((t + 1) * TILE <= m)]  # one >1000-frame stack among 0-frame ones
        choice[tile_rows(ht, np.arange(TILE))] = sh0
        choice[tile_rows(ht, [5])] = huge

    for s in [p0 for p0, _ in parts[1:]][:1]:  # first shard border: in a long labelset run, on a null comm, at a kind change
        ls[s - 100:s + 100] = 1
        comm[s] = 0
        kind[s - 30:s], kind[s:s + 30] = abi.PA_KIND_CPU, abi.PA_KIND_CUDA
        ts[s - 10:s + 10] = T0
        choice[s - 3:s + 3] = 5
    for s in [p0 for p0, _ in parts[2:]][:1]:  # second: a null labelset row in a long comm run, one row after a kind change
        comm[s - 100:s + 100] = c_main
        ls[s - 100:s + 100] = 1
        ls[s] = 4
        kind[s - 30:s - 1], kind[s - 1:s + 30] = abi.PA_KIND_CUDA, abi.PA_KIND_MEM_ALLOC_SPACE
    ls[0], ls[n - 4] = 6, 7  # a label name only in row 0, one only in the last 10 rows

    # frame stream: row i starts at an odd offset exactly when i is odd (one padding id where needed)
    nf = depth[choice]
    dense = _excl_cumsum(nf)
    par = (np.arange(n) - dense) & 1
    pad = np.zeros(n, dtype=np.int64)
    pad[:-1] = (par[1:] - par[:-1]) & 1
    off = dense + _excl_cumsum(pad)
    stream = np.zeros(int(off[-1] + nf[-1]), dtype=np.uint64)
    j = np.arange(int(nf.sum())) - np.repeat(dense, nf)
    stream[np.repeat(off, nf) + j] = pool[np.repeat(pstart[choice], nf) + j]

    hd = np.zeros(n, dtype=abi.HDR_DTYPE)
    hd["hash_hi"], hd["hash_lo"] = id_hi[choice], id_lo[choice]
    hd["timestamp_ns"] = ts
    hd["value"] = rng.integers(-5, 1 << 40, n)
    hd["pid"] = 10 + ls
    hd["tid"] = tid
    hd["comm_sid"] = comm
    hd["labelset_id"] = ls
    hd["cpu"] = cpu
    hd["kind"] = kind
    hd["nframes"] = nf
    hd["frame_off"] = off
    return synth.Workload("scale_edges_%d_sm%d" % (n, sms), st.strings, base.frames, labelsets, hd, _frame_ids=stream,
                          hash_mode=abi.PA_HASH_PROVIDED, external_labels=base.external_labels,
                          meta={"parts": parts, "sms": sms, "stack_choice": choice, "job": name["job"]})


def label_key(w, name_sid):
    """per-row value sid of a labelset-derived label column, -1 = null"""
    table = np.array([dict(s).get(name_sid, -1) for s in w.labelsets], dtype=np.int64)
    return table[w.hdrs["labelset_id"].astype(np.int64)]


def run_starts(key, null):
    """the boundary test of ree_single: row 0, a null row, a row after a null one, or a new key"""
    s = np.ones(len(key), dtype=bool)
    s[1:] = null[1:] | null[:-1] | (key[1:] != key[:-1])
    return s


def crossing_substeps(starts, p0, p1, min_starts):
    """sub-steps (32 rows from p0) with >= min_starts run starts whose validity bits span two 32-bit words"""
    idx = np.cumsum(starts)[p0:p1] - 1
    n32 = (p1 - p0) // 32 * 32
    s = starts[p0:p0 + n32].reshape(-1, 32)
    cnt = s.sum(1)
    first = idx[:n32].reshape(-1, 32)[np.arange(len(s)), s.argmax(1)]
    last = idx[:n32].reshape(-1, 32)[:, -1]
    return np.nonzero((cnt >= min_starts) & (first >> 5 != last >> 5))[0]


def part_of(w, p0, p1):
    """rows [p0, p1) of a batch as a workload of its own (frame stream sliced, offsets kept relative)"""
    h = w.hdrs[p0:p1].copy()
    f0 = int(h["frame_off"][0])
    f1 = int(h["frame_off"][-1] + h["nframes"][-1])
    h["frame_off"] -= np.uint64(f0)
    return dataclasses.replace(w, name=w.name + "[%d:%d]" % (p0, p1), hdrs=h, _frame_ids=w.frame_ids[f0:f1], meta=dict(w.meta))


def merge_parts(sms):
    """three shards of more than 32 rows per run-end warp each (so more than 270 336 rows on 132 SMs)"""
    s = 32 * ree_warps(sms)
    sizes = [s + 4099, s + 70_001, s + 1031]
    cut = np.cumsum([0] + sizes)
    return [(int(cut[i]), int(cut[i + 1])) for i in range(3)]


@functools.lru_cache(maxsize=2)
def batch(per, sms, external=False):
    return scale_batch(n_for_per(per, sms), sms, seed=per, external=external)


@functools.lru_cache(maxsize=1)
def merge_batch(sms):
    parts = merge_parts(sms)
    return scale_batch(parts[-1][1], sms, seed=3, parts=parts)


# ---- placement self-checks (no GPU) -------------------------------------------------------------------------------------
PERS = [64, 160, 288]  # half an iteration; one iteration and a 32-row tail; two iterations and a tail


def check_run_end_features(w, sms, p0, p1):
    h = w.hdrs
    m = p1 - p0
    b, e, per = ree_ranges(m, sms)
    nwe = int(np.sum(b < e))
    b, e = b[:nwe] + p0, e[:nwe] + p0
    job = label_key(w, w.meta["job"])
    jnull = job < 0
    comm = h["comm_sid"].astype(np.int64)
    cnull = comm == 0
    kind = h["kind"].astype(np.int64)
    js, cs = run_starts(job, jnull), run_starts(comm, cnull)
    ks = run_starts(kind, kind >= 3)
    seen = {}
    for g in feature_groups(nwe, 3 if len(w.meta["parts"]) > 1 else 0):
        for wi in g:
            for o in BORDER_OFFSETS + ("last",):
                p = int(e[wi]) - 1 if o == "last" else int(b[wi]) + o
                if not (p0 < p < e[wi]) or (o != "last" and o >= per):
                    continue
                for cname, st, null in (("job", js, jnull), ("comm", cs, cnull), ("kind", ks, kind >= 3)):
                    assert st[p], (cname, o, p)
                    seen.setdefault((cname, o), set()).add((bool(null[p - 1]), bool(null[p])))
    for (cname, o), kinds in seen.items():  # a null / non-null transition falls exactly on every border class
        assert (True, False) in kinds or (False, True) in kinds, (cname, o, kinds)
    for cname, st, null in (("job", js, jnull), ("comm", cs, cnull)):
        assert {o for (c, o) in seen if c == cname} >= {o for o in BORDER_OFFSETS + ("last",) if o == "last" or o < per}
        assert any(null[e[i] - 1] and null[e[i]] for i in range(len(b) - 1)), cname  # consecutive nulls over a border
        assert len(crossing_substeps(st, p0, p1, 31)), cname
    ls = h["labelset_id"]
    chg = np.nonzero(np.diff(ls.astype(np.int64)) != 0)[0] + 1
    run_b, run_e = np.concatenate([[0], chg]), np.concatenate([chg, [len(ls)]])
    assert any(np.sum((b >= rb) & (e <= re) & (b < e)) >= 3 for rb, re in zip(run_b, run_e) if re - rb >= 3 * per)
    kchg = np.nonzero(np.diff(kind) != 0)[0] + 1
    kb, ke = np.concatenate([[p0], kchg[(kchg > p0) & (kchg < p1)]]), np.concatenate([kchg[(kchg > p0) & (kchg < p1)], [p1]])
    assert any(np.sum((b >= rb) & (e <= re) & (b < e)) >= 2 for rb, re in zip(kb, ke))  # one kind over whole ranges
    assert any(re - rb > 32 and kind[rb] >= 3 for rb, re in zip(kb, ke))  # null temporality longer than a sub-step
    ts = h["timestamp_ns"]
    assert any(ts[b[i] - 1] == ts[b[i]] for i in range(1, len(b)) if b[i] < e[i])  # repeated timestamps over a border
    ch = w.meta["stack_choice"]
    assert any(ch[b[i] - 1] == ch[b[i]] for i in range(1, len(b)) if b[i] < e[i])  # one stack over a border


def check_tile_features(w, sms, p0, p1):
    h = w.hdrs
    m = p1 - p0
    T, nwh = -(-m // TILE), hash_warps(m, sms)
    assert T >= 2 * nwh  # every hash warp owns several tiles
    if len(w.meta["parts"]) > 1:  # merge shards: too few tiles per warp for every skip pattern
        return
    assert T >= 2 * header_warps(m, sms) and T >= 4 * nwh
    nf = np.zeros(T * TILE, dtype=np.int64)
    nf[:m] = h["nframes"][p0:p1]
    nb = (nf.reshape(T, TILE) >> 2).max(1)
    shallow = nb == 0
    pat = {"sds": False, "sssd": False, "first": False, "last": False}
    for hw in range(nwh):
        s = shallow[hw::nwh]
        d = ~s
        pat["sds"] |= bool(np.any(d[:-2] & s[1:-1] & d[2:]))
        pat["sssd"] |= bool(np.any(d[:-3] & s[1:-2] & s[2:-1] & d[3:]))
        pat["first"] |= bool(s[0] and d.any())
        pat["last"] |= bool(s[-1] and d.any())
    assert all(pat.values()), pat
    tiles = nf[:T * TILE].reshape(T, TILE)
    assert np.any((tiles.max(1) > 1000) & ((tiles > 0).sum(1) == 1))  # one >1000-frame stack among empty ones
    assert set(DEEP_DEPTHS) <= set(np.unique(nf).tolist())


def check_batch(w, sms):
    h = w.hdrs
    n = w.n
    off = h["frame_off"].astype(np.int64)
    assert np.all(off % 2 == np.arange(n) % 2)  # every other stack starts at an odd frame offset
    assert np.all(off[1:] >= off[:-1] + h["nframes"][:-1]) and off[-1] + h["nframes"][-1] == w.n_frame_ids
    ls = h["labelset_id"]
    assert np.nonzero(ls == 6)[0].tolist() == [0]
    assert np.all(np.nonzero(ls == 7)[0] >= n - 10) and np.any(ls == 7)
    assert {0, 65535} <= set(np.unique(h["cpu"]).tolist()) and {0, 0xFFFFFFFF} <= set(np.unique(h["tid"]).tolist())
    ts = h["timestamp_ns"]
    assert np.any(ts < 0)
    d = ts[1:] ^ ts[:-1]
    assert np.any((d != 0) & (d & 0xFFFFFFFF == 0))  # neighbours that differ only in bits 32..63
    hi, lo = h["hash_hi"], h["hash_lo"]
    assert np.any((hi == 0) & (lo == 0)) and np.any((hi == 0) & (lo != 0)) and np.any((hi != 0) & (lo == 0))
    ch = w.meta["stack_choice"]
    c = np.arange(3, N_BG - 1, 50)
    assert np.any(np.isin(c, ch) & np.isin(c + 1, ch))  # one provided id, two different stacks
    for p0, p1 in w.meta["parts"]:
        check_run_end_features(w, sms, p0, p1)
        check_tile_features(w, sms, p0, p1)


@pytest.mark.parametrize("sms", [132, 114])
@pytest.mark.parametrize("per", PERS)
def test_features_land_where_the_model_says(per, sms):
    w = batch(per, sms)
    assert ree_per(w.n, sms) == per
    check_batch(w, sms)


@pytest.mark.parametrize("sms", [132, 114])
def test_merge_shard_borders(sms):
    w = merge_batch(sms)
    parts = w.meta["parts"]
    for p0, p1 in parts:
        assert p1 - p0 > 32 * ree_warps(sms) and ree_per(p1 - p0, sms) == 64
    check_batch(w, sms)
    h = w.hdrs
    job = label_key(w, w.meta["job"])
    s1, s2 = parts[1][0], parts[2][0]
    ls, comm, kind = h["labelset_id"], h["comm_sid"], h["kind"]
    assert np.all(ls[s1 - 100:s1 + 100] == ls[s1]) and comm[s1] == 0 and kind[s1 - 1] != kind[s1]
    assert job[s2] < 0 and np.all(comm[s2 - 100:s2 + 100] == comm[s2]) and kind[s2 - 2] != kind[s2 - 1] == kind[s2]


def test_model_restates_the_launch_arithmetic():
    """spot values of the partitions on a 132-SM H100 (the table of the run-end, header and hash passes)"""
    assert ree_warps(132) == 8448 and ree_per(270_336, 132) == 32 and ree_per(270_337, 132) == 64
    b, e, per = ree_ranges(1_000_000, 132)
    assert per == 128 and e[-1] == 1_000_000 and np.all(e - b <= per)
    assert header_warps(270_336, 132) == 8448 and header_warps(1000, 132) == 32
    assert hash_warps(101_376, 132) == 3168 and hash_warps(1000, 132) == 48
    assert tile_place(1000, 0, 48) == (31, 0) and tile_place(48 * 32 + 5, 0, 48) == (0, 1)
    assert ree_place(300, 1_000_000, 132) == (2, 0, 1)


# ---- the GPU cases -----------------------------------------------------------------------------------------------------
MODES = [abi.PA_HASH_PROVIDED, abi.PA_HASH_XXH64X2]


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


def first_bad_row(want, got):
    """(column, row) of the first row whose decoded value differs, None if the tables only differ elsewhere"""
    for name in want.schema.names:
        if name not in got.schema.names:
            return name, None
        a, b = want.column(name).combine_chunks(), got.column(name).combine_chunks()
        if a.equals(b):
            continue
        if pa.types.is_run_end_encoded(a.type):
            a, b = pc.run_end_decode(a), pc.run_end_decode(b)
        n = min(len(a), len(b))
        step = 1 << 12
        for s in range(0, n, step):
            if not a.slice(s, step).equals(b.slice(s, step)):
                x, y = a.slice(s, step).to_pylist(), b.slice(s, step).to_pylist()
                return name, s + next(i for i in range(len(x)) if i >= len(y) or x[i] != y[i])
        return name, n
    return None


def mismatch(w, want, got, sms, parts=None):
    v1 = w.schema == abi.PA_SCHEMA_V1
    msg = "IPC bytes differ (len %d vs %d)" % (len(want), len(got))
    if want and got:
        ta, tb = pa.ipc.open_stream(want).read_all(), pa.ipc.open_stream(got).read_all()
        ex = pyref.extract_v1 if v1 else pyref.extract
        msg += "; first logical difference: %s" % pyref.diff(ex(ta), ex(tb))
        bad = first_bad_row(ta, tb)
        if bad and bad[1] is not None:
            msg += "; column %s first differs at row %d, %s" % (bad[0], bad[1], locate(bad[1], parts or [(0, w.n)], sms))
        elif bad:
            msg += "; column %s is missing" % bad[0]
    return AssertionError(msg)


def assert_counts(w, r, st):
    assert r.n_rows == st["rows"] == w.n
    assert r.n_unique_stacks == st["unique_stacks"]
    if w.schema != abi.PA_SCHEMA_V1:
        assert (r.n_locations, r.n_functions) == (st["locations"], st["functions"])


def assert_same(oracle, gpu, w, sms, chunk_samples=None, **kw):
    """chunk_samples defaults to the whole batch: one header and one hash launch over all rows, as the model assumes"""
    want, st = oracle.run(w)
    got, r = gpu.run(w, chunk_samples=chunk_samples or w.n, **kw)
    if got != want:
        raise mismatch(w, want, got, sms)
    assert_counts(w, r, st)


@pytest.mark.gpu
def test_features_land_on_this_device(sms):
    """the placement self-checks for the SM count of the device the cases below run on"""
    for per in PERS:
        check_batch(batch(per, sms), sms)
    check_batch(merge_batch(sms), sms)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("per", PERS)
def test_v2(oracle, gpu, sms, per, mode):
    assert_same(oracle, gpu, dataclasses.replace(batch(per, sms), hash_mode=mode), sms)


@pytest.mark.gpu
@pytest.mark.parametrize("per,mode", [(160, abi.PA_HASH_PROVIDED), (288, abi.PA_HASH_XXH64X2)])
def test_v1_sample_and_stacktrace_records(oracle, gpu, sms, per, mode):
    w = dataclasses.replace(batch(per, sms), hash_mode=mode, schema=abi.PA_SCHEMA_V1)
    o = oracle.Oracle(w)
    a = gpu.from_workload(w, chunk_samples=w.n)
    try:
        o.ingest(w.hdrs, w.frame_ids)
        want, st = o.flush()
        gpu.load(a, w)
        r = a.flush()
        got = r.ipc_bytes()
        if got != want:
            raise mismatch(w, want, got, sms)
        assert_counts(w, r, st)
        ids = a.last_stack_ids(r.n_unique_stacks)
        ids = b"".join(bytes(x) for x in ids) + bytes(16)  # and the all-zero id again (known in provided mode)
        want, nloc = o.stacktraces(ids)
        r = a.stacktraces(ids)
        if r.ipc_bytes() != want:
            d = pyref.diff(pyref.extract_stacktraces(want), pyref.extract_stacktraces(r.ipc_bytes()))
            raise AssertionError("stacktrace record bytes differ: %s" % d)
        assert (r.n_rows, r.n_locations) == (len(ids) // 16, nloc)
    finally:
        a.close()
        o.close()


@pytest.mark.gpu
def test_narrow_ring(oracle, gpu, sms):
    assert_same(oracle, gpu, dataclasses.replace(batch(64, sms), hash_mode=abi.PA_HASH_XXH64X2), sms, frame_id_bytes=4)


@pytest.mark.gpu
@pytest.mark.parametrize("mode", MODES)
def test_chunk_borders_inside_tiles(oracle, gpu, sms, mode):
    """chunks of 100 003 rows: every chunk border falls inside a 32-row tile of the header and hash passes"""
    assert_same(oracle, gpu, dataclasses.replace(batch(160, sms), hash_mode=mode), sms, chunk_samples=100_003)


@pytest.mark.gpu
@pytest.mark.parametrize("flags", [7, 3])
def test_external_labels_and_label_flags(oracle, gpu, sms, flags):
    w = dataclasses.replace(batch(64, sms, external=True), hash_mode=abi.PA_HASH_XXH64X2, label_flags=flags)
    assert w.external_labels
    assert_same(oracle, gpu, w, sms)


@pytest.mark.gpu
def test_merge_group_of_three_shards(oracle, gpu, sms):
    w = dataclasses.replace(merge_batch(sms), hash_mode=abi.PA_HASH_XXH64X2)
    parts = w.meta["parts"]
    want, st = oracle.run(w)
    shards = [part_of(w, p0, p1) for p0, p1 in parts]
    aggs = [gpu.from_workload(p, chunk_samples=p.n) for p in shards]
    g = gpu.MergeGroup.local(aggs)
    try:
        for a, p in zip(aggs, shards):
            gpu.load(a, p)
        res = g.flush()
        got = res.ipc_bytes()
        if got != want:
            raise mismatch(w, want, got, sms, parts)
        assert_counts(w, res, st)
    finally:
        g.close()
        for a in aggs:
            a.close()
