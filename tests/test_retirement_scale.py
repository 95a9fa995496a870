"""Stack retirement (PA_CFG_RETIRE_STACKS, PA_CFG_GROUP_RETIRE) at registry scale: about a million slots, where the scans of idle
selection and of arena compaction run with many blocks.

retire_stacks selects idle slots through a bitmap, a popcount prefix over its words (WordsF) and an emit kernel that ranks each
slot against `cap`; compaction scans the slots (StackLiveF). Both scans use small_grid, so below 65 536 slots the prefix has a
single block. Here a plain-Python model of that launch geometry places idle slots, cap cuts and live stacks at word and block
borders, and the library must give the handles and counters of VecModel (a numpy restatement of test_stack_retirement's Model)
and the ring-mode stream of the same rows, byte for byte.

CPU tests: VecModel against Model, and the placement self-checks for two SM counts. GPU tests: idle selection across scan
blocks, grace / freeing / reuse at a million slots, compaction at StackLiveF block borders, record-array regrowth, idle
windows, and local PA_CFG_GROUP_RETIRE groups."""
import numpy as np
import pytest

from parca_agent_b200 import abi, lib, synth
from test_stack_retirement import Model, ring_workload

EINVAL = -22
REG, RETIRE = abi.PA_CFG_REGISTERED_STACKS, abi.PA_CFG_RETIRE_STACKS
GROUP = REG | abi.PA_CFG_GROUP_STACKS | abi.PA_CFG_GROUP_RETIRE
LIVE, RETIRING, FREE = 0, 1, 2
BIG = (1 << 20) + 1  # 32 769 bitmap words: 17 WordsF blocks, the last one a single word holding a single slot


class VecModel:
    """Model with per-slot arrays, for registries of a million slots. Handles come back as uint64 arrays."""

    def __init__(self, max_frames=None):
        self.state = np.zeros(0, np.uint8)
        self.gen, self.depth, self.last = (np.zeros(0, np.int64) for _ in range(3))
        self.retiring = []  # (slots, stage count at which they are freed)
        self.stages, self.frames_live, self.max_frames, self.retired = 0, 0, max_frames, 0

    def handles(self, slots):
        return self.gen[slots].astype(np.uint64) << np.uint64(32) | np.asarray(slots, np.uint64)

    def register(self, depths):
        depths = np.asarray(depths, np.int64)
        if self.max_frames is not None and self.frames_live + int(depths.sum()) > self.max_frames:
            return None
        free = np.flatnonzero(self.state == FREE)[:len(depths)]  # the lowest free slots, then new ones
        n0, k = len(self.state), len(depths) - len(free)
        self.state = np.concatenate([self.state, np.full(k, FREE, np.uint8)])
        self.gen, self.depth, self.last = (np.concatenate([x, np.zeros(k, np.int64)]) for x in (self.gen, self.depth, self.last))
        s = np.concatenate([free, np.arange(n0, n0 + k)]).astype(np.int64)
        self.state[s], self.depth[s], self.last[s] = LIVE, depths, self.stages
        self.frames_live += int(depths.sum())
        return self.handles(s)

    def stage(self):
        self.stages += 1
        for s, at in self.retiring:
            if at <= self.stages:
                self.state[s] = FREE
                self.gen[s] += 1
                self.frames_live -= int(self.depth[s].sum())
        self.retiring = [(s, at) for s, at in self.retiring if at > self.stages]

    def valid(self, handles):
        h = np.asarray(handles, np.uint64)
        s, g = (h & np.uint64(0xFFFFFFFF)).astype(np.int64), (h >> np.uint64(32)).astype(np.int64)
        ok = s < len(self.state)
        sc = np.where(ok, s, 0)
        return ok & (self.state[sc] != FREE) & (self.gen[sc] == g), s

    def batch(self, handles):
        ok, s = self.valid(handles)
        self.last[s[ok]] = self.stages
        return bool(ok.all())

    def retire(self, idle, cap=None):
        assert idle >= 1
        if self.stages < idle:
            return np.zeros(0, np.uint64)
        out = np.flatnonzero((self.state == LIVE) & (self.last <= self.stages - idle))
        out = out if cap is None else out[:cap]
        self.state[out] = RETIRING
        self.retiring.append((out, self.stages + 2))
        self.retired += len(out)
        return self.handles(out)

    def counters(self):
        live = int(np.sum(self.state != FREE))
        return {"stacks_live": live, "stacks_free": len(self.state) - live, "stack_frames_live": self.frames_live, "stacks_retired": self.retired}


# ---- CPU: VecModel against Model ---------------------------------------------------------------------------------------
def replay(ops, max_frames=None):
    """Run ops on Model and VecModel side by side; every result, counter and slot state must agree after every op."""
    m, v = Model(max_frames), VecModel(max_frames)
    for op in ops:
        if op[0] == "reg":
            a, b = m.register(op[1]), v.register(op[1])
            assert (a is None and b is None) or a == [int(x) for x in b], op
        elif op[0] == "stage":
            m.stage(); v.stage()
        elif op[0] == "batch":
            assert m.batch(op[1]) == v.batch(np.asarray(op[1], np.uint64)), op
        else:
            a, b = m.retire(op[1], op[2]), v.retire(op[1], op[2])
            assert a == [int(x) for x in b], op
        assert m.counters() == v.counters(), op
        assert list(v.state) == m.state and list(v.gen) == m.gen and list(v.last) == m.last, op
        assert sorted(m.free) == list(np.flatnonzero(v.state == FREE)), op
    return m, v


def test_vecmodel_on_the_hand_worked_sequences():
    """the three sequences of test_stack_retirement's model tests"""
    replay([("reg", [2, 3, 4]), ("retire", 1, None), ("stage",), ("batch", [0]), ("retire", 2, None), ("retire", 1, None),
            ("retire", 1, None), ("stage",), ("batch", [1, 2, 0]), ("retire", 1, None), ("retire", 2, None), ("stage",), ("batch", [1]),
            ("retire", 2, None), ("retire", 1, None)])
    g = 1 << 32
    replay([("reg", [1, 1, 1]), ("stage",), ("retire", 1, None), ("stage",), ("reg", [5]), ("stage",), ("reg", [7, 8]),
            ("batch", [0, g, g | 1, 2 * g]), ("stage",), ("stage",), ("retire", 2, None)])
    replay([("stage",), ("reg", [1]), ("retire", 1, None), ("stage",), ("retire", 1, None)])
    _, v = replay([("reg", [4, 4]), ("reg", [3]), ("stage",), ("retire", 1, 1), ("retire", 1, 5), ("reg", [3]), ("stage",), ("stage",),
                   ("reg", [10])], max_frames=10)
    assert v.frames_live == 10 and list(v.gen) == [1, 1]


def test_vecmodel_on_a_random_sequence():
    """about 2000 registrations, stages, batches (valid, retiring and stale handles) and retire calls with and without caps,
    with max_frames refusals"""
    rng = np.random.Generator(np.random.PCG64(17))
    m, v = Model(max_frames=1000), VecModel(max_frames=1000)
    issued, refused, retired = [], 0, 0
    for _ in range(2000):
        r = rng.random()
        if r < 0.3:
            d = [int(x) for x in rng.integers(0, 40, int(rng.integers(1, 12)))]
            a, b = m.register(d), v.register(d)
            assert (a is None) == (b is None)
            if a is None:
                refused += 1
            else:
                assert a == [int(x) for x in b]
                issued += a
        elif r < 0.5:
            m.stage(); v.stage()
        elif r < 0.8 and issued:
            hs = [issued[int(i)] for i in rng.integers(0, len(issued), int(rng.integers(1, 20)))]
            if rng.random() < 0.2:
                hs.append(int(rng.integers(0, 1 << 34)))  # a handle nothing was registered as
            assert m.batch(hs) == v.batch(np.asarray(hs, np.uint64))
        else:
            idle, cap = int(rng.integers(1, 4)), (None if rng.random() < 0.5 else int(rng.integers(0, 30)))
            a = m.retire(idle, cap)
            assert a == [int(x) for x in v.retire(idle, cap)]
            retired += len(a)
        assert m.counters() == v.counters()
        assert list(v.state) == m.state and list(v.gen) == m.gen and list(v.last) == m.last
    assert refused > 20 and retired > 200 and max(v.gen) >= 2


# ---- the launch-geometry model -----------------------------------------------------------------------------------------
THREADS = 256         # kernels.cuh kThreads; block_range rounds each block's span up to a multiple of it
SMALL_GRID_PER = 2048  # agg.cu small_grid: at least 2048 elements per block
BLOCKS_PER_SM = 4     # agg.cu pa_agg_create: G = 4 * SMs, the most blocks small_grid gives


def small_grid(bound, sms):
    return max(1, min(BLOCKS_PER_SM * sms, -(-bound // SMALL_GRID_PER)))


def block_spans(n, grid):
    """[begin, end) of every non-empty block of a scan over n elements (kernels.cuh block_range)"""
    per = -(-n // grid)
    per = -(-per // THREADS) * THREADS
    return [(b * per, min(b * per + per, n)) for b in range(grid) if b * per < n]


def words_blocks(ns, sms):
    """slot spans of the WordsF blocks of retire_stacks (agg.cu: the scan over nw = ceil(ns / 32) bitmap words)"""
    nw = -(-ns // 32)
    return [(32 * b, min(32 * e, ns)) for b, e in block_spans(nw, small_grid(nw, sms))]


def live_blocks(ns, sms):
    """slot spans of the StackLiveF blocks of a compaction (agg.cu rs_upload: the scan over the uploaded slots)"""
    return block_spans(ns, small_grid(ns, sms))


def block_of(slots, blocks):
    return np.searchsorted(np.asarray([b for b, _ in blocks]), slots, side="right") - 1


def idle_plan(ns, sms, seed=3):
    """The slots the first batch of test_idle_selection_across_scan_blocks leaves idle: slot 0 alone in word 0, words 1 and 2 with
    none, word 3 whole, both sides of every WordsF block border, the last word of block 0 and a word of a middle block whole, the
    lone slot of the last word, and a sparse random sprinkle (partial words everywhere)."""
    blocks = words_blocks(ns, sms)
    rng = np.random.Generator(np.random.PCG64(seed))
    idle = np.zeros(ns, bool)
    idle[rng.choice(ns, ns // 500, replace=False)] = True
    idle[:128] = False
    idle[0] = idle[ns - 1] = True
    idle[96:128] = True
    b1, mid = blocks[1][0], blocks[len(blocks) // 2][0]
    idle[b1 - 32:b1] = True
    idle[mid + 64:mid + 96] = True
    idle[b1 + 32:b1 + 96] = False
    for b, _ in blocks[1:]:
        idle[b - 1] = idle[b] = True
    return np.flatnonzero(idle)


def cap_plan(idle, blocks):
    """Caps of successive retire calls, each selecting from what the previous ones left, and the cumulative cut each is meant
    to reach: 1, 31, 32, 33; block 0's idle count -1 / exact / +1; the exact end of block 8; one into block 13; all but the last.
    A cap of 0 comes first and a cap above the idle count (one slot left) last."""
    blk = block_of(idle, blocks)
    r0 = int(np.sum(blk == 0))
    cuts = [1, 32, 64, 97, r0 - 1, r0, r0 + 1, int(np.sum(blk <= 8)), int(np.sum(blk <= 12)) + 1, len(idle) - 1]
    return [0] + [int(x) for x in np.diff([0] + cuts)] + [7], cuts


def live_plan(ns, sms, seed=5):
    """test_compaction_at_live_scan_block_borders: the stacks that stay live (both sides of every StackLiveF block border, a 2 %
    sprinkle, slot 0) with the two slots beyond each retired, and the two 65535-id stacks (the last slot of a block, slot ns - 1)."""
    blocks = live_blocks(ns, sms)
    rng = np.random.Generator(np.random.PCG64(seed))
    live = np.zeros(ns, bool)
    live[rng.choice(ns, ns // 50, replace=False)] = True
    live[0] = True
    for b, _ in blocks[1:]:
        for o, v in zip(range(-3, 3), (False, False, True, True, False, False)):
            if b + o < ns:
                live[b + o] = v
    deep = [blocks[len(blocks) // 3][1] - 1, ns - 1]
    live[deep] = True
    return np.flatnonzero(live), deep


@pytest.mark.parametrize("sms", [132, 114])
def test_patterns_land_where_the_model_says(sms):
    wb = words_blocks(BIG, sms)
    assert len(wb) == 17 >= 16 and wb[-1] == (1 << 20, BIG)  # the 17th block: one word, one slot
    lb = live_blocks(BIG, sms)
    assert len(lb) >= 400 and lb[-1][1] == BIG
    idle = idle_plan(BIG, sms)
    iset = set(idle.tolist())
    assert {0, BIG - 1} <= iset and all({b - 1, b} <= iset for b, _ in wb[1:])
    assert set(range(96, 128)) <= iset and not iset & set(range(1, 96))  # a whole word, and words with none
    b1 = wb[1][0]
    assert set(range(b1 - 32, b1)) <= iset and not iset & set(range(b1 + 32, b1 + 96))
    caps, cuts = cap_plan(idle, wb)
    assert caps[0] == 0 and caps[1:5] == [1, 31, 32, 33] and all(c >= 1 for c in caps[1:]) and caps[-1] > 1
    blk = block_of(idle, wb)
    r0 = int(np.sum(blk == 0))
    assert idle[0] == 0 and idle[1] == 96  # cut 1: slot 0 retired, the next idle slot starts a word
    assert idle[r0 - 1] == b1 - 1 and idle[r0] == b1  # cut r0: exactly at the WordsF block border, one before and one after
    assert blk[cuts[4] - 1] == 0 and blk[cuts[6] - 1] == 1
    assert blk[cuts[7] - 1] == 8 and blk[cuts[7]] == 9 and blk[cuts[8] - 1] == 13
    assert idle[-1] == BIG - 1 and blk[-1] == 16 and cuts[-1] == len(idle) - 1  # the last call takes the lone slot of the last word
    assert np.all(np.diff(cuts) > 0)
    live, deep = live_plan(BIG, sms)
    lset = set(live.tolist())
    assert deep[0] + 1 == lb[len(lb) // 3 + 1][0] and deep[1] == BIG - 1 and set(deep) <= lset
    assert all(b - 1 in lset and b in lset and not {b - 3, b - 2, b + 1, b + 2} & lset for b, _ in lb[1:])
    assert len(words_blocks(300_001, sms)) == 5  # test_group_retire_at_scale's smaller group


def test_geometry_spot_values():
    """the partition on a 132-SM H100 (G = 528) and a 114-SM one (G = 456)"""
    assert small_grid(32769, 132) == 17 and small_grid(BIG, 132) == 513 and small_grid(BIG, 114) == 456
    assert block_spans(32769, 17)[0] == (0, 2048) and block_spans(32769, 17)[-1] == (32768, 32769)
    assert live_blocks(BIG, 132)[-1] == (512 * 2048, BIG) and live_blocks(BIG, 114)[-1] == (455 * 2304, BIG)
    assert words_blocks(65536, 132) == [(0, 65536)] and len(words_blocks(65537, 132)) == 2  # one block up to 2048 words
    assert words_blocks(300_001, 132)[-1] == (4 * 65536, 300_001)


# ---- GPU ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    lib.lib()
    return lib


@pytest.fixture(scope="module")
def sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


MODES = [(abi.PA_HASH_PROVIDED, 8), (abi.PA_HASH_XXH64X2, 4)]  # (hash mode, frame id bytes)


def base(mode):
    """strings, frames, labelsets and a pool of row headers"""
    return synth.ragged(n=20_000, u=2_000, p=8_192, max_depth=8, hash_mode=mode)


def form(w, n, seed, deep=()):
    """n stacks of 0..8 frame ids of w (stacks `deep` have 65535), random provided ids"""
    rng = np.random.Generator(np.random.PCG64(seed))
    depth = rng.integers(0, 9, n)
    depth[list(deep)] = 65535
    offsets = np.zeros(n + 1, np.uint64)
    offsets[1:] = np.cumsum(depth)
    frames = rng.integers(0, len(w.frames), int(offsets[-1]), dtype=np.uint64)
    return lib.StackForm(rng.integers(1, 1 << 63, (n, 2), dtype=np.uint64), frames, offsets, None)


def span(sf, lo, hi):
    """(frames, offsets, hashes) of stacks lo..hi of the form, for one register call"""
    o = sf.offsets[lo:hi + 1]
    return sf.frames[int(o[0]):int(o[-1])], o - o[0], sf.hashes[lo:hi]


def same(got, want, what):
    got, want = np.asarray(got, np.uint64), np.asarray(want, np.uint64)
    if not np.array_equal(got, want):
        n = min(len(got), len(want))
        i = int(np.argmax(got[:n] != want[:n])) if n and np.any(got[:n] != want[:n]) else n
        raise AssertionError("%s: %d handles, want %d; first difference at %d: %s, want %s" % (
            what, len(got), len(want), i, hex(int(got[i])) if i < len(got) else None, hex(int(want[i])) if i < len(want) else None))


class Registry:
    """One PA_CFG_RETIRE_STACKS aggregator, a ring-mode aggregator and VecModel, fed the same registrations and rows. `handle`
    maps each stack of the form to the handle it was last registered under."""

    def __init__(self, w, sf, max_samples, max_frames, ring_frames, idb, seed=9):
        self.w, self.sf = w, sf
        self.depth = np.diff(sf.offsets.astype(np.int64))
        kw = dict(frame_id_bytes=idb)
        self.a = lib.from_workload(w.head(0), max_samples=max_samples, max_frames=max_frames, flags=REG | RETIRE, **kw)
        self.ring = lib.from_workload(w.head(0), max_samples=max_samples, max_frames=ring_frames, **kw)
        self.m = VecModel(max_frames)
        self.handle = np.zeros(len(sf.hashes), np.uint64)
        self.rng = np.random.Generator(np.random.PCG64(seed))

    def register(self, lo, hi):
        fr, o, hs = span(self.sf, lo, hi)
        got = self.a.register_stack_handles(fr, o, hs if self.w.hash_mode == abi.PA_HASH_PROVIDED else None)
        same(got, self.m.register(self.depth[lo:hi]), "registration of stacks %d..%d" % (lo, hi))
        self.handle[lo:hi] = got
        return got

    def hdrs(self, n):
        return np.array(self.w.hdrs[self.rng.integers(0, self.w.n, n)], copy=True)

    def load(self, a, hdrs, handles):
        hv, _, _ = a.acquire(len(hdrs), 0)
        hv[:] = hdrs
        hv["frame_off"] = handles
        a.commit(len(hdrs))

    def ring_bytes(self, hdrs, stacks, oracle=None):
        rw = ring_workload(self.w, self.sf, hdrs, stacks)
        lib.load(self.ring, rw)
        want = self.ring.flush().ipc_bytes()
        if oracle is not None:
            assert oracle.run(rw)[0] == want, "the ring mode differs from the oracle"
        return want

    def flush(self, stacks, handles=None, oracle=None, what=""):
        """rows naming `stacks` of the form, by `handles` (default: their current ones); the stream must be the ring mode's"""
        stacks = np.asarray(stacks, np.int64)
        handles = self.handle[stacks] if handles is None else np.asarray(handles, np.uint64)
        hdrs = self.hdrs(len(stacks))
        self.load(self.a, hdrs, handles)
        self.m.stage()
        assert self.m.batch(handles)
        got = self.a.flush().ipc_bytes()
        assert got == self.ring_bytes(hdrs, stacks, oracle), "%s: the stream differs from the ring mode" % what

    def retire(self, idle, cap=None, what=""):
        got = self.a.retire_stacks(idle, cap)
        same(got, self.m.retire(idle, cap), "%s retire(%d, %s)" % (what, idle, cap))
        self.check()
        return got

    def check(self):
        c = self.a.stack_counters()
        want = self.m.counters()
        assert {k: c[k] for k in want} == want
        return c

    def close(self):
        self.a.close(); self.ring.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode,idb", MODES)
def test_idle_selection_across_scan_blocks(oracle, gpu, sms, mode, idb):
    """2^20 + 1 slots (17 WordsF blocks): one batch leaves the idle_plan slots idle; then retire calls whose caps cut at word
    borders, at block 0's border -1 / exact / +1, in later blocks, and at the lone slot of the last word"""
    w = base(mode)
    sf = form(w, BIG, seed=1)
    r = Registry(w, sf, BIG, int(sf.offsets[-1]) + 1, int(sf.offsets[-1]) + 1, idb)
    for lo, hi in ((0, 300_000), (300_000, 700_001), (700_001, 1_000_000), (1_000_000, BIG)):
        r.register(lo, hi)
    blocks = words_blocks(BIG, sms)
    idle = idle_plan(BIG, sms)
    named = np.setdiff1d(np.arange(BIG), idle)
    r.flush(r.rng.permutation(named), oracle=oracle, what="the batch that leaves the plan idle")
    caps, cuts = cap_plan(idle, blocks)
    done = 0
    for cap in caps:
        got = r.retire(1, cap)
        assert len(got) == min(cap, len(idle) - done)
        same(got & np.uint64(0xFFFFFFFF), idle[done:done + len(got)], "cap %d after %d" % (cap, done))
        done += len(got)
    assert done == len(idle) and len(r.retire(1)) == 0
    c = r.check()
    assert c["stacks_retired"] == len(idle) and r.m.state[BIG - 1] == RETIRING
    r.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode,idb", MODES)
def test_grace_freeing_and_reuse_at_scale(oracle, gpu, mode, idb):
    """2^20 + 40 slots, three in four retired; a million-row grace batch whose last tile names retired handles; the stage after it
    frees them and compacts; new stacks take the lowest freed slots at generation 1 (up to slots >= 2^20); a stale handle in the
    last row fails its flush with PA_EINVAL and the next flush is exact"""
    w = base(mode)
    ns = (1 << 20) + 40
    keep = np.flatnonzero(np.arange(ns) % 4 == 0)
    gone = np.flatnonzero(np.arange(ns) % 4 != 0)
    n_new = len(gone) - 10  # the new stacks take every freed slot but the last ten: 20 of them at or above 2^20
    sf = form(w, ns + n_new, seed=2)
    total = int(sf.offsets[-1])
    r = Registry(w, sf, 1 << 20, total + 1, total + 1, idb)
    r.register(0, ns // 2)
    r.register(ns // 2, ns)
    r.flush(r.rng.permutation(keep), what="the batch that keeps one in four")
    got = r.retire(1)
    same(got, r.handle[gone], "retire(1)")
    # the grace batch: a million rows, retired and live handles mixed, the last 32 rows (one tile) naming retired stacks
    st = r.rng.choice(ns, (1 << 20) - 32)
    r.flush(np.concatenate([st, gone[-32:]]), oracle=oracle, what="the grace batch")
    c0 = r.check()
    r.flush(keep[::7], what="the batch whose stage frees the retired stacks")
    c = r.check()
    assert c["stack_compactions"] == c0["stack_compactions"] + 1 and c["stack_frames_dead"] == 0
    assert c["stacks_free"] == len(gone) and c["stack_frames_live"] == int(r.depth[keep].sum())
    stale = r.handle[gone].copy()
    # reuse: the lowest freed slots, next generation
    h = r.register(ns, ns + n_new)
    slots = h & np.uint64(0xFFFFFFFF)
    same(slots, gone[:n_new], "reused slots")
    assert np.all(h >> np.uint64(32) == 1) and int(slots.max()) >= 1 << 20
    new = np.arange(ns, ns + n_new)
    r.flush(np.concatenate([r.rng.permutation(new), keep[:1000]]), oracle=oracle, what="the batch naming the reused slots")
    # a stale handle (slot >= 2^20, generation 0, now holding another stack) in the last row: PA_EINVAL
    bad = int(stale[n_new - 1])
    assert bad & 0xFFFFFFFF >= 1 << 20 and bad >> 32 == 0
    handles = np.concatenate([r.handle[new[:5000]], [bad]]).astype(np.uint64)
    r.load(r.a, r.hdrs(len(handles)), handles)
    r.m.stage()
    assert not r.m.batch(handles)
    with pytest.raises(lib.PaError) as e:
        r.a.flush()
    assert e.value.code == EINVAL
    r.flush(np.concatenate([new[-3000:], keep[-3000:]]), what="the flush after the refusal")
    r.check()
    r.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode,idb", MODES)
def test_compaction_at_live_scan_block_borders(oracle, gpu, sms, mode, idb):
    """2^20 + 1 slots (several hundred StackLiveF blocks): live stacks on both sides of every block border, the two next to them
    retired, a 65535-id stack on a block's last slot and one on the last slot. The stage after the grace batch compacts; then
    stacks registered while a batch is staged overflow the arena, which regrows (and compacts) before that batch's pass."""
    w = base(mode)
    live, deep = live_plan(BIG, sms)
    n_late = 200
    sf = form(w, BIG + n_late, seed=3, deep=deep + list(range(BIG, BIG + n_late)))
    f0 = int(sf.offsets[BIG])
    r = Registry(w, sf, BIG, 6 * f0, 4 * f0, idb)
    r.register(0, BIG // 2)
    r.register(BIG // 2, BIG)
    r.flush(r.rng.permutation(live), what="the batch naming the live stacks")
    r.retire(1)
    c0 = r.check()
    r.flush(live, what="the grace batch")
    r.flush(r.rng.permutation(live), oracle=oracle, what="the batch after the compaction")
    c = r.check()
    assert c["stack_compactions"] == c0["stack_compactions"] + 1 and c["stack_frames_live"] == r.m.frames_live == int(r.depth[live].sum())
    # the arena holds 2 f0 frame ids (sized at the first upload; a stage compaction keeps the size): pending frames beyond that
    # make the pass of the staged batch regrow it first
    late = -(-(2 * f0) // 65535) + 1
    assert late <= n_late
    stacks = r.rng.permutation(live)
    handles = r.handle[stacks]
    hdrs = r.hdrs(len(stacks))
    r.load(r.a, hdrs, handles)
    r.a.stage()
    r.m.stage()
    assert r.m.batch(handles)
    r.register(BIG, BIG + late)
    r.a.process()
    got = r.a.collect().ipc_bytes()
    assert got == r.ring_bytes(hdrs, stacks), "the batch staged across the regrowth differs from the ring mode"
    c = r.check()
    assert c["stack_compactions"] == c0["stack_compactions"] + 2
    both = np.concatenate([live, np.arange(BIG, BIG + late)])
    r.flush(r.rng.permutation(both), what="every live stack once, after the regrowth")
    assert r.check()["stack_frames_live"] == r.m.frames_live == int(r.depth[both].sum())
    r.close()


def regrow_steps(last=BIG):
    """Slot counts to register up to, stage by stage, and the ones whose stage regrows the record and last_use arrays (agg.cu
    rs_upload: past their capacity they are reallocated for max(2 x slots, 1024) slots). From 1023, 1024 and 1025, every
    capacity is reached exactly and then passed by one."""
    steps, grows, cap = [1023, 1024, 1025], [1023], 2046
    while cap < last:
        steps += [cap, cap + 1]
        grows.append(cap + 1)
        cap = 2 * (cap + 1)
    return steps + [last], grows


def test_regrow_steps():
    steps, grows = regrow_steps()
    assert steps[:7] == [1023, 1024, 1025, 2046, 2047, 4094, 4095] and steps[-1] == BIG and sorted(set(steps)) == steps
    assert len(grows) == 11 and grows[-1] == (1 << 20) - 1  # the last regrowth holds 2^21 - 2 slots: BIG fits


@pytest.mark.gpu
@pytest.mark.parametrize("mode,idb", MODES)
def test_record_arrays_regrow(gpu, mode, idb):
    """The record and last_use arrays grow from 1024 slots by doubling. Between steps a stage uploads the new slots (and regrows
    the arrays); each batch names the oldest and the newest stacks, and retire(2) after it must find exactly the model's idle
    slots: a last_use word or a retiring mark lost in a regrowth's copy would show as a wrong handle list, a lost record as a
    refused batch."""
    w = base(mode)
    sf = form(w, 2 * BIG, seed=4)
    r = Registry(w, sf, 64, int(sf.offsets[-1]) + 1, 64 * 9, idb)
    nxt = 0
    for target in regrow_steps()[0]:
        k = target - len(r.m.state) + int(np.sum(r.m.state == FREE))
        assert nxt + k <= len(sf.hashes)
        r.register(nxt, nxt + k)
        nxt += k
        assert len(r.m.state) == target
        r.flush([0, 1, 2, nxt - 3, nxt - 2, nxt - 1, 0], what="step %d" % target)  # stacks 0..2 hold slots 0..2 throughout
        r.retire(2, what="step %d" % target)
    assert r.check()["stacks_retired"] > BIG
    r.close()


@pytest.mark.gpu
def test_idle_windows(oracle, gpu):
    """idle_batches equal to the stage count (bound 0: the stacks registered before the first stage and never named), the stage
    count + 1 and 2^32 - 1 (nothing), over 2^17 + 33 slots (3 WordsF blocks)"""
    w = base(abi.PA_HASH_XXH64X2)
    ns = (1 << 17) + 33
    sf = form(w, ns, seed=6)
    r = Registry(w, sf, ns, int(sf.offsets[-1]) + 1, int(sf.offsets[-1]) + 1, 8)
    half = ns // 2 + 7
    r.register(0, half)
    r.flush(np.arange(0, half, 3), oracle=oracle, what="batch 1")
    r.register(half, ns)  # last_use 1: never idle for bound 0
    r.flush(np.arange(1, ns, 5), what="batch 2")
    r.flush(np.arange(2, ns, 11), what="batch 3")
    for idle in (r.m.stages + 1, 2**32 - 1):
        assert len(r.retire(idle)) == 0
    got = r.retire(r.m.stages)
    s = got & np.uint64(0xFFFFFFFF)
    assert len(got) > 1000 and int(s.max()) < half
    assert len(r.retire(r.m.stages)) == 0 and len(r.retire(1)) > 1000
    r.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world,ns", [(2, 300_001), (3, BIG)])
def test_group_retire_at_scale(oracle, gpu, sms, world, ns):
    """Local PA_CFG_GROUP_RETIRE groups: each shard names its own slots, all shards name the slots around every WordsF block
    border, the last shard alone names one slot after each border and no shard the one before it. Every member must retire the
    handles of one retiring aggregator fed the concatenated rows, and of VecModel fed their union; so must the next interval."""
    mode = abi.PA_HASH_PROVIDED if world == 2 else abi.PA_HASH_XXH64X2
    w = base(mode)
    sf = form(w, ns, seed=7)
    f0 = int(sf.offsets[-1])
    r = Registry(w, sf, ns + 1000, 2 * f0, f0 + 1, 8)
    members = [lib.from_workload(w.head(0), max_samples=ns, max_frames=2 * f0, flags=GROUP) for _ in range(world)]
    g = lib.MergeGroup.local(members)
    for lo, hi in ((0, ns // 3), (ns // 3, ns)):
        fr, o, hs = span(sf, lo, hi)
        hs = hs if mode == abi.PA_HASH_PROVIDED else None
        for a in members:
            same(a.register_stack_handles(fr, o, hs), np.arange(lo, hi), "member registration")
        r.register(lo, hi)
    slot = np.arange(ns)
    named = np.zeros((world, ns), bool)
    named[(slot // 37) % world, slot] = True
    named[:, slot % 5 == 0] = False
    for b, _ in words_blocks(ns, sms)[1:]:
        named[:, b - 2:b + 2] = True
        named[:, b - 3] = False
        if b + 2 < ns:
            named[:, b + 2] = False
            named[world - 1, b + 2] = True
    rows = [r.rng.permutation(np.flatnonzero(named[i])) for i in range(world)]

    def interval(parts, oracle=None):
        """member i takes parts[i]; the single aggregator the concatenated rows"""
        hdrs = [r.hdrs(len(p)) for p in parts]
        for a, h, p in zip(members, hdrs, parts):
            r.load(a, h, r.handle[p])
        stacks, hd = np.concatenate(parts), np.concatenate(hdrs)
        r.load(r.a, hd, r.handle[stacks])
        r.m.stage()
        assert r.m.batch(r.handle[stacks])
        got, want = g.flush().ipc_bytes(), r.a.flush().ipc_bytes()
        assert got == want, "the group differs from one retiring aggregator"
        assert want == r.ring_bytes(hd, stacks, oracle), "the single aggregator differs from the ring mode"

    interval(rows, oracle)
    wb = words_blocks(ns, sms)
    idle = np.flatnonzero(~named.any(axis=0))
    for cap in (int(np.sum(idle < wb[1][0])) + 1, None):
        got = g.retire_stacks(1, cap)
        same(got, r.a.retire_stacks(1, cap), "group against the single aggregator")
        same(got, r.m.retire(1, cap), "group against the model")
        for a in members:
            assert a.stack_counters() == r.a.stack_counters()
        r.check()
    assert r.m.retired == len(idle)
    live = np.flatnonzero(r.m.state == LIVE)
    st = r.rng.choice(live, 200_000)
    cut = np.sort(r.rng.choice(len(st) + 1, world - 1))
    interval(np.split(st, cut))
    r.check()
    g.close()
    for a in members:
        a.close()
    r.close()
