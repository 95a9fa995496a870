"""Merge groups of PA_IPC_LZ4_FRAME_GPU members: the merged stream must be, byte for byte, the stream ONE such aggregator makes
from [shard 0's rows, shard 1's rows, ...], and must decode to the oracle's record for those rows.

Each buffer is compressed on the whole buffer's 64 KiB block grid. Block k belongs to the member whose part of the buffer holds
the block's first byte; a block that runs past that part needs the heads of the following parts (their bytes up to the next grid
boundary). The plain-Python model below restates that rule; its self-checks run on the CPU tier, and the GPU cases use it to
show that their shard cuts produce the situations they are meant to cover. Multi-process groups run
tests/dist_merge_lz4_check.py under torchrun."""
import os
import subprocess
import sys

import numpy as np
import pyarrow as pa
import pytest

from parca_agent_b200 import abi, sharded, synth
from test_ipc_lz4_gpu import check_buffers

BLOCK = 65536
LZ4 = abi.PA_IPC_LZ4_FRAME_GPU
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


# ---------------------------------------------------------------------------------------------------------------------
# CPU tier: the block-ownership model

def block_owners(extents, length, block=BLOCK):
    """extents: per rank, (offset, bytes) of its part of one buffer of `length` bytes. Returns, per block of the buffer's grid,
    (owner, heads): the rank whose part holds the block's first byte, and the (rank, offset, bytes) pieces of the following parts
    that the block also covers (each one the head of its part: from the part's start up to the next grid boundary)."""
    pos = 0
    for at, n in extents:
        if n:
            assert at == pos, "parts must follow each other"
            pos += n
    assert pos == length, "parts must cover the buffer"
    out = []
    for k in range((length + block - 1) // block):
        s, e = k * block, min((k + 1) * block, length)
        owner = next(r for r, (at, n) in enumerate(extents) if n and at <= s < at + n)
        heads = [(r, at, min(at + n, e) - at) for r, (at, n) in enumerate(extents) if r > owner and n and s < at < e]
        out.append((owner, heads))
    return out


def situations(extents, length, block=BLOCK):
    """Which border situations a cut produces on one buffer's grid."""
    got = set()
    owners = block_owners(extents, length, block)
    for r, (at, n) in enumerate(extents):
        if not n:
            got.add("empty")
            continue
        end = at + n
        if end < length:
            if end % block == 0:
                got.add("ends_on_border")
            elif end % block == block - 1:
                got.add("ends_byte_before")
            elif end % block == 1:
                got.add("ends_byte_after")
        if n // block >= 2:
            got.add("several_blocks")
    for owner, heads in owners:
        if heads:
            got.add("crossing")
        if len(heads) >= 2:
            got.add("three_parts_in_block")
    return got


def row_extents(sizes, width):
    at, out = 0, []
    for n in sizes:
        out.append((at * width, n * width))
        at += n
    return out


def test_model_hand_built_extents():
    B = 16
    # a part ending exactly on the border: no heads, the next part owns the next block
    assert block_owners([(0, 16), (16, 16)], 32, B) == [(0, []), (1, [])]
    # one byte before the border: block 0 takes a 1-byte head of part 1
    assert block_owners([(0, 15), (15, 17)], 32, B) == [(0, [(1, 15, 1)]), (1, [])]
    # one byte after: part 0 owns block 0 whole and block 1's first byte; part 1's head is the rest of block 1
    assert block_owners([(0, 17), (17, 15)], 32, B) == [(0, []), (0, [(1, 17, 15)])]
    # 1-byte part, empty parts and three or more parts inside one block
    ext = [(0, 3), (3, 0), (3, 1), (4, 0), (4, 5), (9, 40)]
    assert block_owners(ext, 49, B) == [(0, [(2, 3, 1), (4, 4, 5), (5, 9, 7)]), (5, []), (5, []), (5, [])]
    assert {"empty", "crossing", "three_parts_in_block", "several_blocks"} <= situations(ext, 49, B)
    # a part longer than several blocks, starting and ending off the grid
    assert block_owners([(0, 5), (5, 60), (65, 3)], 68, B) == [(0, [(1, 5, 11)]), (1, []), (1, []), (1, []), (1, [(2, 65, 3)])]
    assert situations([(0, 16), (16, 15), (31, 2), (33, 31)], 64, B) >= {"ends_on_border", "ends_byte_before", "ends_byte_after", "crossing"}
    # every byte is placed exactly once
    for ext, n in ([(0, 5), (5, 60), (65, 3)], 68), (ext, 49):
        cover = np.zeros(n, np.int64)
        for k, (owner, heads) in enumerate(block_owners(ext, n, B)):
            s, e = k * B, min((k + 1) * B, n)
            own_end = min(e, ext[owner][0] + ext[owner][1])
            cover[s:own_end] += 1
            for _, at, m in heads:
                cover[at:at + m] += 1
        assert (cover == 1).all()


# the contiguous-row cuts of the GPU case below, and what they produce on the 8-, 16- and 4-byte row columns
BORDER_CUTS = [0, 8192, 8193, 8195, 8195, 16383, 16385, 32768, 60000]


def test_model_border_cuts():
    sizes = np.diff(BORDER_CUTS)
    n = BORDER_CUTS[-1]
    s8 = situations(row_extents(sizes, 8), n * 8)        # timestamp, value: 8192 rows per block
    s16 = situations(row_extents(sizes, 16), n * 16)     # stacktrace_id: 4096 rows per block
    s4 = situations(row_extents(sizes, 4), n * 4)        # ListView offsets / sizes: 16384 rows per block
    assert {"ends_on_border", "crossing", "empty", "several_blocks"} <= s8
    assert {"ends_on_border", "crossing", "several_blocks"} <= s16
    assert {"three_parts_in_block", "crossing", "ends_on_border"} <= s4
    # 8 bytes before / after a border on the 8-byte columns: the row-granular "one before / one after"
    ends = {(at + m) % BLOCK for at, m in row_extents(sizes, 8)[:-1] if m}
    assert {0, BLOCK - 8, 8} <= ends


# ---------------------------------------------------------------------------------------------------------------------
# GPU tier

@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from parca_agent_b200 import lib
    lib.lib()
    return lib


def merged_lz4(oracle, gpu, w, idx_lists, staged=False, repeat=1, chunk_samples=0, **kw):
    """Shards = the given row subsets of w (in that order), every member PA_IPC_LZ4_FRAME_GPU. The merged bytes must equal one
    PA_IPC_LZ4_FRAME_GPU aggregator's on the concatenated rows and decode to the oracle's stream. Returns the merged bytes."""
    parts = [w.rows(ix) for ix in idx_lists]
    ref = w.rows(np.concatenate([np.asarray(ix, dtype=np.int64) for ix in idx_lists]))
    plain, st = oracle.run(ref)
    single = gpu.run(ref, chunk_samples=chunk_samples, ipc_compression=LZ4, **kw)[0] if ref.n else b""
    aggs = [gpu.from_workload(p, chunk_samples=chunk_samples, ipc_compression=LZ4, **kw) for p in parts]
    g = gpu.MergeGroup.local(aggs)
    got = None
    for _ in range(repeat):
        for a, p in zip(aggs, parts):
            gpu.load(a, p)
        if staged:
            for a in aggs:
                a.stage()
            g.process()
            n = g.plan()
            res = g.collect()
            assert res.ipc_len == n
        else:
            res = g.flush()
        got = res.ipc_bytes()
        assert res.n_rows == st["rows"]
        assert got == single, "merged GPU-LZ4 stream differs from the single aggregator's (%d vs %d bytes)" % (len(got), len(single))
    if plain:
        check_buffers(got, plain, python_decoder=len(plain) < (4 << 20))
    else:
        assert not got
    g.close()
    for a in aggs:
        a.close()
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
@pytest.mark.parametrize("mode", [abi.PA_HASH_PROVIDED, abi.PA_HASH_XXH64X2])
def test_config1_and_edge_workloads(oracle, gpu, world, mode):
    w = synth.config1(hash_mode=mode).head(40_000)
    merged_lz4(oracle, gpu, w, sharded.shard_rows(w, world))
    e = synth.edge_workload(seed=3 + world, n=3000, hash_mode=mode, external=False)
    merged_lz4(oracle, gpu, e, sharded.shard_rows(e, world))


@pytest.mark.gpu
def test_contiguous_cuts_at_block_borders(oracle, gpu):
    """contiguous rows cut at and around the 8-, 16- and 4-byte columns' block borders, with tiny and empty shards (see
    test_model_border_cuts for what each cut produces)"""
    w = synth.config1().head(BORDER_CUTS[-1])
    idx = [np.arange(BORDER_CUTS[i], BORDER_CUTS[i + 1]) for i in range(len(BORDER_CUTS) - 1)]
    merged_lz4(oracle, gpu, w, idx)


@pytest.mark.gpu
def test_null_label_runs_with_a_crossing_bitmap_block(oracle, gpu):
    """label columns with nulls and more than 8 x 64 Ki runs: validity bitmaps longer than one block, parts that meet inside a byte,
    and bitmap blocks that need the heads of the following parts"""
    e = synth.edge_workload(seed=21, n=3000, external=False)
    w = e.rows(np.tile(np.arange(3000), 300))
    cuts = [0, 200_001, 450_003, 450_010, 700_005, w.n]
    idx = [np.arange(cuts[i], cuts[i + 1]) for i in range(len(cuts) - 1)]
    plain, _ = oracle.run(w)
    labels = pa.ipc.open_stream(plain).read_all().column("labels").chunk(0)
    long_nullable = [f.name for f in labels.type if labels.field(f.name).values.null_count and len(labels.field(f.name).values) > 8 * BLOCK]
    assert long_nullable, "the workload must have a nullable label column whose bitmap spans more than one block"
    merged_lz4(oracle, gpu, w, idx)


@pytest.mark.gpu
def test_external_label_new_column(oracle, gpu):
    w = synth.edge_workload(seed=8, n=1500, external=False)
    w.strings = list(w.strings) + [b"cluster", b"prod"]
    w.external_labels = [(len(w.strings) - 2, len(w.strings) - 1)]
    merged_lz4(oracle, gpu, w, sharded.shard_rows(w, 3))


@pytest.mark.gpu
def test_narrow_ring_members(oracle, gpu):
    w = synth.edge_workload(seed=14, n=4000, hash_mode=abi.PA_HASH_XXH64X2, external=False)
    merged_lz4(oracle, gpu, w, sharded.shard_rows(w, 3), frame_id_bytes=4)


@pytest.mark.gpu
def test_config3_in_chunks(oracle, gpu):
    w = synth.config3(n=150_000, u=12_000, p=8_192, npids=300, lsets=8)
    merged_lz4(oracle, gpu, w, sharded.shard_rows(w, 4), chunk_samples=20_000)


@pytest.mark.gpu
def test_config2_scaled_staged_two_intervals(oracle, gpu):
    """stage / process / plan / collect, ipc_len == the planned length, two intervals back to back"""
    w = synth.config2(n=300_000, u=15_000, p=32_768)
    merged_lz4(oracle, gpu, w, sharded.shard_rows(w, 4), staged=True, repeat=2)


@pytest.mark.gpu
def test_raw_buffer_beside_compressed_ones(oracle, gpu):
    """random timestamps do not compress: that buffer is stored raw (-1 and its bytes, each member its part) while its
    neighbours are frames"""
    w = synth.config1().head(60_000)
    w.hdrs["timestamp_ns"][:] = np.random.default_rng(5).integers(0, 2**62, w.n, dtype=np.int64).astype(w.hdrs["timestamp_ns"].dtype)
    idx = sharded.shard_rows(w, 3)
    got = merged_lz4(oracle, gpu, w, idx)
    plain = oracle.run(w.rows(np.concatenate(idx)))[0]
    stats = check_buffers(got, plain, python_decoder=False)
    assert stats["raw"] >= 1 and stats["frame"] >= 1, stats


@pytest.mark.gpu
def test_empty_shards_and_all_empty_group(oracle, gpu):
    w = synth.config1().head(5000)
    idx = sharded.shard_rows(w, 2)
    merged_lz4(oracle, gpu, w, [idx[0], np.zeros(0, np.int64), idx[1]])
    parts = [w.rows(np.zeros(0, np.int64)) for _ in range(2)]
    aggs = [gpu.from_workload(p, max_samples=16, max_frames=64, ipc_compression=LZ4) for p in parts]
    g = gpu.MergeGroup.local(aggs)
    for a in aggs:
        a.stage()
    g.process()
    assert g.plan() == 0
    r = g.collect()
    assert r.n_rows == 0 and r.ipc_len == 0
    g.close()
    for a in aggs:
        a.close()


@pytest.mark.gpu
def test_two_groups_give_identical_bytes(oracle, gpu):
    w = synth.edge_workload(seed=9, n=5000, hash_mode=abi.PA_HASH_XXH64X2, external=False)
    idx = sharded.shard_rows(w, 4)
    assert merged_lz4(oracle, gpu, w, idx) == merged_lz4(oracle, gpu, w, idx)


@pytest.mark.gpu
def test_member_flushes_alone_after_a_merged_interval(oracle, gpu):
    """a member goes back to its own GPU-LZ4 flush; every member reports its share of the lz4 kernels"""
    w = synth.config1().head(100_000)
    idx = sharded.shard_rows(w, 3)
    parts = [w.rows(ix) for ix in idx]
    aggs = [gpu.from_workload(p, ipc_compression=LZ4) for p in parts]
    g = gpu.MergeGroup.local(aggs)
    for a, p in zip(aggs, parts):
        gpu.load(a, p)
    got = g.flush().ipc_bytes()
    assert got == gpu.run(w.rows(np.concatenate(idx)), ipc_compression=LZ4)[0]
    for a in aggs:
        ms, launches = a.kernel_ms("lz4")
        assert launches == 3 and ms > 0  # compress, layout, pack of its blocks
    heads = [a.kernel_ms("lz4_heads")[1] for a in aggs]
    assert heads[0] == 0 and sum(heads) > 0  # shard 0's parts start on the grid
    for a, p in zip(aggs, parts):
        gpu.load(a, p)
        assert a.flush().ipc_bytes() == gpu.run(p, ipc_compression=LZ4)[0]
    g.close()
    for a in aggs:
        a.close()


@pytest.mark.gpu
@pytest.mark.parametrize("order", [(0, 1), (1, 0)])
def test_mixed_local_groups_are_refused(gpu, order):
    w = synth.edge_workload(seed=4, n=200, hash_mode=abi.PA_HASH_XXH64X2, external=False)
    ms = [gpu.from_workload(w), gpu.from_workload(w, ipc_compression=LZ4)]
    with pytest.raises(gpu.PaError) as e:
        gpu.MergeGroup.local([ms[i] for i in order])
    assert e.value.code == -22
    assert b"PA_IPC_LZ4_FRAME_GPU" in gpu.lib().pa_agg_last_error(ms[1].h)
    for a in ms:
        a.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world,transport,mailbox", [(2, "gloo", 0), (3, "gloo", 0), (2, "shm", 0), (3, "shm", 0), (3, "shm", 8192)])
def test_multi_process_groups(world, transport, mailbox):
    """one shard per process on this one GPU, the stream in shared memory; an 8 KiB mailbox makes the heads exchange take many
    rounds; the last case mixes modes and must fail pa_merge_process on every rank"""
    env = dict(os.environ, MASTER_ADDR="127.0.0.1", PA_ONE_GPU="1", PA_MERGE_TRANSPORT=transport, PA_SHM_MAILBOX=str(mailbox))
    port = 29571 + world + (10 if transport == "shm" else 0) + (5 if mailbox else 0)
    p = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", str(world), "--master-addr", "127.0.0.1",
                        "--master-port", str(port), os.path.join(ROOT, "tests", "dist_merge_lz4_check.py")], capture_output=True, text=True, env=env, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    assert "merge-lz4 ok world=%d transport=%s" % (world, transport) in p.stdout
