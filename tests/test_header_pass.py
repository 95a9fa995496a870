"""The sample-header pass (k_header) stages the headers of 32-row tiles in shared memory, one tile per warp at a time,
eight warps (256 rows) per block. These batches put rows, chunk borders, bad ids and first occurrences at the borders of
those tiles and blocks; every output must equal the oracle's byte for byte, and bad ids must be reported as before."""
import numpy as np
import pyarrow as pa
import pytest

import pyref
from parca_agent_b200 import abi, sharded, synth

pytestmark = pytest.mark.gpu

TILE = 32    # rows per k_header tile (one per lane of a warp)
BLOCK = 256  # rows per round of a block's eight warps
MODES = [abi.PA_HASH_PROVIDED, abi.PA_HASH_XXH64X2]


@pytest.fixture(scope="module")
def gpu():
    import torch
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    from parca_agent_b200 import lib
    lib.lib()
    return lib


def assert_same(oracle, gpu, w, **kw_run):
    want, st = oracle.run(w)
    got, r = gpu.run(w, **kw_run)
    assert r.n_rows == st["rows"] == w.n
    if got != want:
        v1 = getattr(w, "schema", 0) == abi.PA_SCHEMA_V1
        ex = pyref.extract_v1 if v1 else pyref.extract
        d = pyref.diff(ex(pa.ipc.open_stream(want).read_all()), ex(pa.ipc.open_stream(got).read_all())) if want and got else None
        raise AssertionError("IPC bytes differ (len %d vs %d); first logical difference: %s" % (len(want), len(got), d))
    assert r.n_unique_stacks == st["unique_stacks"]


def edge(n, mode, seed=5):
    return synth.edge_workload(seed=seed, n=n, hash_mode=mode, external=False)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("n", [1, TILE - 1, TILE, TILE + 1, 5 * TILE + 17, BLOCK - 1, BLOCK, BLOCK + 1, 5 * BLOCK + 77])
def test_batch_sizes_around_the_tile(oracle, gpu, n, mode):
    assert_same(oracle, gpu, edge(n, mode, seed=n))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("chunk", [100, 300, 1000])
def test_chunk_borders_inside_tiles(oracle, gpu, mode, chunk):
    """several chunks per flush whose borders fall inside a tile: one header launch per chunk (provided ids) or all headers
    first (XXH64, with the early copy-out of the trailing columns)"""
    assert_same(oracle, gpu, edge(9 * BLOCK + 13, mode, seed=chunk), chunk_samples=chunk)


@pytest.mark.parametrize("field,value,message", [
    ("kind", 9, "sample kind out of range"),
    ("labelset_id", 10_000, "unregistered labelset"),
    ("cpu", 70_000, "cpu id >= 65536"),
    ("frame_off", 1 << 40, "frame range outside the staged frames"),
])
@pytest.mark.parametrize("row", [-1, -13])
@pytest.mark.parametrize("mode", MODES)
def test_bad_id_in_the_last_partial_tile(gpu, field, value, message, row, mode):
    """3 * BLOCK + 50 rows: the last tile holds 18 rows (one launch over all rows with XXH64 ids; with provided ids one
    launch per 259-row chunk, whose last tile holds 9)"""
    w = edge(3 * BLOCK + 50, mode)
    w.hdrs[field][row] = value
    a = gpu.from_workload(w, chunk_samples=BLOCK + 3)
    gpu.load(a, w)
    with pytest.raises(gpu.PaError, match=message):
        a.flush()
    gpu.load(a, edge(3 * BLOCK + 50, mode))  # the aggregator stays usable after the rejected batch
    assert a.flush().n_rows == 3 * BLOCK + 50
    a.close()


def first_rows_at_the_ends(mode):
    """labelset 4, cpu 50 and tid 4242 occur only in row 0; labelset 5, cpu 77 and tid 31337 only in the last tile"""
    n = 4 * BLOCK + 45
    w = edge(n, mode)
    h = w.hdrs
    h["labelset_id"][h["labelset_id"] == 4] = 1
    h["labelset_id"][h["labelset_id"] == 5] = 2
    h["labelset_id"][0], h["cpu"][0], h["tid"][0] = 4, 50, 4242
    h["labelset_id"][n - 5], h["cpu"][n - 7], h["tid"][n - 1] = 5, 77, 31337  # the last tile holds 13 rows
    return w


@pytest.mark.parametrize("mode", MODES)
def test_first_rows_in_row_zero_and_the_last_tile(oracle, gpu, mode):
    w = first_rows_at_the_ends(mode)
    assert_same(oracle, gpu, w)
    assert_same(oracle, gpu, w, chunk_samples=BLOCK + 1)
    w.schema = abi.PA_SCHEMA_V1
    assert_same(oracle, gpu, w)


@pytest.mark.parametrize("mode", MODES)
def test_v1_and_narrow_ring_off_the_tile(oracle, gpu, mode):
    w = edge(7 * BLOCK + 129, mode, seed=17)
    assert_same(oracle, gpu, w, frame_id_bytes=4)
    assert_same(oracle, gpu, w, frame_id_bytes=4, chunk_samples=2 * BLOCK - 1)
    w.schema = abi.PA_SCHEMA_V1
    assert_same(oracle, gpu, w)
    assert_same(oracle, gpu, w, chunk_samples=BLOCK + 1)


def test_config1_prefix_provided_ids(oracle, gpu):
    """provided ids: the stack-table insert runs in the header pass (converged warps at the ragged end of the batch)"""
    assert_same(oracle, gpu, synth.config1(hash_mode=abi.PA_HASH_PROVIDED).head(40 * BLOCK + 211))


@pytest.mark.parametrize("mode", MODES)
def test_two_shard_merge_group_off_the_tile(oracle, gpu, mode):
    """a merge group records GLOBAL first rows (row_base): shards of 2 * BLOCK + 33 and 3 * BLOCK + 7 rows"""
    w = edge(5 * BLOCK + 40, mode, seed=23)
    idx = [np.arange(0, 2 * BLOCK + 33), np.arange(2 * BLOCK + 33, w.n)]
    want, st = oracle.run(w.rows(np.concatenate(idx)))
    parts = [w.rows(ix) for ix in idx]
    aggs = [gpu.from_workload(p) for p in parts]
    g = gpu.MergeGroup.local(aggs)
    try:
        for _ in range(2):  # a second interval over the same members
            for a, p in zip(aggs, parts):
                gpu.load(a, p)
            res = g.flush()
            assert res.ipc_bytes() == want
            assert res.n_rows == st["rows"] and res.n_unique_stacks == st["unique_stacks"]
    finally:
        g.close()
        for a in aggs:
            a.close()
    # the same rows sharded by pid (interleaved rows, no contiguous blocks)
    parts = sharded.shard_rows(w, 2)
    want = oracle.run(w.rows(np.concatenate(parts)))[0]
    aggs = [gpu.from_workload(w.rows(ix)) for ix in parts]
    g = gpu.MergeGroup.local(aggs)
    try:
        for a, ix in zip(aggs, parts):
            gpu.load(a, w.rows(ix))
        assert g.flush().ipc_bytes() == want
    finally:
        g.close()
        for a in aggs:
            a.close()
