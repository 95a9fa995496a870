"""PA_IPC_LZ4_FRAME_GPU: the record and dictionary batch bodies LZ4_FRAME-compressed on the device (ipc.WithLZ4() framing).

Not byte-identical to any other writer, so every check compares with the PLAIN stream of the same batch through three
independent decoders: pyarrow's reader (record equality), pyarrow.decompress per buffer (buffer equality), and the
plain-Python frame and block decoder below, which also enforces the LZ4 block rules that a strict decoder such as
pierrec/lz4 relies on and liblz4 tolerates being broken. The decoder's own tests run on the CPU tier."""
import struct

import numpy as np
import pyarrow as pa
import pytest

import ipc_inspect
from parca_agent_b200 import abi, lib, synth

FRAME_HEADER = bytes.fromhex("04224d18604082")  # magic, FLG 0x60, BD 0x40 (64 KiB blocks), HC 0x82
BLOCK = 65536


class FrameError(AssertionError):
    pass


def _need(cond, what):
    if not cond:
        raise FrameError(what)


def _length(b, i, base):
    n = base
    if base == 15:
        while True:
            _need(i < len(b), "length extension runs past the block")
            x = b[i]
            i += 1
            n += x
            if x != 255:
                break
    return n, i


def decode_block(b):
    """One LZ4 block; raises FrameError when a rule of the format is broken."""
    out = bytearray()
    i, last_match = 0, None
    while True:
        _need(i < len(b), "block ends with a match (no closing literals)")
        tok = b[i]
        i += 1
        lit, i = _length(b, i, tok >> 4)
        _need(i + lit <= len(b), "literals run past the block")
        out += b[i:i + lit]
        i += lit
        if i == len(b):
            break
        _need(i + 2 <= len(b), "truncated offset")
        off = b[i] | b[i + 1] << 8
        i += 2
        _need(1 <= off <= len(out), "offset %d reaches before the block start (at %d)" % (off, len(out)))
        ml, i = _length(b, i, tok & 15)
        ml += 4
        start = len(out)
        src = start - off
        while len(out) < start + ml:  # overlapping copies repeat the last `off` bytes
            k = min(off, start + ml - len(out))
            out += out[src:src + k]
            src += k
        last_match = (start, start + ml)
    n = len(out)
    _need(n <= BLOCK, "block decodes to %d bytes (> 64 KiB)" % n)
    if last_match is not None:
        _need(n >= 13, "a block shorter than 13 bytes holds a match")
        _need(last_match[0] <= n - 12, "last match starts %d bytes before the end" % (n - last_match[0]))
        _need(last_match[1] <= n - 5, "last match ends %d bytes before the end" % (n - last_match[1]))
    return bytes(out)


def decode_frame(f):
    """One whole frame as this library writes it: exact header, independent blocks, EndMark, nothing after it."""
    _need(bytes(f[:7]) == FRAME_HEADER, "frame header %s" % bytes(f[:7]).hex())
    i, out = 7, bytearray()
    while True:
        _need(i + 4 <= len(f), "missing EndMark")
        bs = struct.unpack_from("<I", f, i)[0]
        i += 4
        if bs == 0:
            break
        n = bs & 0x7FFFFFFF
        _need(n <= BLOCK and i + n <= len(f), "block of %d stored bytes" % n)
        blk = bytes(f[i:i + n])
        i += n
        out += blk if bs >> 31 else decode_block(blk)
    _need(i == len(f), "bytes after the EndMark")
    return bytes(out)


def check_stream(packed, plain):
    """Record, buffer and frame equality of a GPU-LZ4 stream with the plain stream of the same batch."""
    if not plain:
        assert not packed
        return
    a, b = pa.ipc.open_stream(plain).read_all(), pa.ipc.open_stream(packed).read_all()
    assert a.schema.equals(b.schema, check_metadata=True) and _rewritten(a) == _rewritten(b)
    if a.num_rows <= 5_000:  # Table.equals is slow on run-end encoded columns
        assert a.equals(b)
    assert _validation(b) == _validation(a)  # external labels give the reference's repeated run end, in both streams
    return check_buffers(packed, plain)


def _rewritten(t):
    """The decoded record written again by pyarrow's own (uncompressed) writer: equal bytes = equal records."""
    sink = pa.BufferOutputStream()
    with pa.ipc.new_stream(sink, t.schema) as w:
        w.write_table(t)
    return sink.getvalue().to_pybytes()


def _validation(t):
    try:
        t.validate(full=True)
        return None
    except pa.ArrowInvalid as e:
        return str(e)


def check_buffers(packed, plain, python_decoder=True):
    """Per message: the same nodes, lengths and variadic counts, compression set, the schema message byte-equal, and every
    buffer either an LZ4 frame that decodes to the plain buffer or -1 and the plain buffer's bytes."""
    mp, mc = ipc_inspect.messages(plain), ipc_inspect.messages(packed)
    assert [m["header"] for m in mp] == [m["header"] for m in mc] and mp[0]["header"] == "Schema" and mp[-1]["header"] == "EOS"
    assert plain[:mp[0]["body_at"]] == packed[:mc[0]["body_at"]]
    stats = {"frame": 0, "raw": 0}
    for m, c in zip(mp[1:-1], mc[1:-1]):
        pb, cb = m["batch"], c["batch"]
        assert cb["compression"] and pb["nodes"] == cb["nodes"] and pb["length"] == cb["length"] and pb.get("variadic") == cb.get("variadic")
        assert len(pb["buffers"]) == len(cb["buffers"]) and c["bodyLength"] % 8 == 0
        body = packed[c["body_at"]:c["body_at"] + c["bodyLength"]]
        end = 0
        for (off, n), (coff, cn) in zip(pb["buffers"], cb["buffers"]):
            want = plain[m["body_at"] + off:m["body_at"] + off + n]
            assert coff % 8 == 0 and coff >= end and body[end:coff] == bytes(coff - end)  # zero padding between buffers
            end = coff + cn
            if n == 0:
                assert cn == 0
                continue
            seg = body[coff:coff + cn]
            prefix = struct.unpack_from("<q", seg)[0]
            if prefix == -1:
                stats["raw"] += 1
                assert seg[8:] == want
                continue
            stats["frame"] += 1
            assert prefix == n and cn - 8 < n
            assert pa.decompress(seg[8:], decompressed_size=n, codec="lz4").to_pybytes() == want
            if python_decoder:
                assert decode_frame(seg[8:]) == want
        assert body[end:] == bytes(len(body) - end)
    return stats


def run_both(w, **kw):
    plain, _ = lib.run(w, **kw)
    packed, r = lib.run(w, ipc_compression=abi.PA_IPC_LZ4_FRAME_GPU, **kw)
    assert r.n_rows == w.n
    return packed, plain


# ---------------------------------------------------------------------------------------------------------------------
# CPU tier: the decoder and rule checker on hand-built frames

def _seq(lits, off=0, ml=0):
    """One sequence; ml == 0: closing literals."""
    def ext(n):
        return b"" if n < 15 else bytes([255] * ((n - 15) // 255) + [(n - 15) % 255])
    m = ml - 4 if ml else 0
    out = bytes([min(len(lits), 15) << 4 | min(m, 15)]) + ext(len(lits)) + lits
    return out + struct.pack("<H", off) + ext(m) if ml else out


def _frame(*blocks, header=FRAME_HEADER):
    out = bytearray(header)
    for b, raw in blocks:
        out += struct.pack("<I", len(b) | (0x80000000 if raw else 0)) + b
    return bytes(out + bytes(4))


def test_decoder_accepts_valid_frames():
    lits = bytes(range(20))
    blk = _seq(lits, 20, 300) + _seq(b"abcdefghijklm")  # 20 literals, a 300-byte repeat, 13 closing literals
    want = lits + (lits * 16)[:300] + b"abcdefghijklm"
    assert decode_frame(_frame((blk, False), (b"xyz", True))) == want + b"xyz"
    assert decode_frame(_frame((_seq(b"a"), False), (_seq(b"x" * 270), False))) == b"a" + b"x" * 270  # literal-only blocks
    run = _seq(b"\x07", 1, 100) + _seq(b"\x00" * 5)  # an offset-1 run overlaps its own output
    assert decode_frame(_frame((run, False))) == b"\x07" * 101 + b"\x00" * 5
    assert decode_frame(_frame()) == b""
    # pyarrow's decoder agrees with ours on these frames
    assert pa.decompress(_frame((blk, False)), decompressed_size=len(want), codec="lz4").to_pybytes() == want


def test_decoder_rejects_broken_frames():
    good = _seq(bytes(range(16)), 16, 16) + _seq(b"12345678")
    assert decode_frame(_frame((good, False)))
    cases = {
        "wrong HC": _frame((good, False), header=FRAME_HEADER[:6] + b"\x83"),
        "linked blocks FLG": _frame((good, False), header=b"\x04\x22\x4d\x18\x40\x40\xc0"),
        "match ends within 5 bytes of the end": _frame((_seq(bytes(range(16)), 16, 16) + _seq(b"1234"), False)),
        "match starts within 12 bytes of the end": _frame((_seq(bytes(range(16)), 16, 4) + _seq(b"1234567"), False)),
        "block ends with a match": _frame((_seq(bytes(range(16)), 16, 16), False)),
        "offset before the block start": _frame((_seq(bytes(range(16)), 17, 16) + _seq(b"12345678"), False)),
        "offset 0": _frame((_seq(bytes(range(16)), 0, 16) + _seq(b"12345678"), False)),
        "match in a block shorter than 13 bytes": _frame((_seq(b"ab", 1, 4) + _seq(b"12345"), False)),
        "block of more than 64 KiB": _frame((_seq(b"\x00" * 20, 1, BLOCK) + _seq(b"\x00" * 12), False)),
        "stored block of more than 64 KiB": _frame((b"\x00" * (BLOCK + 1), True)),
        "missing EndMark": _frame((good, False))[:-4],
        "trailing bytes": _frame((good, False)) + b"\x00",
    }
    for what, f in cases.items():
        with pytest.raises(FrameError):
            decode_frame(f)
            pytest.fail(what)


def test_header_checksum():
    """HC is the second byte of XXH32 over FLG and BD (seed 0), as the frame format defines it."""
    def xxh32(data, seed=0):
        P1, P2, P3, P4, P5 = 2654435761, 2246822519, 3266489917, 668265263, 374761393
        M = 0xFFFFFFFF
        rot = lambda x, r: ((x << r) | (x >> (32 - r))) & M  # noqa: E731
        h = (seed + P5 + len(data)) & M
        for c in data:
            h = rot((h + c * P5) & M, 11) * P1 & M
        h ^= h >> 15; h = h * P2 & M; h ^= h >> 13; h = h * P3 & M; h ^= h >> 16
        return h
    assert (xxh32(FRAME_HEADER[4:6]) >> 8) & 0xFF == FRAME_HEADER[6]


# ---------------------------------------------------------------------------------------------------------------------
# GPU: whole workloads

@pytest.mark.gpu
@pytest.mark.parametrize("seed", [1, 2, 3])
@pytest.mark.parametrize("hash_mode", [abi.PA_HASH_PROVIDED, abi.PA_HASH_XXH64X2])
def test_edge_workloads(seed, hash_mode):
    for flags in (0, 7):
        w = synth.edge_workload(seed=seed, n=900, hash_mode=hash_mode, label_flags=flags, external=True)
        check_stream(*run_both(w))


@pytest.mark.gpu
def test_configs_ragged_narrow_ring_and_chunks():
    seen = {"frame": 0, "raw": 0}
    for w, kw in [(synth.config1(), {}),
                  (synth.config3(n=50_000, u=3_000, p=4_096, npids=64, lsets=6), {}),
                  (synth.config3(n=50_000, u=3_000, p=4_096, npids=64, lsets=6), {"frame_id_bytes": 4, "chunk_samples": 7_000}),
                  (synth.ragged(n=30_000, u=2_000, p=4_096), {"chunk_samples": 4_096})]:
        st = check_stream(*run_both(w, **kw))
        seen = {k: seen[k] + st[k] for k in seen}
    assert seen["frame"] > 0 and seen["raw"] > 0


@pytest.mark.gpu
def test_v1_records_and_stacktraces():
    """v1 sample records, and the stacktrace record, whose buffers come from host memory (ids, offsets) and zero fills."""
    for w in (synth.config3(n=20_000, u=2_000, p=4_096, npids=64, lsets=6), synth.edge_workload(seed=5, n=700, hash_mode=abi.PA_HASH_XXH64X2)):
        w.schema = abi.PA_SCHEMA_V1
        out = {}
        for mode in (abi.PA_IPC_PLAIN, abi.PA_IPC_LZ4_FRAME_GPU):
            a = lib.from_workload(w, ipc_compression=mode)
            lib.load(a, w)
            r = a.flush()
            ids = a.last_stack_ids(r.n_unique_stacks).tobytes()
            probe = ids[: 16 * (r.n_unique_stacks // 2)] + bytes(range(16))  # known stacks and one unknown id
            out[mode] = (r.ipc_bytes(), a.stacktraces(probe).ipc_bytes())
            if mode == abi.PA_IPC_LZ4_FRAME_GPU:
                ms, launches = a.kernel_ms("lz4")
                assert launches == 3 and ms > 0
            a.close()
        check_stream(out[abi.PA_IPC_LZ4_FRAME_GPU][0], out[abi.PA_IPC_PLAIN][0])
        check_stream(out[abi.PA_IPC_LZ4_FRAME_GPU][1], out[abi.PA_IPC_PLAIN][1])


@pytest.mark.gpu
def test_empty_batch_and_repeat_flushes():
    w = synth.edge_workload(seed=6, n=500, hash_mode=abi.PA_HASH_XXH64X2)
    a = lib.from_workload(w, ipc_compression=abi.PA_IPC_LZ4_FRAME_GPU)
    r = a.flush()
    assert r.n_rows == 0 and r.ipc_len == 0
    lib.load(a, w)
    first = a.flush().ipc_bytes()
    lib.load(a, w)
    second = a.flush().ipc_bytes()
    assert first == second  # the same batch collected twice
    lib.load(a, w)
    a.stage(); a.process(); a.process()
    assert a.collect().ipc_bytes() == first
    a.close()
    packed, plain = run_both(w)
    assert packed == first  # and from a second aggregator
    check_stream(packed, plain)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: encoder edges, shaped through the timestamp column (8 bytes per row) and through a registered label value (the
# dictionary data of its column)

def _rng(seed):
    return np.random.Generator(np.random.PCG64(seed))


def _rand(rng, n):
    return rng.integers(0, 256, n, dtype=np.uint8).tobytes()


def _shapes():
    r = _rng(11)
    out = {"random": _rand(r, 70_000), "zeros": bytes(BLOCK + 8), "run_ab": b"\xab" * 140_000}
    for n in range(1, 14):
        out["short%d" % n] = _rand(r, n)
    for n in (BLOCK - 1, BLOCK, BLOCK + 1, 2 * BLOCK - 1, 2 * BLOCK, 2 * BLOCK + 1):
        out["len%d" % n] = (_rand(r, 5_000) * (n // 5_000 + 1))[:n]
    base = _rand(r, 300)
    seqs = bytearray(base)
    for lit in (14, 15, 19, 270, 271):
        for ml in (14, 15, 19, 270, 271):
            seqs += _rand(r, lit) + base[:ml]
    out["lengths"] = bytes(seqs) + _rand(r, 32)
    far = bytearray(_rand(r, 2 * BLOCK + 200))
    far[BLOCK - 1:BLOCK + 39] = far[0:40]          # exactly 65535 bytes back (across the block border)
    far[BLOCK + 100:BLOCK + 140] = far[100:140]    # exactly 65536 bytes back
    far[BLOCK + 2:BLOCK + 60] = far[BLOCK - 90:BLOCK - 32]  # a repeat of bytes just before the border
    out["far"] = bytes(far)
    straddle = bytearray(_rand(r, 2 * BLOCK))
    straddle[BLOCK - 50:BLOCK + 50] = straddle[1_000:1_100]  # a match that would run across the border
    out["straddle"] = bytes(straddle)
    return out


def _with_timestamps(w, data):
    data = data + bytes(-len(data) % 8)
    n = len(data) // 8
    x = w.head(min(w.n, n)) if n <= w.n else w.rows(np.arange(n) % w.n)
    x.hdrs["timestamp_ns"] = np.frombuffer(data, dtype="<i8")
    return x


def _with_label_value(w, value):
    strings = list(w.strings) + [b"zz_payload", value]
    labelsets = list(w.labelsets) + [[(len(strings) - 2, len(strings) - 1)]]
    hd = w.hdrs.copy()
    hd["labelset_id"][1::3] = len(labelsets) - 1
    x = synth.Workload(w.name + "+label", strings, w.frames, labelsets, hd, _frame_ids=w.frame_ids, hash_mode=w.hash_mode,
                       label_flags=w.label_flags, samples_per_second=w.samples_per_second, external_labels=list(w.external_labels))
    return x


@pytest.mark.gpu
def test_encoder_edges_through_timestamps():
    base = synth.edge_workload(seed=8, n=600, hash_mode=abi.PA_HASH_XXH64X2, external=False)
    for name, data in _shapes().items():
        if len(data) < 8:
            continue
        try:
            check_stream(*run_both(_with_timestamps(base, data)))
        except AssertionError as e:
            raise AssertionError("%s: %s" % (name, e)) from e


@pytest.mark.gpu
def test_encoder_edges_through_label_strings():
    base = synth.edge_workload(seed=9, n=300, hash_mode=abi.PA_HASH_XXH64X2, external=False)
    for name, data in _shapes().items():
        try:
            check_stream(*run_both(_with_label_value(base, data)))
        except AssertionError as e:
            raise AssertionError("%s: %s" % (name, e)) from e


# ---------------------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_merge_groups_refuse_gpu_lz4_members():
    w = synth.edge_workload(seed=4, n=200, hash_mode=abi.PA_HASH_XXH64X2, external=False)
    a = lib.from_workload(w, ipc_compression=abi.PA_IPC_LZ4_FRAME_GPU)
    b = lib.from_workload(w)
    with pytest.raises(lib.PaError) as e:
        lib.MergeGroup.local([b, a])
    assert e.value.code == -22
    assert b"PA_IPC_LZ4_FRAME_GPU" in lib.lib().pa_agg_last_error(a.h)
    a.close(); b.close()


@pytest.mark.gpu
def test_create_rejects_unknown_compression():
    w = synth.edge_workload(seed=4, n=10)
    with pytest.raises(lib.PaError):
        lib.from_workload(w, ipc_compression=3)


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", ["config2", "config3"])
def test_ratio_against_host_mode(cfg):
    """At 1M rows the independent 64 KiB blocks cost little against liblz4's linked frames."""
    w = getattr(synth, cfg)(n=1_000_000)
    packed, plain = run_both(w)
    host = lib.compress_lz4(plain)
    assert len(packed) <= 1.08 * len(host), (len(packed), len(host), len(plain))
    mp, mc = ipc_inspect.messages(plain), ipc_inspect.messages(packed)
    assert [m["header"] for m in mp] == [m["header"] for m in mc]
    a, b = pa.ipc.open_stream(plain).read_all(), pa.ipc.open_stream(packed).read_all()
    assert a.num_rows == b.num_rows and a.column("value").equals(b.column("value"))
