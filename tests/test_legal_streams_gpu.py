"""The generated-stream population of tests/test_legal_streams_emu.py on the H100, through every raw and frame decode
entry point: raw.Decoder (sb_decompress), sb_decompress_device_ws, snappy_uncompress, host batches with and without
multi-block units, sb_decompress_batch_device and sb_decompress_batch_device_ws; frame.decode_all, read.FrameDecoder
and sb_frame_decode_device(_ws) with and without an index. Every result must be the oracle's, unit for unit. Plus what
only the GPU runs cheaply: literals of 2^24 - 1 and 2^24 + 3 bytes, a 2^32 - 1 literal length, 100,000 units in one
batch, 64 blocked units of 1 to 16 MiB and an unblocked 64 MiB stream."""
import ctypes as C
import io
import random

import pytest

import legal_streams as G
import test_legal_streams_emu as pop
from test_raw_batch_decode_gpu import Units
from test_raw_decode_parallel_gpu import decode_ws, status, to_dev

pytestmark = pytest.mark.gpu

BLOCK = G.BLOCK
MIB = 1 << 20


@pytest.fixture(scope="module")
def snap():
    import torch
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)
    import gpu_helpers
    return gpu_helpers.snap()


def _oracle(oracle, s, cap):
    return pop._oracle(oracle, s, cap)


def _decoder(snap, s, cap):
    import gpu_helpers
    out = bytearray(cap)
    try:
        n = snap.raw.Decoder().decompress(s, out)
    except Exception as e:  # noqa: BLE001
        return gpu_helpers.err_tuple(e), None
    return ("Ok", 0, 0, 0), bytes(out[:n])


def _device_ws(snap, s, cap):
    rc, res, out = decode_ws(snap, to_dev(s), len(s), cap)
    assert rc == 0
    st = status(snap, res)
    return st, (bytes(out[:res.bytes].cpu().numpy()) if st[0] == "Ok" else None), res.nchunks


def _uncompress(snap, s, cap):
    L = snap._lib.lib()
    out, k = C.create_string_buffer(max(cap, 1)), C.c_size_t(cap)
    rc = L.snappy_uncompress(s, len(s), out, C.byref(k))
    return rc, (out.raw[:k.value] if rc == 0 else None)


def check_raw_one_by_one(snap, oracle, streams, caps):
    """raw.Decoder, sb_decompress_device_ws and snappy_uncompress on each stream: the oracle's status and bytes."""
    for s, cap in zip(streams, caps):
        want_st, want = _oracle(oracle, s, cap)
        assert _decoder(snap, s, cap) == (want_st, want), s[:16].hex()
        st, out, _ = _device_ws(snap, s, cap)
        assert (st, out) == (want_st, want), s[:16].hex()
        rc, out = _uncompress(snap, s, cap)
        assert rc == (0 if want is not None else 2 if want_st[0] == "BufferTooSmall" else 1)
        assert out == want


def check_batches(snap, oracle, streams, caps, wants=None, host=True):
    """sb_decompress_batch_device, sb_decompress_batch_device_ws and (host) the host batch: every unit the oracle's."""
    if wants is None:
        wants = [_oracle(oracle, s, c) for s, c in zip(streams, caps)]
    u = Units(streams, caps)
    results = []
    for ws in (False, True):
        rc, res, blocks, t_out = u.run(ws=ws)
        assert rc == 0
        host_out = t_out.cpu().numpy()
        for i, (want_st, want) in enumerate(wants):
            assert res[i][0] == want_st, (ws, i, res[i][0], want_st)
            if want is not None:
                o = u.ooffs[i]
                assert res[i][1] == len(want) and host_out[o:o + len(want)].tobytes() == want, (ws, i)
            o = u.ooffs[i] + caps[i]
            assert host_out[o:o + 16].tobytes() == b"\xee" * 16, (ws, i)
        results.append(blocks)
    if host:
        import gpu_helpers
        got = gpu_helpers.decompress_batch_host(streams, caps)
        for i, (want_st, want) in enumerate(wants):
            assert got[i][0] == want_st, i
            if want is not None:
                assert got[i][1] == want, i
    return results[1]


def _sane(s, limit=70000):
    return pop._header_cap(s, limit)


# ---------------------------------------------------------------------------------------------------------------
# the emulator population


def test_single_block_population_every_raw_entry_point(snap, oracle):
    ss, bad = pop.singles()
    streams = [s.stream for s in ss] + bad
    caps = [len(s.data) for s in ss] + [_sane(b) for b in bad]
    check_batches(snap, oracle, streams, caps)                          # host waves of <= 64 KB units: K2 only
    rng = random.Random(1)
    pick = rng.sample(range(len(streams)), 1500)
    check_raw_one_by_one(snap, oracle, [streams[i] for i in pick], [caps[i] for i in pick])


def test_multi_block_population_every_raw_entry_point(snap, oracle):
    blocked, unblocked, bad = pop.multis()
    ss, sbad = pop.singles()
    streams = [s.stream for s in blocked + unblocked] + bad
    caps = [len(s.data) for s in blocked + unblocked] + [_sane(b, 5 * BLOCK) for b in bad]
    check_raw_one_by_one(snap, oracle, streams, caps)
    for s in blocked:
        if G.model_decode(s.stream, len(s.data))[0][0] == "Ok":
            st, out, nchunks = _device_ws(snap, s.stream, len(s.data))
            assert st[0] == "Ok" and nchunks == (len(s.data) + BLOCK - 1) // BLOCK
    for s in unblocked:
        assert _device_ws(snap, s.stream, len(s.data))[2] == 0
    # one mixed batch: host waves that hold multi-block units
    mixed = streams + [s.stream for s in ss[:300]] + sbad[:300]
    mcaps = caps + [len(s.data) for s in ss[:300]] + [_sane(b) for b in sbad[:300]]
    blocks = check_batches(snap, oracle, mixed, mcaps)
    for i, s in enumerate(blocked):
        if G.model_decode(s.stream, len(s.data))[0][0] == "Ok":
            assert blocks[i] == (len(s.data) + BLOCK - 1) // BLOCK, i
    assert blocks[len(blocked):len(blocked) + len(unblocked)] == [0] * len(unblocked)


def test_frame_population_every_frame_entry_point(snap, oracle):
    import gpu_helpers
    rng = random.Random(4)
    cases = []
    for f in pop.frames():
        cases.append((f.stream, f.offs))
        bodies = [(a + 4, b) for a, b in zip(f.offs, f.offs[1:]) if f.stream[a] in (0, 1) and b > a + 4]
        if bodies:
            a, b = rng.choice(bodies)
            flip = bytearray(f.stream)
            flip[rng.randrange(a, b)] ^= 1 << rng.randrange(8)
            cases.append((bytes(flip), f.offs))
        cases.append((f.stream[:rng.randrange(11, len(f.stream))] if len(f.stream) > 11 else f.stream[:10], f.offs))
    for s, offs in cases:
        want_st, want = pop._frame_expect(oracle, s, offs)
        cap = BLOCK * (len(offs) + 1)
        for index in (offs if offs[-1] == len(s) else None, None):
            for ws in (False, True):
                assert gpu_helpers.frame_decode_device(s, cap, index=index, ws=ws) == (want_st, want), (index is None, ws)
        full = oracle.frame_decode(s) if want_st[0] == "Ok" else None
        for impl in (snap.frame.decode_all, lambda x: snap.read.FrameDecoder(io.BytesIO(x)).read_to_end()):
            try:
                got = (("Ok", 0, 0, 0), impl(s))
            except Exception as e:  # noqa: BLE001
                got = (gpu_helpers.err_tuple(e), None)
            assert got == (want_st, full)


@pytest.mark.parametrize("body", [b"\x80", b"\xff\xff\xff", b"\x80" * 5, b"\x80" * 9 + b"\x10", b"\xff" * 9 + b"\x01"])
def test_frame_chunk_varint_longer_than_its_body(snap, oracle, body):
    import gpu_helpers
    prev = G.chunk(0xFE, bytes([0x11, 0x22, 0x33, 0x44, 0x55, 0x80, 0x80, 0x81, 0x01, 0x00, 0x00]))
    stream = G.IDENT + prev + G.chunk(0x00, body, oracle.crc32c_masked(b""))
    offs = [10, 10 + len(prev), len(stream)]
    want_st, want = pop._frame_expect(oracle, stream, offs)
    for index in (offs, None):
        for ws in (False, True):
            assert gpu_helpers.frame_decode_device(stream, 1 << 17, index=index, ws=ws) == (want_st, want)
    try:
        got = snap.frame.decode_all(stream)
        assert want_st[0] == "Ok" and got == want
    except snap.Error as e:
        assert gpu_helpers.err_tuple(e) == want_st


# ---------------------------------------------------------------------------------------------------------------
# what only the GPU runs cheaply


def test_giant_literals(snap, oracle):
    rng = random.Random(16)
    cases = [G.giant_literal(rng, (1 << 24) + 3, "lit63"), G.giant_literal(rng, (1 << 24) - 1, "lit62")]
    for s, data in cases:
        assert oracle.decompress(s) == data
    streams, caps = [s for s, _ in cases], [len(d) for _, d in cases]
    check_raw_one_by_one(snap, oracle, streams, caps)
    check_batches(snap, oracle, streams, caps, wants=[(("Ok", 0, 0, 0), d) for _, d in cases])


def test_literal_length_of_two_to_the_32_minus_one(snap, oracle):
    s = G.varint(100) + bytes([63 << 2]) + ((1 << 32) - 2).to_bytes(4, "little") + b"x" * 100
    want_st, want = _oracle(oracle, s, 100)
    assert want_st == ("Literal", (1 << 32) - 1, 100, 100) and want is None
    check_raw_one_by_one(snap, oracle, [s], [100])
    check_batches(snap, oracle, [s, s], [100, 1000])


def test_hundred_thousand_units_in_one_batch(snap, oracle):
    ss, bad = pop.singles()
    distinct = [s.stream for s in ss] + bad
    dcaps = [len(s.data) for s in ss] + [_sane(b) for b in bad]
    dwants = [_oracle(oracle, s, c) for s, c in zip(distinct, dcaps)]
    rng = random.Random(17)
    pick = [rng.randrange(len(distinct)) for _ in range(100000)]
    check_batches(snap, oracle, [distinct[i] for i in pick], [dcaps[i] for i in pick], [dwants[i] for i in pick],
                  host=False)


@pytest.fixture(scope="module")
def block_pool():
    return _block_pool()


def _block_pool():
    """64 KB blocked block bodies (each a legal stream alone, so legal as an interior block) and their data."""
    rng = random.Random(18)
    pool = []
    while len(pool) < 48:
        s = G.gen_stream(rng, BLOCK, "blocked", copy_share=rng.choice([0.3, 0.6]), alphabet=rng.choice([3, 256]))
        if G.model_decode(s.stream, BLOCK)[0][0] == "Ok":
            pool.append((s.stream[s.hl:], s.data))
    return pool


def _assemble(rng, pool, nblocks, tail):
    bodies, data = [], []
    for _ in range(nblocks):
        b, d = rng.choice(pool)
        bodies.append(b)
        data.append(d)
    return bodies + [tail.stream[tail.hl:]], data + [tail.data]


def test_blocked_units_of_1_to_16_mib(snap, oracle, block_pool):
    import torch
    rng = random.Random(19)
    streams, datas = [], []
    for k in range(64):
        nblocks = 16 + (k * 239) // 63
        tail = G.gen_stream(rng, rng.randint(1, 3000), "blocked", pad=None)
        while G.model_decode(tail.stream, len(tail.data))[0][0] != "Ok":
            tail = G.gen_stream(rng, rng.randint(1, 3000), "blocked", pad=None)
        bodies, data = _assemble(rng, block_pool, nblocks, tail)
        d = b"".join(data)
        streams.append(G.varint(len(d), rng.choice([None, 10])) + b"".join(bodies))
        datas.append(d)
    assert MIB <= min(map(len, datas)) and max(map(len, datas)) <= 16 * MIB
    for s, d in zip(streams[::9], datas[::9]):
        assert oracle.decompress(s) == d
    u = Units(streams, [len(d) for d in datas])
    rc, res, blocks, t_out = u.run(ws=True)
    assert rc == 0 and blocks == [(len(d) + BLOCK - 1) // BLOCK for d in datas]
    for i, d in enumerate(datas):
        assert res[i] == (("Ok", 0, 0, 0), len(d))
        want = torch.frombuffer(bytearray(d), dtype=torch.uint8).cuda()
        assert torch.equal(t_out[u.ooffs[i]:u.ooffs[i] + len(d)], want), i
    for s, d in zip(streams[::16], datas[::16]):
        assert snap.raw.Decoder().decompress_vec(s) == d
        st, out, nchunks = _device_ws(snap, s, len(d))
        assert st[0] == "Ok" and out == d and nchunks == (len(d) + BLOCK - 1) // BLOCK


def test_unblocked_64_mib_stream_is_declined_and_decoded(snap, oracle, block_pool):
    """The pool's blocks behind a 100-byte literal: every block boundary falls inside an element, and a final copy-4
    reaches 60 MB back. K8 declines; the one-warp decode must still give the oracle's bytes."""
    rng = random.Random(20)
    head = rng.randbytes(100)
    tail = G.gen_stream(rng, 500, "blocked")
    bodies, data = _assemble(rng, block_pool, 1024, tail)
    d = bytearray(head + b"".join(data))
    far = 60_000_000
    for _ in range(64):
        d.append(d[-far])
    d = bytes(d)
    s = G.varint(len(d)) + G.literal_header(100, "lit60") + head + b"".join(bodies) + G.copy_elem(64, far, "copy4")
    assert len(d) > 64 * MIB
    want = oracle.decompress(s)
    assert want == d
    st, out, nchunks = _device_ws(snap, s, len(d))
    assert st == ("Ok", 0, 0, 0) and nchunks == 0 and out == d
    assert snap.raw.Decoder().decompress_vec(s) == d
    rc, out = _uncompress(snap, s, len(d))
    assert rc == 0 and out == d
