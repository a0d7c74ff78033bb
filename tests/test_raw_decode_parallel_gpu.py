"""K8 on the GPU: large raw streams split into their 64 KB blocks and decoded in parallel, through sb_decompress /
raw.Decoder and through sb_decompress_device_ws. Clean streams must take the parallel path (nchunks == blocks), every
other stream the one-warp path with the oracle's exact bytes or error."""
import ctypes as C
import random

import numpy as np
import pytest

from conftest import corpus

pytestmark = pytest.mark.gpu

BLOCK = 65536
INVALID = 202


@pytest.fixture(scope="module")
def snap():
    import torch
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)
    import gpu_helpers
    return gpu_helpers.snap()


def varint(v):
    out = b""
    while v >= 0x80:
        out += bytes([v & 0x7F | 0x80])
        v >>= 7
    return out + bytes([v])


def to_dev(b, pad=16, off=0):
    import torch
    t = torch.empty(off + len(b) + pad, dtype=torch.uint8, device="cuda")
    t[off:off + len(b)] = torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda() if len(b) else t[off:off]
    return t


def decode_ws(snap, t_in, n, cap, in_off=0, out_off=0, scratch_bytes=None):
    """sb_decompress_device_ws over device buffers: (rc, result record, output tensor)."""
    import torch
    L = snap._lib.lib()
    t_out = torch.full((out_off + cap + 16,), 0xEE, dtype=torch.uint8, device="cuda")
    need = L.sb_decompress_scratch_bytes(n)
    sb = need if scratch_bytes is None else scratch_bytes
    t_scr = torch.empty(max(sb, 1), dtype=torch.uint8, device="cuda")
    t_res = torch.zeros(64, dtype=torch.uint8, device="cuda")
    e = snap._lib.SbError()
    rc = L.sb_decompress_device_ws(t_in.data_ptr() + in_off, n, t_out.data_ptr() + out_off, cap, t_res.data_ptr(),
                                   t_scr.data_ptr(), sb, torch.cuda.current_stream().cuda_stream, C.byref(e))
    torch.cuda.synchronize()
    res = snap._lib.SbFrameResult.from_buffer_copy(bytes(t_res.cpu().numpy()[:C.sizeof(snap._lib.SbFrameResult)]))
    if rc == 0:
        assert bytes(t_out[out_off + cap:out_off + cap + 16].cpu().numpy()) == b"\xee" * 16
    return rc, res, t_out[out_off:out_off + cap]


def status(snap, res):
    import gpu_helpers
    return ("Ok", 0, 0, 0) if res.status.code == 0 else gpu_helpers.err_tuple(snap.error.from_c(res.status))


def oracle_result(oracle, stream, cap):
    from oracle.oracle import OracleError
    try:
        return ("Ok", 0, 0, 0), oracle.decompress(stream, cap)
    except OracleError as e:
        return tuple(e.err), None


def host_decode(snap, stream):
    import gpu_helpers
    try:
        return ("Ok", 0, 0, 0), snap.raw.Decoder().decompress_vec(stream)
    except Exception as e:  # noqa: BLE001
        return gpu_helpers.err_tuple(e), None


def check_parallel_ws(snap, comp, data_t):
    """comp: host bytes or a device tensor of the stream; data_t: the expected output on the device."""
    import torch
    t_in = comp if isinstance(comp, torch.Tensor) else to_dev(comp)
    n = t_in.numel() - 16 if not isinstance(comp, torch.Tensor) else comp.numel()
    dn = data_t.numel()
    rc, res, out = decode_ws(snap, t_in, n, dn)
    assert rc == 0 and res.status.code == 0 and res.bytes == dn
    assert res.nchunks == (dn + BLOCK - 1) // BLOCK
    assert torch.equal(out, data_t)


def _tiled(b, n):
    return np.resize(np.frombuffer(b, dtype=np.uint8), n)


def _host_compress(snap, arr):
    """sb_compress over a numpy array (no bytes copies of large inputs)."""
    L = snap._lib.lib()
    cap = L.sb_max_compress_len(arr.size)
    out = np.empty(cap, dtype=np.uint8)
    n = C.c_size_t(0)
    e = snap._lib.SbError()
    assert L.sb_compress(arr.ctypes.data, arr.size, out.ctypes.data, cap, C.byref(n), C.byref(e)) == 0
    return out[:n.value]


def test_24mb_mixed_stream(snap, oracle):
    import torch
    data = (corpus("lcet10.txt") + corpus("kppkn.gtb") + corpus("html_x_4")) * 24
    comp = snap.raw.Encoder().compress_vec(data)
    assert host_decode(snap, comp) == (("Ok", 0, 0, 0), data)
    check_parallel_ws(snap, comp, torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda())


def test_100mb_pyarrow_stream(snap):
    import torch
    pa = pytest.importorskip("pyarrow")
    base = corpus("alice29.txt") + corpus("html") + corpus("kppkn.gtb") + corpus("urls.10K")
    data = (base * (100 * 1000 * 1000 // len(base) + 1))[:100 * 1000 * 1000]
    comp = pa.compress(data, codec="snappy", asbytes=True)
    assert snap.raw.Decoder().decompress_vec(comp) == data
    check_parallel_ws(snap, comp, torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda())


@pytest.mark.parametrize("name,size", [("text", (1 << 30) + 12345), ("fireworks.jpeg", 256 << 20)])
def test_large_streams_from_sb_compress(snap, name, size):
    import torch
    base = corpus("alice29.txt") + corpus("lcet10.txt") + corpus("html_x_4") if name == "text" else corpus(name)
    arr = _tiled(base, size)
    comp = _host_compress(snap, arr)
    t_in = torch.from_numpy(comp).cuda()
    check_parallel_ws(snap, t_in, torch.from_numpy(arr).cuda())


@pytest.mark.parametrize("kind", ["zeros", "text"])
def test_output_of_4gib_minus_one(snap, oracle, kind):
    """dn = 2^32 - 1: one block's body repeated 65535 times behind the header, then a 65,535-byte last block."""
    import torch
    blk = b"\0" * BLOCK if kind == "zeros" else _tiled(corpus("alice29.txt")[:1000], BLOCK).tobytes()
    body = oracle.compress(blk)[len(varint(BLOCK)):]
    last = blk[:BLOCK - 1]
    last_body = oracle.compress(last)[len(varint(BLOCK - 1)):]
    dn = (1 << 32) - 1
    head = varint(dn)
    n = len(head) + len(body) * 65535 + len(last_body)
    t_in = torch.empty(n + 16, dtype=torch.uint8, device="cuda")
    t_in[:len(head)] = torch.tensor(list(head), dtype=torch.uint8)
    t_in[len(head):len(head) + len(body) * 65535].view(65535, len(body))[:] = \
        torch.frombuffer(bytearray(body), dtype=torch.uint8).cuda()
    t_in[n - len(last_body):n] = torch.frombuffer(bytearray(last_body), dtype=torch.uint8).cuda()
    rc, res, out = decode_ws(snap, t_in, n, dn)
    assert rc == 0 and res.status.code == 0 and res.bytes == dn and res.nchunks == 65536
    b = torch.frombuffer(bytearray(blk), dtype=torch.uint8).cuda()
    assert torch.equal(out[:65535 * BLOCK].view(65535, BLOCK), b.expand(65535, BLOCK))
    assert torch.equal(out[65535 * BLOCK:], b[:BLOCK - 1])
    del out, t_in
    torch.cuda.empty_cache()


def _lit(b):
    n = len(b) - 1
    if n < 60:
        return bytes([n << 2]) + b
    if n < 256:
        return bytes([60 << 2, n]) + b
    return bytes([61 << 2]) + n.to_bytes(2, "little") + b


def _declined_streams():
    rng = random.Random(11)
    head = bytes(rng.getrandbits(8) for _ in range(70000))
    want = head + head[:40] + head[100:131] + head[65500:65560]
    lits = b"".join(_lit(head[i:i + 60]) for i in range(0, len(head), 60))
    c4 = lambda ln, off: bytes([((ln - 1) << 2) | 3]) + off.to_bytes(4, "little")  # noqa: E731
    far = varint(len(want)) + lits + c4(40, 70000) + c4(31, 70040 - 100) + c4(60, 70071 - 65500)
    blk = head[:BLOCK]
    near = varint(BLOCK + 120) + _lit(blk) + _lit(head[:100]) + bytes([(19 << 2) | 2]) + (1000).to_bytes(2, "little")
    data = bytes(rng.choice((0, 0, 1)) for _ in range(300000))
    parity = varint(len(data)) + b"".join(b"\x00" + bytes([c]) for c in data)
    big = 140000
    longlit = varint(big) + bytes([62 << 2]) + (big - 1).to_bytes(3, "little") + (head * 2)[:big]
    return {"far offsets": far, "near copy into previous block": near, "parity": parity, "long literal": longlit}


def test_declined_streams_take_the_one_warp_path(snap, oracle):
    good = oracle.compress((corpus("lcet10.txt") * 2)[:5 * BLOCK + 99])
    rng = random.Random(12)
    streams = dict(_declined_streams())
    for i in range(6):
        b = bytearray(good)
        b[rng.randrange(3, len(b))] ^= 1 << rng.randrange(8)
        streams["flip %d" % i] = bytes(b)
    streams["truncated"] = good[:len(good) // 2]
    streams["trailing"] = good + b"\x00"
    streams["header +1"] = varint(5 * BLOCK + 100) + good[3:]
    for name, s in streams.items():
        cap = 400000
        want_st, want = oracle_result(oracle, s, cap)
        rc, res, out = decode_ws(snap, to_dev(s), len(s), cap)
        assert rc == 0 and status(snap, res) == want_st, name
        if want is None or not name.startswith("flip"):                # a flipped literal byte is still a clean stream
            assert res.nchunks == 0, name
        if want is not None:
            assert res.bytes == len(want) and bytes(out[:len(want)].cpu().numpy()) == want, name
        from oracle.oracle import OracleError
        try:
            host_want = (("Ok", 0, 0, 0), oracle.decompress(s))
        except OracleError as e:
            host_want = (tuple(e.err), None)
        assert host_decode(snap, s) == host_want, name


def test_unaligned_buffers(snap, oracle):
    import torch
    data = (corpus("html_x_4") * 3)[:13 * BLOCK + 7]
    comp = oracle.compress(data)
    want = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    for off in range(1, 16):
        t_in = to_dev(comp, off=off)
        rc, res, out = decode_ws(snap, t_in, len(comp), len(data), in_off=off, out_off=16 - off)
        assert rc == 0 and res.status.code == 0 and res.nchunks == 14 and torch.equal(out, want), off


def test_cap_above_and_below_dn(snap, oracle):
    import torch
    data = (corpus("kppkn.gtb") * 4)[:6 * BLOCK + 5]
    comp = oracle.compress(data)
    t_in = to_dev(comp)
    rc, res, out = decode_ws(snap, t_in, len(comp), len(data) + 1000)
    assert rc == 0 and res.status.code == 0 and res.bytes == len(data) and res.nchunks == 7
    assert torch.equal(out[:len(data)], torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda())
    rc, res, _ = decode_ws(snap, t_in, len(comp), len(data) - 1)
    assert rc == 0 and res.nchunks == 0 and res.bytes == 0
    assert status(snap, res) == oracle_result(oracle, comp, len(data) - 1)[0] == ("BufferTooSmall", len(data) - 1, len(data), 0)


def test_scratch_one_byte_short(snap, oracle):
    L = snap._lib.lib()
    comp = oracle.compress(corpus("lcet10.txt"))
    need = L.sb_decompress_scratch_bytes(len(comp))
    rc, _, _ = decode_ws(snap, to_dev(comp), len(comp), 500000, scratch_bytes=need - 1)
    assert rc == INVALID


def test_repeated_host_decodes_allocate_nothing(snap):
    data = (corpus("lcet10.txt") + corpus("kppkn.gtb") + corpus("html_x_4")) * 24
    comp = snap.raw.Encoder().compress_vec(data)
    L = snap._lib.lib()
    dec = snap.raw.Decoder()
    assert dec.decompress_vec(comp) == data
    before = L.sb_alloc_count()
    for _ in range(3):
        assert dec.decompress_vec(comp) == data
    assert L.sb_alloc_count() == before
