"""K8 over a batch on the GPU: sb_decompress_batch_device_ws splits every unit of more than one block into its 64 KB
blocks and decodes the blocks of all units in one grid. Per-unit results must be those of sb_decompress_batch_device
(and the oracle's); clean multi-block units must take the parallel path (unit_blocks == blocks), all others one warp."""
import ctypes as C
import random

import numpy as np
import pytest

from conftest import corpus

pytestmark = pytest.mark.gpu

BLOCK = 65536
MIB = 1 << 20
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


def _lit(b):
    n = len(b) - 1
    if n < 60:
        return bytes([n << 2]) + b
    if n < 256:
        return bytes([60 << 2, n]) + b
    return bytes([61 << 2]) + n.to_bytes(2, "little") + b


class Units:
    """Streams packed into one device buffer (unit i at offs[i], start offset `off`), with per-unit outputs in another."""

    def __init__(self, streams, caps, off=0, out_off=0, even=False):
        """even: every unit in a slot of the same width (odd), as base + stride addressing needs."""
        import torch
        self.n = len(streams)
        self.lens = [len(s) for s in streams]
        self.caps = list(caps)
        iw, ow = (max(self.lens) + 7) | 1, (max(self.caps) + 21) | 1
        self.offs, at = [], off
        for s in streams:
            self.offs.append(at)
            at += iw if even else len(s) + 7
        host = np.zeros(at + 16, dtype=np.uint8)
        for o, s in zip(self.offs, streams):
            host[o:o + len(s)] = np.frombuffer(s, dtype=np.uint8)
        self.t_in = torch.from_numpy(host).cuda()
        self.ooffs, at = [], out_off
        for c in caps:
            self.ooffs.append(at)
            at += ow if even else c + 16 + 5
        self.out_total = at + 16

    def run(self, ws=True, addressing="ptrs", in_bytes=None, scratch_bytes=None, stream=None, blocks=True):
        """Returns rc, [(status tuple, bytes)] (bytes only for Ok), unit_blocks, the output tensor."""
        import torch
        import gpu_helpers
        s = gpu_helpers.snap()
        L = s._lib.lib()
        n = self.n
        t_out = torch.full((self.out_total,), 0xEE, dtype=torch.uint8, device="cuda")
        t_lens = torch.tensor(self.lens + [0], dtype=torch.int32, device="cuda")
        t_caps = torch.tensor(self.caps + [0], dtype=torch.int32, device="cuda")
        t_ol = torch.full((n + 1,), -1, dtype=torch.int32, device="cuda")
        t_st = torch.zeros((max(n, 1) * 32,), dtype=torch.uint8, device="cuda")
        t_blk = torch.full((n + 1,), -1, dtype=torch.int32, device="cuda")
        b = s._lib.SbBatch()
        if addressing == "ptrs":
            t_ip = torch.tensor([self.t_in.data_ptr() + o for o in self.offs] + [0], dtype=torch.int64, device="cuda")
            t_op = torch.tensor([t_out.data_ptr() + o for o in self.ooffs] + [0], dtype=torch.int64, device="cuda")
            b.in_ptrs, b.out_ptrs = t_ip.data_ptr(), t_op.data_ptr()
        else:                                  # base + stride: the units must be evenly spaced
            stride = self.offs[1] - self.offs[0] if n > 1 else 0
            ostride = self.ooffs[1] - self.ooffs[0] if n > 1 else 0
            assert all(self.offs[i] == self.offs[0] + i * stride for i in range(n))
            assert all(self.ooffs[i] == self.ooffs[0] + i * ostride for i in range(n))
            b.in_base, b.in_stride = self.t_in.data_ptr() + self.offs[0], stride
            b.out_base, b.out_stride = t_out.data_ptr() + self.ooffs[0], ostride
        b.in_lens, b.out_caps = t_lens.data_ptr(), t_caps.data_ptr()
        b.out_lens, b.statuses, b.count = t_ol.data_ptr(), t_st.data_ptr(), n
        e = s._lib.SbError()
        st = (stream or torch.cuda.current_stream()).cuda_stream
        t_scr = None
        if ws:
            ib = sum(self.lens) if in_bytes is None else in_bytes
            need = L.sb_decompress_batch_scratch_bytes(n, ib)
            sb = need if scratch_bytes is None else scratch_bytes
            t_scr = torch.full((sb + 4096,), 0x5A, dtype=torch.uint8, device="cuda")
            rc = L.sb_decompress_batch_device_ws(C.byref(b), ib, t_blk.data_ptr() if blocks else None, t_scr.data_ptr(), sb,
                                                 st, C.byref(e))
        else:
            rc = L.sb_decompress_batch_device(C.byref(b), st, C.byref(e))
        torch.cuda.synchronize()
        if rc:
            return rc, None, None, t_out
        if t_scr is not None:
            assert bool((t_scr[sb:] == 0x5A).all()), "scratch overrun"
        sts = np.frombuffer(t_st.cpu().numpy().tobytes(), dtype=np.uint64).reshape(-1, 4)
        ol = t_ol.cpu().numpy().astype(np.uint32)
        assert ol[n] == 0xFFFFFFFF
        res = []
        for i in range(n):
            code = int(sts[i][0] & 0xFFFFFFFF)
            if code == 0:
                res.append((("Ok", 0, 0, 0), int(ol[i])))
            else:
                res.append((gpu_helpers.err_tuple(s.error.from_c(s._lib.SbError(code, 0, int(sts[i][1]), int(sts[i][2]), int(sts[i][3])))),
                            None))
        return 0, res, [int(x) for x in t_blk.cpu().numpy()[:n]], t_out

    def out_bytes(self, t_out, i, length):
        return bytes(t_out[self.ooffs[i]:self.ooffs[i] + length].cpu().numpy())


def oracle_result(oracle, stream, cap):
    from oracle.oracle import OracleError
    try:
        return ("Ok", 0, 0, 0), oracle.decompress(stream, cap)
    except OracleError as e:
        return tuple(e.err), None


def _text(n, seed):
    base = corpus("alice29.txt") + corpus("lcet10.txt") + corpus("html_x_4") + corpus("kppkn.gtb")
    k = seed * 7919 % len(base)
    return ((base[k:] + base) * (n // len(base) + 2))[:n]


def _declined():
    rng = random.Random(11)
    head = bytes(rng.getrandbits(8) for _ in range(70000))
    blk = head[:BLOCK]
    near = varint(BLOCK + 120) + _lit(blk) + _lit(head[:100]) + bytes([(19 << 2) | 2]) + (1000).to_bytes(2, "little")
    data = bytes(rng.choice((0, 0, 1)) for _ in range(300000))
    parity = varint(len(data)) + b"".join(b"\x00" + bytes([c]) for c in data)
    d = head[:3 * 20000]
    straddle = varint(len(d) + 2 * BLOCK) + _lit(head[:65500]) + _lit(head[:100]) + _lit(head[:2 * BLOCK - 65600]) + _lit(d)
    return [near, parity, straddle]


def test_1mib_units_from_sb_compress_and_pyarrow(snap, oracle):
    import torch
    enc = snap.raw.Encoder()
    datas = [_text(MIB, i) for i in range(512)]
    streams = [enc.compress_vec(d) for d in datas]
    pa = pytest.importorskip("pyarrow")
    pages = [_text(MIB, 1000 + i) for i in range(32)]
    streams += [pa.compress(d, codec="snappy", asbytes=True) for d in pages]
    datas += pages
    u = Units(streams, [MIB] * len(streams))
    rc, res, blocks, t_out = u.run()
    assert rc == 0 and blocks == [16] * len(streams)
    assert all(r == (("Ok", 0, 0, 0), MIB) for r in res)
    want = torch.from_numpy(np.frombuffer(b"".join(datas), dtype=np.uint8).copy()).cuda().view(len(datas), MIB)
    got = torch.stack([t_out[o:o + MIB] for o in u.ooffs])
    assert torch.equal(got, want)


def test_mixed_batch_equals_batch_device(snap, oracle):
    """One 256 MiB unit among 65,536 units of 64 KB, with declined, corrupt and small units: every unit's bytes, status
    and length equal sb_decompress_batch_device's; the small ones also the oracle's."""
    import torch
    enc = snap.raw.Encoder()
    big = enc.compress_vec(_text(256 * MIB, 3))
    small_data = [_text(BLOCK, i) for i in range(64)]
    small = [enc.compress_vec(d) for d in small_data]
    good = enc.compress_vec(_text(5 * BLOCK + 99, 5))
    rng = random.Random(12)
    bad = []
    for _ in range(4):
        b = bytearray(good)
        b[rng.randrange(3, len(b))] ^= 1 << rng.randrange(8)
        bad.append(bytes(b))
    bad += [good[:len(good) // 2], good + b"\x00", varint(5 * BLOCK + 100) + good[3:], b"", b"\x00", b"\xff" * 6]
    odd = _declined() + bad + [oracle.compress(b"tiny unit")]
    streams = [small[i % 64] for i in range(65536)]
    streams[40000] = big
    for k, s in enumerate(odd):
        streams[100 + 977 * k] = s
    caps = [BLOCK] * 65536
    caps[40000] = 256 * MIB
    for k in range(len(odd)):
        caps[100 + 977 * k] = 400000
    u = Units(streams, caps)
    rc, res, blocks, t_out = u.run()
    assert rc == 0
    rc0, res0, _, t_out0 = u.run(ws=False)
    assert rc0 == 0 and res == res0
    assert blocks[40000] == 4096 and blocks[0] == 0
    # bytes past an error are unspecified: compare every other output byte for byte
    for k in range(len(odd)):
        i = 100 + 977 * k
        if res[i][0][0] != "Ok":
            t_out[u.ooffs[i]:u.ooffs[i] + caps[i]] = 0
            t_out0[u.ooffs[i]:u.ooffs[i] + caps[i]] = 0
    assert torch.equal(t_out, t_out0)
    for k, s in enumerate(odd):
        i = 100 + 977 * k
        want_st, want = oracle_result(oracle, s, 400000)
        assert res[i][0] == want_st, k
        if want is not None:
            assert u.out_bytes(t_out, i, res[i][1]) == want, k
    for i in range(0, 64):
        assert res[i] == (("Ok", 0, 0, 0), BLOCK) and u.out_bytes(t_out, i, BLOCK) == small_data[i % 64]


@pytest.mark.parametrize("addressing", ["ptrs", "base"])
def test_unaligned_buffers(snap, oracle, addressing):
    import torch
    datas = [_text(13 * BLOCK + 7, 1), _text(3 * BLOCK, 2), _text(500, 3), _text(2 * BLOCK + 1, 4)]
    streams = [oracle.compress(d) for d in datas]
    caps = [len(d) for d in datas]
    for off in range(1, 16):
        u = Units(streams, caps, off=off, out_off=16 - off, even=addressing == "base")
        rc, res, blocks, t_out = u.run(addressing=addressing)
        assert rc == 0 and blocks == [14, 3, 0, 3], off
        for i, d in enumerate(datas):
            assert res[i] == (("Ok", 0, 0, 0), len(d)) and u.out_bytes(t_out, i, len(d)) == d, (off, i)
            assert u.out_bytes(t_out, i, len(d) + 16)[len(d):] == b"\xee" * 16


def test_count_zero_and_one(snap, oracle):
    import torch
    L = snap._lib.lib()
    b = snap._lib.SbBatch()
    t_ol = torch.zeros(4, dtype=torch.int32, device="cuda")
    b.out_lens, b.count = t_ol.data_ptr(), 0
    e = snap._lib.SbError()
    t_scr = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    before = L.sb_launch_count()
    assert L.sb_decompress_batch_device_ws(C.byref(b), 0, None, t_scr.data_ptr(), 4096, None, C.byref(e)) == 0
    assert L.sb_launch_count() == before
    for s, cap in ((oracle.compress(_text(7 * BLOCK + 3, 9)), 7 * BLOCK + 3), (_declined()[1], 300000),
                   (oracle.compress(_text(7 * BLOCK + 3, 9))[:-5], 7 * BLOCK + 3)):
        u = Units([s], [cap])
        rc, res, blocks, t_out = u.run()
        assert rc == 0
        t_in = torch.frombuffer(bytearray(s + bytes(16)), dtype=torch.uint8).cuda()
        t_o2 = torch.full((cap + 16,), 0xEE, dtype=torch.uint8, device="cuda")
        need = L.sb_decompress_scratch_bytes(len(s))
        t_s2 = torch.empty(need, dtype=torch.uint8, device="cuda")
        t_res = torch.zeros(64, dtype=torch.uint8, device="cuda")
        assert L.sb_decompress_device_ws(t_in.data_ptr(), len(s), t_o2.data_ptr(), cap, t_res.data_ptr(), t_s2.data_ptr(), need,
                                         None, C.byref(e)) == 0
        torch.cuda.synchronize()
        r = snap._lib.SbFrameResult.from_buffer_copy(bytes(t_res.cpu().numpy()[:C.sizeof(snap._lib.SbFrameResult)]))
        import gpu_helpers
        want_st = ("Ok", 0, 0, 0) if r.status.code == 0 else gpu_helpers.err_tuple(snap.error.from_c(r.status))
        assert res[0][0] == want_st and blocks[0] == r.nchunks
        if r.status.code == 0:
            assert res[0][1] == r.bytes and u.out_bytes(t_out, 0, r.bytes) == bytes(t_o2[:r.bytes].cpu().numpy())


def test_short_scratch_and_underestimated_in_bytes(snap, oracle):
    streams = [oracle.compress(_text(4 * BLOCK + i, i)) for i in range(5)] + [oracle.compress(b"abc")]
    caps = [4 * BLOCK + i for i in range(5)] + [3]
    u = Units(streams, caps)
    L = snap._lib.lib()
    total = sum(len(s) for s in streams)
    need = L.sb_decompress_batch_scratch_bytes(len(streams), total)
    before = L.sb_launch_count()
    rc, _, _, _ = u.run(scratch_bytes=need - 1)
    assert rc == INVALID and L.sb_launch_count() == before
    rc, res, blocks, t_out = u.run(in_bytes=total - 1)
    assert rc == 0 and blocks == [0] * 6
    rc, res2, blocks2, t_out2 = u.run()
    assert rc == 0 and blocks2 == [4, 5, 5, 5, 5, 0]
    assert res == res2
    for i, s in enumerate(streams):
        want = oracle.decompress(s)
        assert u.out_bytes(t_out, i, len(want)) == want == u.out_bytes(t_out2, i, len(want))


def test_host_batch_with_multi_block_units(snap, oracle):
    import gpu_helpers
    datas = [_text(3 * BLOCK + 17 * i, i) for i in range(6)] + [_text(1000, 7), b""]
    streams = [oracle.compress(d) for d in datas] + [_declined()[0], b"\xff\xff"]
    caps = [len(d) for d in datas] + [BLOCK + 120, 100]
    got = gpu_helpers.decompress_batch_host(streams, caps)
    for i, s in enumerate(streams):
        want_st, want = oracle_result(oracle, s, caps[i])
        assert got[i][0] == want_st, i
        if want is not None:
            assert got[i][1] == want, i
    L = snap._lib.lib()
    e = snap._lib.SbError()
    assert L.sb_reserve(64, 64 * MIB, 64 * MIB, C.byref(e)) == 0
    before = L.sb_alloc_count()
    for _ in range(3):
        assert gpu_helpers.decompress_batch_host(streams, caps) == got
    assert L.sb_alloc_count() == before


def test_enqueued_behind_pending_work_on_a_side_stream(snap, oracle):
    import torch
    datas = [_text(9 * BLOCK + i, i) for i in range(8)]
    streams = [oracle.compress(d) for d in datas]
    u = Units(streams, [len(d) for d in datas])
    _, res0, blocks0, t0 = u.run()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)
        _, res, blocks, t1 = u.run(stream=side)
    assert res == res0 and blocks == blocks0 == [9] + [10] * 7
    assert torch.equal(t0, t1)
