"""Frame decode of a batch of streams on the GPU (sb_frame_decode_batch_device_ws): every unit's chunk index is built by K7
or checked against the caller's, and the chunks of all units are decoded in one grid. Every unit must give exactly what
sb_frame_decode_device_ws gives it (status, bytes produced, output) and, where it applies, what the oracle's
frame_decode gives; d_unit_chunks must show which path ran."""
import ctypes as C
import random

import numpy as np
import pytest

import legal_streams as ls
from conftest import corpus
from test_frame_batch_decode_emu import chain, data_chunks, mixed_streams, oracle_decode

pytestmark = pytest.mark.gpu

BLOCK = 65536
MIB = 1 << 20
INVALID = 202
NAMES = {0: "Ok", 1: "TooBig", 2: "BufferTooSmall", 4: "Header", 6: "Literal", 7: "CopyRead", 8: "CopyWrite", 9: "Offset",
         10: "StreamHeader", 11: "StreamHeaderMismatch", 12: "UnsupportedChunkType", 13: "UnsupportedChunkLength",
         14: "Checksum", 100: "UnexpectedEof", 202: "Invalid"}


@pytest.fixture(scope="module")
def snap():
    import torch
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)
    import gpu_helpers
    return gpu_helpers.snap()


def _text(n, seed):
    base = corpus("alice29.txt") + corpus("lcet10.txt") + corpus("html_x_4") + corpus("kppkn.gtb")
    k = seed * 7919 % len(base)
    return ((base[k:] + base) * (n // len(base) + 2))[:n]


def _u32(values):
    import torch
    return torch.from_numpy(np.array(values, dtype=np.uint32).view(np.int32)).cuda()


def _status(row):
    code = int(row[0] & 0xFFFFFFFF)
    return (NAMES.get(code, str(code)), int(row[1]), int(row[2]), int(row[3]))


class Batch:
    """Streams packed into one device input buffer at odd offsets, outputs of cap + 16 guard bytes at odd offsets."""

    def __init__(self, streams, caps, off=1):
        import torch
        self.streams, self.caps = streams, list(caps)
        self.lens = [len(s) for s in streams]
        iw, ow = (max(self.lens + [1]) + 7) | 1, (max(self.caps + [1]) + 21) | 1
        self.iw, self.ow, self.off = iw, ow, off
        host = np.zeros(off + iw * len(streams) + 16, dtype=np.uint8)
        for i, s in enumerate(streams):
            host[off + i * iw:off + i * iw + len(s)] = np.frombuffer(s, dtype=np.uint8)
        self.t_in = torch.from_numpy(host).cuda()
        self.t_out = torch.full((3 + ow * len(streams) + 16,), 0xEE, dtype=torch.uint8, device="cuda")
        self.in_ptrs = [self.t_in.data_ptr() + off + i * iw for i in range(len(streams))]
        self.out_ptrs = [self.t_out.data_ptr() + 3 + i * ow for i in range(len(streams))]

    def output(self, i, k):
        o = 3 + i * self.ow
        return self.t_out[o:o + k].cpu().numpy().tobytes()

    def guards_untouched(self):
        back = self.t_out.cpu().numpy()
        return all((back[3 + i * self.ow + c:3 + i * self.ow + c + 16] == 0xEE).all() for i, c in enumerate(self.caps))


def index_arrays(indexes, base=0):
    import torch
    flat, at = [7] * base, []
    for ix in indexes:
        at.append(len(flat))
        flat += list(ix)
    at.append(len(flat))
    to64 = lambda v: torch.from_numpy(np.array(v, dtype=np.uint64).view(np.int64)).cuda()
    return to64(flat + [0]), to64(at)


def decode_ws(snap, bt, flags=0, index=None, max_chunks=None, in_bytes=None, scratch_bytes=None, stream=None,
              addressing="ptrs", uniform=False, sync=True):
    """One sb_frame_decode_batch_device_ws call over a Batch. Returns rc, [(status, bytes)], d_unit_chunks."""
    import torch
    L = snap._lib.lib()
    n = len(bt.streams)
    if in_bytes is None:
        in_bytes = sum(bt.lens)
    if max_chunks is None:
        max_chunks = sum(k // 8 + 2 for k in bt.lens)
    t_ol = torch.full((n + 1,), -1, dtype=torch.int32, device="cuda")
    t_uc = torch.full((n + 1,), -1, dtype=torch.int32, device="cuda")
    t_st = torch.full((max(n, 1) * 32,), 0x77, dtype=torch.uint8, device="cuda")
    b = snap._lib.SbBatch()
    if addressing == "ptrs":
        t_ip = torch.tensor(bt.in_ptrs + [0], dtype=torch.int64, device="cuda")
        t_op = torch.tensor(bt.out_ptrs + [0], dtype=torch.int64, device="cuda")
        b.in_ptrs, b.out_ptrs = t_ip.data_ptr(), t_op.data_ptr()
    else:
        b.in_base, b.in_stride = bt.in_ptrs[0], bt.iw
        b.out_base, b.out_stride = bt.out_ptrs[0], bt.ow
    if uniform:
        b.in_len_uniform, b.out_cap_uniform = bt.lens[0], bt.caps[0]
    else:
        t_lens, t_caps = _u32(bt.lens + [0]), _u32(bt.caps + [0])
        b.in_lens, b.out_caps = t_lens.data_ptr(), t_caps.data_ptr()
    b.out_lens, b.statuses, b.count = t_ol.data_ptr(), t_st.data_ptr(), n
    cidx, cat = index_arrays(index) if index is not None else (None, None)
    need = L.sb_frame_decode_batch_scratch_bytes(n, in_bytes, max_chunks)
    sb = need if scratch_bytes is None else scratch_bytes
    t_scr = torch.full((sb + 4096,), 0x5A, dtype=torch.uint8, device="cuda")
    e = snap._lib.SbError()
    st = (stream or torch.cuda.current_stream()).cuda_stream
    rc = L.sb_frame_decode_batch_device_ws(C.byref(b), in_bytes, flags, cidx.data_ptr() if cidx is not None else None,
                                           cat.data_ptr() if cat is not None else None, max_chunks, t_uc.data_ptr(),
                                           t_scr.data_ptr(), sb, st, C.byref(e))
    if not sync:
        return rc, (t_ol, t_st, t_uc, t_scr, cidx, cat)
    torch.cuda.synchronize()
    if rc:
        assert bool((t_ol == -1).all()) and bool((t_st == 0x77).all()) and bool((t_uc == -1).all())
        return rc, None, None
    assert bool((t_scr[sb:] == 0x5A).all()), "scratch overrun"
    assert bt.guards_untouched(), "output overrun"
    ol = t_ol.cpu().numpy().view(np.uint32)
    uc = t_uc.cpu().numpy().view(np.uint32)
    assert ol[n] == 0xFFFFFFFF and uc[n] == 0xFFFFFFFF
    sts = np.frombuffer(t_st.cpu().numpy().tobytes(), dtype=np.uint64).reshape(-1, 4)
    return rc, [(_status(sts[i]), bt.output(i, int(ol[i]))) for i in range(n)], [int(x) for x in uc[:n]]


def single(snap, stream, cap, flags=0, index=None):
    """sb_frame_decode_device_ws of one stream with a chunk table large enough: (status, bytes)."""
    import torch
    L = snap._lib.lib()
    n = len(stream)
    t_in = torch.from_numpy(np.frombuffer(stream + b"\0", dtype=np.uint8).copy()).cuda()
    t_out = torch.zeros(cap + 1, dtype=torch.uint8, device="cuda")
    maxc = n // 8 + 16
    t_ws = torch.empty(L.sb_frame_decode_scratch_bytes(maxc), dtype=torch.uint8, device="cuda")
    t_res = torch.zeros(48, dtype=torch.uint8, device="cuda")
    t_ix = torch.from_numpy(np.array(index, dtype=np.uint64).view(np.int64)).cuda() if index is not None else None
    e = snap._lib.SbError()
    rc = L.sb_frame_decode_device_ws(t_in.data_ptr(), n, t_out.data_ptr(), cap, t_ix.data_ptr() if t_ix is not None else None,
                                     len(index) - 1 if index is not None else 0, flags, t_res.data_ptr(), t_ws.data_ptr(),
                                     t_ws.numel(), maxc, torch.cuda.current_stream().cuda_stream, C.byref(e))
    assert rc == 0
    torch.cuda.synchronize()
    r = np.frombuffer(t_res.cpu().numpy().tobytes(), dtype=np.uint64)
    return _status(r[:4]), t_out[:int(r[4])].cpu().numpy().tobytes()


def check(snap, oracle, streams, caps=None, flags=0, index=None, **kw):
    if caps is None:
        caps = [len(single(snap, s, 1 << 24, flags)[1]) + 5 for s in streams]
    bt = Batch(streams, caps)
    rc, res, uc = decode_ws(snap, bt, flags=flags, index=index, **kw)
    assert rc == 0
    for i, s in enumerate(streams):
        want = single(snap, s, caps[i], flags)
        assert res[i] == want, (i, len(s), res[i][0], want[0])
        if not flags & 1 and want[0][0] != "BufferTooSmall" and oracle is not None:
            ost, odata = oracle_decode(oracle, s)
            assert res[i][0] == ost, (i, res[i][0], ost)
            if odata is not None:
                assert res[i][1] == odata
    return res, uc


@pytest.mark.parametrize("indexed", [False, True])
def test_mixed_batch_matches_single_stream_decoder_and_oracle(snap, oracle, indexed):
    units = mixed_streams(oracle)
    streams = [s for s, _ in units]
    index = [chain(s) if s else [0] for s in streams] if indexed else None
    res, uc = check(snap, oracle, streams, index=index)
    for i, (s, clean) in enumerate(units):
        if not clean:
            assert uc[i] == 0, i
        elif res[i][0][0] == "Ok" and i < len(units) - 4:
            assert uc[i] == data_chunks(s), i


def test_wrong_caller_index(snap, oracle):
    good = [oracle.frame_encode(_text(n, n)) for n in (70000, 200000, 140000, 30000, 9000)]
    wrong = [list(chain(s)) for s in good]
    wrong[0][1] += 1
    wrong[1][-1] -= 1
    del wrong[2][1]
    wrong[3] = [123456789, 5, 77]
    res0, uc0 = check(snap, oracle, good, index=[chain(s) for s in good])
    res, uc = check(snap, oracle, good, index=wrong)
    assert res == res0 and uc == [0, 0, 0, 0, data_chunks(good[4])] and uc0 == [data_chunks(s) for s in good]


def test_fragments(snap, oracle):
    rng = random.Random(5)
    frags = [oracle.frame_encode(_text(n, n))[10:] for n in (1, 65536, 300000)]
    frags += [b"", ls.gen_frame(rng, oracle.crc32c_masked, 9).stream[10:]]
    res, uc = check(snap, None, frags, flags=1)
    assert [r[0][0] for r in res] == ["Ok"] * 5 and uc == [1, 1, 5, 0, 0]


def test_chunk_table_one_short_and_caps_one_byte_short(snap, oracle):
    datas = [_text(n, n) for n in (100000, 5000, 200000, 70000)]
    streams = [oracle.frame_encode(d) for d in datas]
    need = [data_chunks(s) for s in streams]
    mc = sum(need[:3]) - 1
    bt = Batch(streams, [len(d) for d in datas])
    _, res, _ = decode_ws(snap, bt, max_chunks=mc)
    assert [r[1] for r in res[:2]] == datas[:2]
    assert all(r == (("Invalid", mc, 1, 0), b"") for r in res[2:])
    bt = Batch(streams, [len(d) - 1 for d in datas])
    _, res, _ = decode_ws(snap, bt, index=[chain(s) for s in streams])
    assert res == [(("BufferTooSmall", len(d) - 1, len(d), 0), b"") for d in datas]


def test_in_bytes_underestimated(snap, oracle):
    streams = [s for s, _ in mixed_streams(oracle)]
    res0, _ = check(snap, oracle, streams)
    res, uc = check(snap, oracle, streams, in_bytes=sum(len(s) for s in streams) - 1)
    assert res == res0 and uc == [0] * len(streams)


def _k10_encode(snap, datas, index=True):
    """sb_frame_encode_batch_device_ws of the datas: (streams, per-unit index lists)."""
    import torch
    L = snap._lib.lib()
    lens = [len(d) for d in datas]
    caps = [10 + (k + BLOCK - 1) // BLOCK * (8 + 76490) for k in lens]
    bt = Batch(datas, caps)
    t_ol = torch.zeros(len(datas), dtype=torch.int32, device="cuda")
    nidx = sum((k + BLOCK - 1) // BLOCK + 1 for k in lens)
    t_idx = torch.zeros(nidx, dtype=torch.int64, device="cuda")
    t_ip = torch.tensor(bt.in_ptrs, dtype=torch.int64, device="cuda")
    t_op = torch.tensor(bt.out_ptrs, dtype=torch.int64, device="cuda")
    t_l, t_c = _u32(lens), _u32(caps)
    b = snap._lib.SbBatch()
    b.in_ptrs, b.out_ptrs, b.in_lens, b.out_caps = t_ip.data_ptr(), t_op.data_ptr(), t_l.data_ptr(), t_c.data_ptr()
    b.out_lens, b.count = t_ol.data_ptr(), len(datas)
    in_bytes = sum(k for k in lens if k > BLOCK)
    need = L.sb_frame_encode_batch_scratch_bytes(len(datas), in_bytes)
    t_scr = torch.empty(need, dtype=torch.uint8, device="cuda")
    e = snap._lib.SbError()
    assert L.sb_frame_encode_batch_device_ws(C.byref(b), in_bytes, t_idx.data_ptr(), t_scr.data_ptr(), need,
                                             torch.cuda.current_stream().cuda_stream, C.byref(e)) == 0
    torch.cuda.synchronize()
    ol = t_ol.cpu().numpy().view(np.uint32)
    streams = [bt.output(i, int(ol[i])) for i in range(len(datas))]
    ix, at = [], 0
    allix = t_idx.cpu().numpy().view(np.uint64)
    for k in lens:
        m = (k + BLOCK - 1) // BLOCK + 1
        ix.append([int(x) for x in allix[at:at + m]])
        at += m
    return streams, ix


@pytest.mark.parametrize("kind", ["512x1MiB", "mixed"])
def test_round_trip_of_the_batch_encoder(snap, oracle, kind):
    if kind == "512x1MiB":
        datas = [_text(MIB, s) for s in range(512)]
    else:
        rng = random.Random(3)
        datas = [_text(rng.choice([0, 1, 100, BLOCK - 1, BLOCK, BLOCK + 1, 300000, 2 * MIB + 7]), s) for s in range(300)]
    streams, ix = _k10_encode(snap, datas)
    assert all(x == (chain(s) if s else [0]) for x, s in zip(ix, streams))
    caps = [len(d) for d in datas]
    for index in (None, ix):
        bt = Batch(streams, caps)
        rc, res, uc = decode_ws(snap, bt, index=index, max_chunks=sum(len(x) - 1 for x in ix))
        assert rc == 0
        assert [r[1] for r in res] == datas
        assert all(r[0] == ("Ok", 0, 0, 0) for r in res)
        assert uc == [len(x) - 1 for x in ix]
    for i in range(0, len(datas), 37):
        assert single(snap, streams[i], caps[i]) == (("Ok", 0, 0, 0), datas[i])


@pytest.mark.parametrize("addressing,uniform", [("ptrs", False), ("base", False), ("base", True), ("ptrs", True)])
def test_addressing_on_unaligned_buffers(snap, oracle, addressing, uniform):
    datas = [_text(150001, s) for s in range(5)]
    streams = [oracle.frame_encode(d) for d in datas]
    if uniform:
        n = min(len(s) for s in streams)
        streams = [s[:n] for s in streams]
    caps = [150001] * 5
    bt = Batch(streams, caps, off=3)
    rc, res, _ = decode_ws(snap, bt, addressing=addressing, uniform=uniform)
    for i, s in enumerate(streams):
        assert res[i] == single(snap, s, caps[i])


def test_call_level_checks(snap, oracle):
    import torch
    L = snap._lib.lib()
    s = oracle.frame_encode(_text(1000, 1))
    bt = Batch([s], [2000])
    assert decode_ws(snap, bt, scratch_bytes=L.sb_frame_decode_batch_scratch_bytes(1, len(s), 129) - 1)[0] == INVALID
    assert decode_ws(snap, bt, max_chunks=0)[0] == INVALID
    assert decode_ws(snap, bt, max_chunks=1 << 22)[0] == INVALID
    e = snap._lib.SbError()
    t = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    b = snap._lib.SbBatch()
    b.count = 0
    assert L.sb_frame_decode_batch_device_ws(None, 0, 0, None, None, 8, None, t.data_ptr(), 1 << 16, None, C.byref(e)) == INVALID
    assert L.sb_frame_decode_batch_device_ws(C.byref(b), 0, 0, None, None, 8, None, t.data_ptr(), 1 << 16, None, C.byref(e)) == INVALID
    b.out_lens, b.statuses = t.data_ptr(), t.data_ptr() + 4096
    assert L.sb_frame_decode_batch_device_ws(C.byref(b), 0, 0, None, None, 8, None, t.data_ptr(), 1 << 16, None, C.byref(e)) == 0
    assert L.sb_frame_decode_batch_device_ws(C.byref(b), 0, 0, t.data_ptr(), None, 8, None, t.data_ptr(), 1 << 16, None,
                                             C.byref(e)) == INVALID
    b.count = 1 << 31
    assert L.sb_frame_decode_batch_device_ws(C.byref(b), 0, 0, None, None, 8, None, t.data_ptr(), 1 << 16, None, C.byref(e)) == INVALID


def test_enqueued_behind_pending_work_on_a_side_stream(snap, oracle):
    import torch
    datas = [_text(300000, s) for s in range(8)]
    streams = [oracle.frame_encode(d) for d in datas]
    bt = Batch(streams, [len(d) for d in datas])
    side = torch.cuda.Stream()
    big = torch.empty(1 << 28, dtype=torch.uint8, device="cuda")
    with torch.cuda.stream(side):
        for _ in range(4):
            big.fill_(1)                                               # pending work ahead of the call
        rc, keep = decode_ws(snap, bt, stream=side, sync=False)
    assert rc == 0
    side.synchronize()
    ol = keep[0].cpu().numpy().view(np.uint32)
    assert [bt.output(i, int(ol[i])) for i in range(len(datas))] == datas


def test_no_allocation_and_fixed_launch_count(snap, oracle):
    L = snap._lib.lib()
    s = oracle.frame_encode(_text(BLOCK, 2))
    for index in (None, [chain(s)]):
        deltas = []
        for count in (1, 65536):
            bt = Batch([s] * count, [BLOCK] * count) if count == 1 else None
            if count > 1:
                bt = Batch([s], [BLOCK])
                bt.streams, bt.lens, bt.caps = [s] * count, [len(s)] * count, [BLOCK] * count
                bt.in_ptrs, bt.out_ptrs = bt.in_ptrs * count, bt.out_ptrs * count   # every unit reads and writes the same buffers
            ix = None if index is None else index * count
            decode_ws(snap, bt, index=ix, max_chunks=count)            # warm the pools
            a0, l0 = L.sb_alloc_count(), L.sb_launch_count()
            rc, res, uc = decode_ws(snap, bt, index=ix, max_chunks=count)
            deltas.append(L.sb_launch_count() - l0)
            assert L.sb_alloc_count() == a0
            assert rc == 0 and res[0][1] == _text(BLOCK, 2) and set(uc) == {1}
            assert all(r[0] == ("Ok", 0, 0, 0) for r in res)
        assert deltas[0] == deltas[1], (index is None, deltas)


def test_python_decode_batch(snap, oracle):
    from oracle.oracle import OracleError
    rng = random.Random(9)
    units = [b"", b"x", _text(BLOCK, 1), _text(3 * BLOCK + 17, 2), bytes(200000), rng.randbytes(70000)]
    assert snap.frame.decode_batch(snap.frame.encode_batch(units)) == units
    assert snap.frame.decode_batch([]) == []
    streams = [oracle.frame_encode(u) for u in units] + [ls.gen_frame(rng, oracle.crc32c_masked, 8).stream]
    got = snap.frame.decode_batch(streams)
    assert got[:len(units)] == units and got[-1] == oracle.frame_decode(streams[-1])
    bad = bytearray(streams[3])
    bad[chain(streams[3])[1] + 5] ^= 1
    try:
        oracle.frame_decode(bytes(bad))
        raise AssertionError("the oracle accepted a corrupt stream")
    except OracleError as e:
        want = e.err
    with pytest.raises(snap.Error) as ex:
        snap.frame.decode_batch(streams[:3] + [bytes(bad)] + streams[4:] + [bytes(bad)[:-3]])
    assert ex.value.as_tuple() == tuple(want)
