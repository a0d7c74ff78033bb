"""Raw seek tables and ranges over tabled raw streams on the GPU (sb_raw_table_build_batch_device_ws,
sb_raw_table_decode_ranges_device_ws, raw.TableReader). A unit must be seekable exactly when sb_decompress_batch_device_ws
decodes it block-parallel with Ok (more than one block) or decodes it Ok (one block at most); every table must equal its
count == 1 build; every range of a seekable table must equal the oracle's slice, with guard bytes around every output
untouched; reads over other bytes, other tables or tampered tables must give the documented statuses."""
import ctypes as C
import random

import numpy as np
import pytest

import legal_streams as ls
from test_raw_batch_decode_gpu import Units, _text

pytestmark = pytest.mark.gpu

BLOCK = 65536
MIB = 1 << 20
HEAD = 64
GUARD = 256
OK = ("Ok", 0, 0, 0)
FRAME_MAGIC = 0x0001000042545342


@pytest.fixture(scope="module")
def snap():
    import torch
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)
    import gpu_helpers
    return gpu_helpers.snap()


def _dev(b):
    import torch
    return torch.from_numpy(np.frombuffer(bytes(b) + bytes(16), dtype=np.uint8).copy()).cuda()


def _i64(v):
    import torch
    return torch.from_numpy(np.array(list(v), dtype=np.uint64).view(np.int64)).cuda()


def _u32(v):
    import torch
    return torch.from_numpy(np.array(list(v), dtype=np.uint32).view(np.int32)).cuda()


def status(s):
    code = int(s[0]) & 0xFFFFFFFF
    return ({0: "Ok", 202: "Invalid"}.get(code, str(code)), int(s[1]), int(s[2]), int(s[3]))


def device_compress(snap, datas):
    """Raw streams of `datas` from one sb_compress_batch_device_ws call."""
    import torch
    L = snap._lib.lib()
    n = len(datas)
    ins = [_dev(d) for d in datas]
    caps = [L.sb_max_compress_len(len(d)) for d in datas]
    t_out = torch.empty(sum(caps) + 16, dtype=torch.uint8, device="cuda")
    at = np.concatenate([[0], np.cumsum(caps[:-1])]).astype(np.int64)
    t_ip, t_op = _i64([t.data_ptr() for t in ins] + [0]), _i64([t_out.data_ptr() + int(o) for o in at] + [0])
    t_lens, t_caps = _u32([len(d) for d in datas] + [0]), _u32(caps + [0])
    t_ol, t_st = torch.zeros(n + 1, dtype=torch.int32, device="cuda"), torch.zeros(32 * n, dtype=torch.uint8, device="cuda")
    b = snap._lib.SbBatch()
    b.in_ptrs, b.out_ptrs, b.in_lens, b.out_caps = t_ip.data_ptr(), t_op.data_ptr(), t_lens.data_ptr(), t_caps.data_ptr()
    b.out_lens, b.statuses, b.count = t_ol.data_ptr(), t_st.data_ptr(), n
    ib = sum(len(d) for d in datas)
    need = L.sb_compress_batch_scratch_bytes(n, ib)
    scr = torch.empty(need, dtype=torch.uint8, device="cuda")
    e = snap._lib.SbError()
    assert L.sb_compress_batch_device_ws(C.byref(b), ib, scr.data_ptr(), need, torch.cuda.current_stream().cuda_stream,
                                         C.byref(e)) == 0
    ol = t_ol.cpu().numpy().view(np.uint32)
    back = t_out.cpu().numpy()
    return [back[int(o):int(o) + int(k)].tobytes() for o, k in zip(at, ol[:n])]


class Tables:
    """One batch build over streams already on the device (ins: tensors with 16 bytes of slack)."""

    def __init__(self, snap, streams, in_bytes=None, stream=None, ins=None, run=True):
        import torch
        self.snap, self.L = snap, snap._lib.lib()
        self.streams = streams
        self.ins = ins if ins is not None else [_dev(s) for s in streams]
        self.n = len(streams)
        self.in_bytes = sum(len(s) for s in streams) if in_bytes is None else in_bytes
        self.t_ip = _i64([t.data_ptr() for t in self.ins] + [0])
        self.t_lens = _u32([len(s) for s in streams] + [0])
        self.tb = self.L.sb_raw_table_batch_bytes(self.n, self.in_bytes)
        self.t_tab = torch.full((self.tb + GUARD,), 0xAB, dtype=torch.uint8, device="cuda")
        self.t_offs = torch.full((self.n + 2,), -1, dtype=torch.int64, device="cuda")
        self.t_res = torch.full((48 * self.n + 48,), 0xA5, dtype=torch.uint8, device="cuda")
        self.need = self.L.sb_raw_table_build_batch_scratch_bytes(self.n, self.in_bytes)
        self.t_scr = torch.full((self.need + GUARD,), 0xCD, dtype=torch.uint8, device="cuda")
        if run:
            assert self.call(stream=stream) == 0
            torch.cuda.synchronize()
            self.check()

    def batch(self):
        b = self.snap._lib.SbBatch()
        b.in_ptrs, b.in_lens, b.count = self.t_ip.data_ptr(), self.t_lens.data_ptr(), self.n
        return b

    def call(self, b=None, tables=True, offs=True, res=True, scr=True, tb=None, sb=None, stream=None):
        import torch
        e = self.snap._lib.SbError()
        st = (stream or torch.cuda.current_stream()).cuda_stream
        return self.L.sb_raw_table_build_batch_device_ws(
            C.byref(b or self.batch()), self.in_bytes, self.t_tab.data_ptr() if tables else None,
            self.tb if tb is None else tb, self.t_offs.data_ptr() if offs else None, self.t_res.data_ptr() if res else None,
            self.t_scr.data_ptr() if scr else None, self.need if sb is None else sb, st, C.byref(e))

    def check(self):
        n = self.n
        self.offs = [int(x) for x in self.t_offs.cpu().numpy().view(np.uint64)]
        r = self.t_res.cpu().numpy()
        self.res = np.frombuffer(r[:48 * n].tobytes(), dtype=np.uint64).reshape(n, 6)
        assert (r[48 * n:] == 0xA5).all() and self.offs[n + 1] == 0xFFFFFFFFFFFFFFFF and self.offs[0] == 0
        self.buf = self.t_tab.cpu().numpy()
        assert (self.buf[self.offs[n]:] == 0xAB).all()
        assert bool((self.t_scr[self.need:] == 0xCD).all())
        for i in range(n):
            assert self.offs[i + 1] - self.offs[i] == HEAD + 8 * (int(self.res[i][5]) & 0xFFFFFFFF), i
            assert int(self.res[i][5]) >> 32 == 0 and (int(self.res[i][0]) >> 32) == 0, i

    def table(self, i):
        return self.buf[self.offs[i]:self.offs[i + 1]]

    def seekable(self, i):
        return int(np.frombuffer(self.table(i)[32:36].tobytes(), dtype=np.uint32)[0]) == 1

    def device_tables(self):
        return [self.t_tab.data_ptr() + self.offs[i] for i in range(self.n)]


def read(snap, tables, ins, lens, ranges, count=None, stream=None):
    """One sb_raw_table_decode_ranges_device_ws call: [(status, bytes)]. Every range's buffer holds
    max(0, min(n, lens[u] - lo)) bytes between guard bytes that must stay untouched."""
    import torch
    L = snap._lib.lib()
    k = len(ranges)
    count = len(tables) if count is None else count
    room = [max(0, min(n, lens[u] - lo)) if u < len(lens) else 0 for u, lo, n in ranges]
    at, pos = [], GUARD
    for r in room:
        at.append(pos)
        pos += r + GUARD
    t_out = torch.full((pos,), 0xEE, dtype=torch.uint8, device="cuda")
    t_tabs, t_ins = _i64(list(tables) + [0]), _i64([t.data_ptr() for t in ins] + [0])
    t_lens = _i64([t.numel() - 16 for t in ins] + [0])
    t_unit = _u32([u for u, _, _ in ranges] + [0])
    t_lo, t_len = _i64([lo for _, lo, _ in ranges] + [0]), _i64([n for _, _, n in ranges] + [0])
    t_op = _i64([t_out.data_ptr() + a for a in at] + [0])
    t_ol = torch.full((k + 1,), -1, dtype=torch.int64, device="cuda")
    t_st = torch.zeros(4 * k + 4, dtype=torch.int64, device="cuda")
    need = L.sb_raw_table_ranges_scratch_bytes(k)
    scr = torch.full((need + GUARD,), 0xCD, dtype=torch.uint8, device="cuda")
    e = snap._lib.SbError()
    st = (stream or torch.cuda.current_stream()).cuda_stream
    assert L.sb_raw_table_decode_ranges_device_ws(t_tabs.data_ptr(), t_ins.data_ptr(), t_lens.data_ptr(), count,
                                                  t_unit.data_ptr(), t_lo.data_ptr(), t_len.data_ptr(), t_op.data_ptr(),
                                                  t_ol.data_ptr(), t_st.data_ptr(), k, scr.data_ptr(), need, st,
                                                  C.byref(e)) == 0
    torch.cuda.synchronize()
    assert bool((scr[need:] == 0xCD).all())
    out = t_out.cpu().numpy()
    ol = t_ol.cpu().numpy().view(np.uint64)
    sts = t_st.cpu().numpy().view(np.uint64).reshape(-1, 4)
    assert ol[k] == 0xFFFFFFFFFFFFFFFF
    got = []
    for i in range(k):
        a, r, m = at[i], room[i], int(ol[i])
        assert (out[a - GUARD:a] == 0xEE).all() and (out[a + r:a + r + GUARD] == 0xEE).all(), i
        assert m <= r, i
        got.append((status(sts[i]), out[a:a + m].tobytes()))
    return got


def head(t):
    w = np.frombuffer(t[:HEAD].tobytes(), dtype=np.uint64)
    return {"n": int(w[1]), "dn": int(w[2]), "hl": int(w[3]) & 0xFFFFFFFF, "nblocks": int(w[3]) >> 32,
            "seekable": int(w[4]) & 0xFFFFFFFF, "reason": int(w[4]) >> 32}


def res_of(t, i):
    """(status, bytes, nblocks) of unit i's result."""
    w = t.res[i]
    return status(w[:4]), int(w[4]), int(w[5]) & 0xFFFFFFFF


def mixed_streams(snap, oracle):
    rng = random.Random(7)
    datas = [_text(n, n) for n in (3 * MIB + 5, MIB + 1, BLOCK, BLOCK + 1, 100, 0)]
    ss = device_compress(snap, datas)
    ss += [oracle.compress(_text(n, 3 * n)) for n in (2 * MIB, 70000, 10)]
    good = ls.gen_stream(rng, 600000, "blocked", copy_share=0.3)
    ss.append(good.stream)
    ss += [s.stream for s in (ls.gen_stream(rng, 300000, "unblocked") for _ in range(4)) if s.straddles][:2]
    ss += [ls.giant_literal(rng, 80000, "lit63")[0]]
    ss += ls.corrupt(rng, good)
    ss += [b"", b"\x00", b"\x00\x00", b"\x80", b"\xff" * 11, ls.varint(3) + b"\x08abc"]
    return ss


def verdicts(snap, oracle, t, streams):
    """Seekable ⇔ the batch decode splits the unit Ok (multi-block) or decodes it Ok (single block)."""
    dns = []
    for s in streams:
        try:
            dns.append(oracle.decompress_len(s) if s else None)
        except Exception:
            dns.append(None)
    caps = [d if d is not None and d < (1 << 32) else 0 for d in dns]
    rc, res, blocks, _ = Units(streams, caps).run()
    assert rc == 0
    for i, s in enumerate(streams):
        multi = caps[i] > BLOCK
        want = res[i][0] == OK and (blocks[i] > 0 if multi else True)
        assert t.seekable(i) == want, (i, len(s), res[i][0], blocks[i], head(t.table(i)))
    return [r[0] == OK for r in res]


def test_mixed_batch_verdicts_tables_and_single_builds(snap, oracle):
    streams = mixed_streams(snap, oracle)
    t = Tables(snap, streams)
    verdicts(snap, oracle, t, streams)
    assert all(t.seekable(i) for i in range(9))                           # the encoders' streams
    for i, s in enumerate(streams):
        h = head(t.table(i))
        st, nbytes, _ = res_of(t, i)
        if t.seekable(i):
            data = oracle.decompress(s)
            nb = (len(data) + BLOCK - 1) // BLOCK
            assert (st, nbytes, h["dn"], h["nblocks"]) == (OK, len(data), len(data), nb), i
            crcs = np.frombuffer(t.table(i)[HEAD:].tobytes(), dtype=np.uint32)[1::2]
            assert [int(c) for c in crcs] == [oracle.crc32c_masked(data[j * BLOCK:(j + 1) * BLOCK]) for j in range(nb)]
        else:
            assert st == ("Invalid", i, 0, 5) and nbytes == 0 and len(t.table(i)) == HEAD and h["reason"], i
        one = Tables(snap, [s], ins=[t.ins[i]])
        assert one.table(0).tobytes() == t.table(i).tobytes(), i


def test_ranges_equal_the_oracle(snap, oracle):
    rng = random.Random(8)
    streams = mixed_streams(snap, oracle)
    t = Tables(snap, streams)
    seek = [i for i in range(len(streams)) if t.seekable(i)]
    datas = {i: oracle.decompress(streams[i]) for i in seek}
    ranges = []
    for i in seek:
        dn = len(datas[i])
        ranges += [(i, 0, dn), (i, dn, 4), (i, dn + 9, 1), (i, 0, 0), (i, 0, 1 << 62)]
        for j in range(0, dn + 1, BLOCK)[:40]:
            ranges += [(i, max(j - 3, 0), 7), (i, j, BLOCK), (i, max(j - 1, 0), BLOCK + 2)]
        ranges += [(i, rng.randrange(dn + 1), rng.choice([1, 4096, 3 * BLOCK])) for _ in range(20)]
    ranges += ranges[:50]
    rng.shuffle(ranges)
    lens = [head(t.table(i))["dn"] for i in range(len(streams))]
    got = read(snap, t.device_tables(), t.ins, lens, ranges)
    for (i, lo, n), (st, b) in zip(ranges, got):
        assert st == OK and b == datas[i][lo:lo + n], (i, lo, n)


def test_read_statuses(snap, oracle):
    import torch
    streams = device_compress(snap, [_text(5 * BLOCK + 77, 1)]) + [ls.varint(3) + b"\x04ab"]
    t = Tables(snap, streams)
    data = oracle.decompress(streams[0])
    n = len(streams[0])
    frame = torch.zeros(HEAD, dtype=torch.uint8, device="cuda")
    frame[:16] = torch.from_numpy(np.array([FRAME_MAGIC, n], dtype=np.uint64).view(np.uint8).copy()).cuda()
    flip = bytearray(streams[0])
    flip[n - 10] ^= 0x01                                                # inside the last block's bytes
    short = _dev(streams[0][:-1])
    tabs = t.device_tables() + [frame.data_ptr(), t.device_tables()[0], t.device_tables()[0]]
    ins = t.ins + [t.ins[0], short, _dev(flip)]
    lens = [len(data), 0, 0, len(data), len(data)]
    got = read(snap, tabs, ins, lens, [(0, 3, 10), (9, 0, 1), (1, 0, 1), (2, 0, 1), (3, 0, 1), (4, 0, BLOCK),
                                       (4, 5 * BLOCK - 2, 50), (4, 4 * BLOCK, 10)])
    st = [s for s, _ in got]
    assert st[:5] == [OK, ("Invalid", 9, 5, 1), ("Invalid", 1, 0, 5), ("Invalid", n, 0, 2), ("Invalid", n - 1, n, 2)]
    assert got[0][1] == data[3:13]
    # the changed byte lies in block 5 (the last): ranges over other blocks are Ok, those covering it fail with c=4
    assert got[5] == (OK, data[:BLOCK]) and got[7] == (OK, data[4 * BLOCK:4 * BLOCK + 10])
    assert got[6] == (("Invalid", 5, 0, 4), data[5 * BLOCK - 2:5 * BLOCK])
    # a tampered record: c=3
    tab = t.t_tab[t.offs[0]:t.offs[1]].clone()
    tab[HEAD + 8 * 3:HEAD + 8 * 3 + 4] = torch.from_numpy(np.array([n + 1], dtype=np.uint32).view(np.uint8)).cuda()
    got = read(snap, [tab.data_ptr()], [t.ins[0]], [len(data)], [(0, 0, 2 * BLOCK), (0, 2 * BLOCK + 5, BLOCK)])
    assert got[0] == (OK, data[:2 * BLOCK]) and got[1] == (("Invalid", 2, 0, 3), b"")


def test_in_bytes_under_the_sum(snap, oracle):
    streams = device_compress(snap, [_text(n, n) for n in (MIB, 3000, BLOCK + 9)])
    t = Tables(snap, streams, in_bytes=sum(len(s) for s in streams) - 1)
    assert [t.seekable(i) for i in range(3)] == [False, True, False]
    assert [head(t.table(i))["reason"] for i in (0, 2)] == [2, 2]


def test_call_rules(snap, oracle):
    """Argument errors launch nothing; the same launches for 1 and 300 units; no allocation; a call on a side stream
    behind pending work."""
    import torch
    L = snap._lib.lib()
    small = device_compress(snap, [_text(200000, 5)])
    many = device_compress(snap, [_text(1000 + 300 * i, i) for i in range(300)])
    t1, t2 = Tables(snap, small, run=False), Tables(snap, many, run=False)
    for t in (t1, t2):                                                   # warm up
        assert t.call() == 0
    torch.cuda.synchronize()
    counts = []
    for t in (t1, t2):
        l0, a0 = L.sb_launch_count(), L.sb_alloc_count()
        assert t.call() == 0
        counts.append(L.sb_launch_count() - l0)
        assert L.sb_alloc_count() == a0
    assert counts[0] == counts[1] == 13
    l0 = L.sb_launch_count()
    for kw in ({"tables": False}, {"offs": False}, {"res": False}, {"scr": False}, {"tb": t1.tb - 1},
               {"sb": t1.need - 1}):
        assert t1.call(**kw) == 202, kw
    b = t1.batch()
    b.count = 1 << 31
    assert t1.call(b=b) == 202
    b.count = 0
    assert t1.call(b=b) == 0
    e = snap._lib.SbError()
    assert L.sb_raw_table_decode_ranges_device_ws(None, None, None, 1, None, None, None, None, None, None, 1, None, 0, None,
                                                  C.byref(e)) == 202
    assert L.sb_launch_count() == l0
    # behind pending work: the input is written on the side stream just before the build there
    side = torch.cuda.Stream()
    data = _text(4 * MIB, 9)
    s = device_compress(snap, [data])[0]
    src = _dev(s)
    dst = torch.zeros_like(src)
    torch.cuda.synchronize()
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)
        dst.copy_(src)
        t = Tables(snap, [s], ins=[dst], stream=side, run=False)
        assert t.call(stream=side) == 0
        got = read(snap, [t.t_tab.data_ptr()], [dst], [len(data)], [(0, MIB - 5, 2 * MIB)], stream=side)
    t.check()
    assert t.seekable(0) and got == [(OK, data[MIB - 5:3 * MIB - 5])]


def test_pyarrow_pages(snap, oracle):
    pa = pytest.importorskip("pyarrow")
    pages = [_text(MIB, 500 + i) for i in range(24)]
    streams = [pa.compress(d, codec="snappy", asbytes=True) for d in pages]
    t = Tables(snap, streams)
    assert all(t.seekable(i) for i in range(len(streams)))
    rng = random.Random(3)
    ranges = [(rng.randrange(24), rng.randrange(MIB), 4096) for _ in range(500)]
    got = read(snap, t.device_tables(), t.ins, [MIB] * 24, ranges)
    for (i, lo, n), (st, b) in zip(ranges, got):
        assert st == OK and b == pages[i][lo:lo + n]


def test_table_reader(snap, oracle):
    import torch
    rng = random.Random(4)
    streams = mixed_streams(snap, oracle)
    streams[1] = _dev(streams[1])[:-16]                                  # a tensor stream
    r = snap.raw.TableReader(streams)
    dec = snap.raw.Decoder()
    host = [bytes(s.cpu().numpy().tobytes()) if isinstance(s, torch.Tensor) else s for s in streams]
    assert len(r) == len(streams)
    ranges = []
    for i, s in enumerate(host):
        try:
            want = dec.decompress_vec(s)
        except Exception as x:
            with pytest.raises(type(x)) as got:
                r.read(i, 0, 10)
            assert str(got.value) == str(x) and repr(got.value) == repr(x), i
            assert not r.seekable[i] and r.lengths[i] is None
            continue
        assert r.seekable[i] == (r.lengths[i] is not None)
        if r.seekable[i]:
            assert r.lengths[i] == len(want)
        for lo, n in ((0, len(want)), (max(len(want) - 5, 0), 100), (rng.randrange(len(want) + 1), 5000)):
            ranges.append((i, lo, n, want[lo:lo + n]))
    rng.shuffle(ranges)
    got = r.read_ranges([(i, lo, n) for i, lo, n, _ in ranges])
    assert got == [w for *_, w in ranges]
    with pytest.raises(IndexError):
        r.read(len(streams), 0, 1)
    big = torch.empty(1 << 32, dtype=torch.uint8, device="cuda")
    with pytest.raises(ValueError):
        snap.raw.TableReader([big])
    del big
