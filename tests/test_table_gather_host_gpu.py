"""Gathers over streams in pinned host memory on the GPU (sb_frame_table_gather_host_streams_ws,
sb_raw_table_gather_host_streams_ws, TableReader(..., host=True)). Every range must get exactly the status, out_len and
bytes of the device gather over device copies of the same streams, with the bytes between the ranges' buffers
untouched: streams in a torch pinned buffer, in numpy memory registered with cudaHostRegister, and in device memory.
The scratch must follow its documented formula, the launches must not depend on nranges, nothing may be allocated, and
argument errors must launch nothing. Only page-locked or device memory is ever handed to the library."""
import ctypes as C
import random

import numpy as np
import pytest

from test_table_gather_gpu import BLOCK, GAP, _text, random_ranges

pytestmark = pytest.mark.gpu

CSLOT = 76544


@pytest.fixture(scope="module")
def snap():
    import torch
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)
    import gpu_helpers
    return gpu_helpers.snap()


@pytest.fixture(scope="module")
def corpus(snap):
    """1,024 text streams tabled by the batch encoders, frame and raw: (datas, frames, ftabs, raws, rtabs)."""
    rng = random.Random(1)
    datas = [_text(rng.randrange(40000, 400000), s) for s in range(1024)]
    frames, ftabs = snap.frame.encode_batch(datas, tables=True)
    raws, rtabs = snap.raw.compress_batch(datas, tables=True)
    return datas, frames, ftabs, raws, rtabs


@pytest.fixture(scope="module")
def readers(snap, corpus):
    """{fmt: (device-resident reader, host reader)} over the stored tables."""
    datas, frames, ftabs, raws, rtabs = corpus
    return {"frame": (snap.frame.TableReader(frames, tables=ftabs), snap.frame.TableReader(frames, tables=ftabs, host=True)),
            "raw": (snap.raw.TableReader(raws, tables=rtabs), snap.raw.TableReader(raws, tables=rtabs, host=True))}


def run(snap, reader, fmt, ranges, host, ins=None, scratch_bytes=None):
    """One gather call over a reader's tables, the host-stream or the device one: (statuses, out_lens, bytes)."""
    import torch
    L = snap._lib.lib()
    k = len(ranges)
    rooms = [max(0, n) if n < (1 << 40) else 0 for _, _, n in ranges]
    at = np.zeros(k + 1, dtype=np.int64)
    at[1:] = np.cumsum(np.array(rooms, dtype=np.int64) + GAP)
    out = torch.full((int(at[-1]) + GAP,), 0xEE, dtype=torch.uint8, device="cuda")
    lo = np.array([r[1] for r in ranges], dtype=np.uint64)
    ln = np.array([r[2] for r in ranges], dtype=np.uint64)
    unit = np.array([r[0] for r in ranges], dtype=np.uint32)
    ptr = (at[:k] + out.data_ptr()).astype(np.uint64)
    t_lo, t_ln, t_ptr = (torch.from_numpy(x.view(np.int64)).cuda() for x in (lo, ln, ptr))
    t_unit = torch.from_numpy(unit.view(np.int32)).cuda()
    t_ol = torch.full((k + 1,), -1, dtype=torch.int64, device="cuda")
    t_st = torch.full((4 * k + 4,), -1, dtype=torch.int64, device="cuda")
    t_ins = reader._t_ins if ins is None else ins
    kind = "gather_host_streams" if host else "gather"
    nb = getattr(L, "sb_%s_table_%s_scratch_bytes" % (fmt, kind))
    fn = getattr(L, "sb_%s_table_%s" % (fmt, kind + ("_ws" if host else "_device_ws")))
    need = nb(k) if scratch_bytes is None else scratch_bytes
    scr = torch.empty(need, dtype=torch.uint8, device="cuda")
    e = snap._lib.SbError()
    assert fn(reader._t_tables.data_ptr(), t_ins.data_ptr(), reader._t_lens.data_ptr(), len(reader._ins),
              t_unit.data_ptr(), t_lo.data_ptr(), t_ln.data_ptr(), t_ptr.data_ptr(), t_ol.data_ptr(), t_st.data_ptr(), k,
              scr.data_ptr(), need, torch.cuda.current_stream().cuda_stream, C.byref(e)) == 0
    torch.cuda.synchronize()
    ol = t_ol.cpu().numpy().view(np.uint64)
    sts = t_st.cpu().numpy().view(np.uint64).reshape(-1, 4)
    back = out.cpu().numpy()
    assert int(ol[k]) == 0xFFFFFFFFFFFFFFFF and (sts[k] == 0xFFFFFFFFFFFFFFFF).all()
    got = []
    for j in range(k):
        m = int(ol[j])
        assert m <= rooms[j]
        assert (back[int(at[j]) + rooms[j]:int(at[j + 1])] == 0xEE).all(), j
        got.append((tuple(int(x) for x in sts[j]), m, back[int(at[j]):int(at[j]) + m].tobytes()))
    assert (back[int(at[k]):] == 0xEE).all()
    return got


@pytest.mark.parametrize("fmt", ["frame", "raw"])
@pytest.mark.parametrize("zipf", [False, True])
def test_host_gather_equals_device_gather(snap, corpus, readers, fmt, zipf):
    datas = corpus[0]
    dev, host = readers[fmt]
    ranges = random_ranges([len(d) for d in datas], 100000, random.Random(2 + zipf), zipf)
    got = run(snap, host, fmt, ranges, True)
    assert got == run(snap, dev, fmt, ranges, False)
    for (u, lo, n), (st, m, b) in zip(ranges, got):
        assert st[0] & 0xFFFFFFFF == 0 and b == datas[u][lo:lo + n], (u, lo, n)


@pytest.mark.parametrize("fmt", ["frame", "raw"])
def test_one_call_of_2_20_ranges(snap, corpus, readers, fmt):
    datas = corpus[0]
    dev, host = readers[fmt]
    ranges = random_ranges([len(d) for d in datas], 1 << 20, random.Random(9), size=128)[:1 << 20]
    assert run(snap, host, fmt, ranges, True) == run(snap, dev, fmt, ranges, False)


@pytest.mark.parametrize("fmt", ["frame", "raw"])
def test_registered_numpy_and_device_streams(snap, corpus, readers, fmt):
    """The same streams in numpy memory registered with cudaHostRegister, and the device reader's own device copies,
    handed to the host-stream call: the device gather's results."""
    import torch
    datas, frames, _, raws, _ = corpus
    streams = frames if fmt == "frame" else raws
    dev, _ = readers[fmt]
    L = snap._lib.lib()
    at = np.cumsum([0] + [len(s) for s in streams])
    buf = np.empty(int(at[-1]) + 4096, dtype=np.uint8)
    base = (-buf.ctypes.data) % 4096                                   # page-aligned registration
    cat = buf[base:base + int(at[-1])]
    for s, o in zip(streams, at):
        cat[o:o + len(s)] = np.frombuffer(s, dtype=np.uint8)
    rt = torch.cuda.cudart()
    assert int(rt.cudaHostRegister(cat.ctypes.data, cat.nbytes, 3)) == 0   # portable | mapped
    try:
        e = snap._lib.SbError()
        for s, o in zip(streams, at):
            assert L.sb_host_stream_check(cat.ctypes.data + int(o), len(s), C.byref(e)) == 0
        ptrs = np.append((at[:-1] + cat.ctypes.data).astype(np.uint64), np.uint64(0))
        ins = torch.from_numpy(ptrs.view(np.int64)).cuda()
        ranges = random_ranges([len(d) for d in datas], 30000, random.Random(4), True)
        want = run(snap, dev, fmt, ranges, False)
        assert run(snap, dev, fmt, ranges, True, ins=ins) == want
        assert run(snap, dev, fmt, ranges, True) == want                   # device-memory streams
    finally:
        torch.cuda.synchronize()
        assert int(rt.cudaHostUnregister(cat.ctypes.data)) == 0


@pytest.mark.parametrize("fmt", ["frame", "raw"])
def test_other_bytes_and_a_whole_16_mib_stream(snap, fmt):
    """A 16 MiB stream read whole and in pieces, and a copy with one byte changed: the device gather's results."""
    data = _text(16 << 20, 77)
    enc = snap.frame.encode_batch if fmt == "frame" else snap.raw.compress_batch
    (s,), (t,) = enc([data], tables=True)
    b = bytearray(s)
    b[len(b) // 3] ^= 0x21
    Reader = snap.frame.TableReader if fmt == "frame" else snap.raw.TableReader
    dev = Reader([s, bytes(b)], tables=[t, t])
    host = Reader([s, bytes(b)], tables=[t, t], host=True)
    rng = random.Random(6)
    ranges = [(0, 0, len(data)), (1, 0, len(data)), (0, 5, 3 * BLOCK)] + \
        [(u, rng.randrange(len(data)), rng.randrange(1, 5000)) for u in (0, 1) for _ in range(500)]
    got = run(snap, host, fmt, ranges, True)
    assert got == run(snap, dev, fmt, ranges, False)
    assert got[0][2] == data and got[1][0][0] & 0xFFFFFFFF


def test_oversized_raw_block(snap, oracle):
    """A raw block of 327,677 compressed bytes (one-byte copy-4 elements), larger than a compressed slot, decodes in
    place and gives the device gather's bytes."""
    from test_table_gather_host_emu import oversized_raw
    stream, table, data = oversized_raw(oracle)
    dev = snap.raw.TableReader([stream], tables=[table.tobytes()])
    host = snap.raw.TableReader([stream], tables=[table.tobytes()], host=True)
    assert host.seekable == [True]
    ranges = [(0, 5, 10), (0, BLOCK - 7, 20), (0, 0, len(data)), (0, BLOCK + 3, 100), (0, 0, BLOCK)]
    got = run(snap, host, "raw", ranges, True)
    assert got == run(snap, dev, "raw", ranges, False)
    assert [g[2] for g in got] == [data[lo:lo + n] for _, lo, n in ranges]
    assert host.read_ranges(ranges) == dev.read_ranges(ranges)


@pytest.mark.parametrize("fmt", ["frame", "raw"])
def test_call_rules_and_scratch(snap, corpus, readers, fmt):
    """The same launches for 1, 5,000 and 200,000 ranges; no allocation once warm; the documented scratch; argument
    errors launch nothing."""
    import torch
    datas = corpus[0]
    _, host = readers[fmt]
    L = snap._lib.lib()
    nb = getattr(L, "sb_%s_table_gather_host_streams_scratch_bytes" % fmt)
    dnb = getattr(L, "sb_%s_table_gather_scratch_bytes" % fmt)
    for n in (1, 7, 2048, 4096, 1 << 20):
        assert nb(n) == dnb(n) + min(2 * n, 4096) * CSLOT
        assert nb(n) <= 128 * n + 4096 * (65536 + CSLOT) + (64 << 10)
    lens = [len(d) for d in datas]
    sets = [[(3, 10, 20)], random_ranges(lens, 5000, random.Random(1)), [(0, 100 + i % 900, 50) for i in range(200000)]]
    big = max(nb(len(s)) for s in sets)
    run(snap, host, fmt, sets[2], True, scratch_bytes=big)
    deltas, a0 = set(), L.sb_alloc_count()
    for s in sets:
        l0 = L.sb_launch_count()
        run(snap, host, fmt, s, True)
        deltas.add(L.sb_launch_count() - l0)
    assert deltas == {10} and L.sb_alloc_count() == a0
    fn = getattr(L, "sb_%s_table_gather_host_streams_ws" % fmt)
    scr = torch.empty(nb(4), dtype=torch.uint8, device="cuda")
    p = host._t_tables.data_ptr()
    e = snap._lib.SbError()
    st = torch.cuda.current_stream().cuda_stream
    l0 = L.sb_launch_count()
    assert fn(p, p, p, 3, p, p, p, p, p, p, 4, scr.data_ptr(), nb(4) - 1, st, C.byref(e)) == 202
    assert fn(p, p, p, 3, p, p, p, p, p, p, (1 << 28) + 1, scr.data_ptr(), 1 << 62, st, C.byref(e)) == 202
    assert fn(p, p, p, 1 << 31, p, p, p, p, p, p, 4, scr.data_ptr(), nb(4), st, C.byref(e)) == 202
    assert fn(p, p, p, 3, None, p, p, p, p, p, 4, scr.data_ptr(), nb(4), st, C.byref(e)) == 202
    assert fn(p, p, p, 3, p, p, p, p, p, p, 0, None, 0, st, C.byref(e)) == 0
    assert L.sb_launch_count() == l0
    assert L.sb_host_stream_check(None, 0, C.byref(e)) == 0
    assert L.sb_host_stream_check(None, 5, C.byref(e)) == 202 and (e.a, e.b, e.c) == (0, 5, 6)


def test_table_reader_host(snap, corpus, readers):
    """read, read_ranges and gather of host readers equal the device-resident readers': stored and built tables, a raw
    stream that is not seekable, the first failing range's error; unpinned CPU and CUDA tensors are refused before
    the library sees them."""
    import torch
    import legal_streams as ls
    datas, frames, _, raws, _ = corpus
    rng = random.Random(11)
    ranges = random_ranges([len(d) for d in datas], 20000, rng, True)
    for fmt in ("frame", "raw"):
        dev, host = readers[fmt]
        assert host.read_ranges(ranges[:3000]) == dev.read_ranges(ranges[:3000])
        assert host.read(5, 100, 1000) == dev.read(5, 100, 1000)
        hd, ho = host.gather(ranges)
        dd, do = dev.gather(ranges)
        assert list(ho) == list(do) and torch.equal(hd, dd)
    g = random.Random(3)
    unblocked = next(s for s in (ls.gen_stream(g, 200000, "unblocked") for _ in range(50)) if s.straddles)
    pinned = torch.from_numpy(np.frombuffer(raws[1], dtype=np.uint8).copy()).pin_memory()
    built = [raws[0], unblocked.stream, pinned, b"\x05\x00"]
    r_dev = snap.raw.TableReader([raws[0], unblocked.stream, raws[1], b"\x05\x00"])
    r_host = snap.raw.TableReader(built, host=True)
    assert r_host.seekable == r_dev.seekable == [True, False, True, False]
    rs = [(1, 5, 100), (0, 7, 300), (1, 150000, 70000), (2, 0, 10), (1, 0, 0), (1, 10 ** 6, 4)] * 3
    assert r_host.read_ranges(rs) == r_dev.read_ranges(rs)
    hd, ho = r_host.gather(rs)
    dd, do = r_dev.gather(rs)
    assert list(ho) == list(do) and torch.equal(hd, dd)
    for rs in ([(0, 5, 10), (3, 0, 1)], [(3, 0, 1), (0, 5, 10)]):
        with pytest.raises(Exception) as want:
            r_dev.read_ranges(rs)
        for call in (r_host.read_ranges, r_host.gather):
            with pytest.raises(type(want.value)) as got:
                call(rs)
            assert str(got.value) == str(want.value)
    f_dev = snap.frame.TableReader(frames[:3])
    f_host = snap.frame.TableReader(frames[:3], host=True)
    rs = [(0, 0, 100), (2, BLOCK - 5, 10), (1, 7, 0), (2, len(datas[2]) + 3, 5)]
    assert f_host.read_ranges(rs) == f_dev.read_ranges(rs)
    with pytest.raises(IndexError):
        f_host.gather([(3, 0, 1)])
    L = snap._lib.lib()
    l0 = L.sb_launch_count()
    for Reader in (snap.frame.TableReader, snap.raw.TableReader):
        for bad in (torch.frombuffer(bytearray(frames[0]), dtype=torch.uint8), torch.tensor([1, 2], dtype=torch.uint8,
                                                                                            device="cuda")):
            with pytest.raises(ValueError):
                Reader([bad], host=True)
    assert L.sb_launch_count() == l0
