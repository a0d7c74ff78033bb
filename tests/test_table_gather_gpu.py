"""Gathers over tabled frame and raw streams on the GPU (sb_frame_table_gather_device_ws, sb_raw_table_gather_device_ws,
TableReader.gather). Every range must get exactly the status, out_len and bytes of the range calls
(sb_*_table_decode_ranges_device_ws, run in groups of 4,096) and, where Ok, the batch decode's slice, with the bytes
between the ranges' buffers untouched; a call of 2^20 ranges must fit the documented scratch bound; the launches must
not depend on nranges or the sharing pattern, nothing may be allocated, and argument errors must launch nothing."""
import ctypes as C
import random

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

BLOCK = 65536
GAP = 16
GROUP = 4096


@pytest.fixture(scope="module")
def snap():
    import torch
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)
    import gpu_helpers
    return gpu_helpers.snap()


def _text(n, seed):
    from conftest import corpus
    base = corpus("alice29.txt") + corpus("lcet10.txt") + corpus("html_x_4") + corpus("urls.10K")
    k = seed * 7919 % len(base)
    return ((base[k:] + base) * (n // len(base) + 2))[:n]


@pytest.fixture(scope="module")
def datas():
    rng = random.Random(1)
    return [_text(rng.randrange(40000, 400000), s) for s in range(1024)]


@pytest.fixture(scope="module")
def readers(snap, datas):
    """A frame and a raw TableReader over 1,024 streams each, tabled by the batch encoders."""
    frames, ftabs = snap.frame.encode_batch(datas, tables=True)
    raws, rtabs = snap.raw.compress_batch(datas, tables=True)
    return snap.frame.TableReader(frames, tables=ftabs), snap.raw.TableReader(raws, tables=rtabs), frames, raws


def random_ranges(lengths, n, rng, zipf=False, size=256):
    """n small ranges: uniform over all streams, or Zipf-skewed over streams with a hot chunk shared by >256 ranges."""
    out = []
    if zipf:
        w = 1.0 / np.arange(1, len(lengths) + 1) ** 1.1
        units = np.random.default_rng(rng.randrange(1 << 30)).choice(len(lengths), n, p=w / w.sum())
    else:
        units = [rng.randrange(len(lengths)) for _ in range(n)]
    for u in units:
        u = int(u)
        out.append((u, rng.randrange(lengths[u] + 10), rng.randrange(0, 2 * size)))
    if zipf:
        out += [(0, BLOCK + rng.randrange(BLOCK - 600), rng.randrange(1, 512)) for _ in range(700)]   # one hot chunk
        out += [(1, 0, 0), (1, lengths[1], 5), (2, BLOCK - 100, 2 * BLOCK + 200)] * 3
    rng.shuffle(out)
    return out


def run(snap, reader, fmt, ranges, gather, ins=None, stream=None, scratch_bytes=None):
    """One gather call (or range calls in groups of 4,096) over a reader's tables: (statuses, out_lens, bytes)."""
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
    st = (stream or torch.cuda.current_stream()).cuda_stream
    e = snap._lib.SbError()
    parts = [(0, k)] if gather else [(a, min(a + GROUP, k)) for a in range(0, k, GROUP)]
    nb = getattr(L, "sb_%s_table_%s_scratch_bytes" % (fmt, "gather" if gather else "ranges"))
    fn = getattr(L, "sb_%s_table_%s_device_ws" % (fmt, "gather" if gather else "decode_ranges"))
    scr = torch.empty(max(nb(b - a) for a, b in parts), dtype=torch.uint8, device="cuda")
    for a, b in parts:
        need = nb(b - a) if scratch_bytes is None else scratch_bytes
        assert fn(reader._t_tables.data_ptr(), t_ins.data_ptr(), reader._t_lens.data_ptr(), len(reader._ins),
                  t_unit.data_ptr() + 4 * a, t_lo.data_ptr() + 8 * a, t_ln.data_ptr() + 8 * a, t_ptr.data_ptr() + 8 * a,
                  t_ol.data_ptr() + 8 * a, t_st.data_ptr() + 32 * a, b - a, scr.data_ptr(), need, st, C.byref(e)) == 0
    (stream or torch.cuda.current_stream()).synchronize()
    ol = t_ol.cpu().numpy().view(np.uint64)
    sts = t_st.cpu().numpy().view(np.uint64).reshape(-1, 4)
    back = out.cpu().numpy()
    assert int(ol[k]) == 0xFFFFFFFFFFFFFFFF and (sts[k] == 0xFFFFFFFFFFFFFFFF).all()
    got = []
    for j in range(k):
        m = int(ol[j])
        assert m <= rooms[j]
        assert (back[int(at[j]) + rooms[j]:int(at[j + 1])] == 0xEE).all(), j     # the gap behind the buffer
        got.append((tuple(int(x) for x in sts[j]), m, back[int(at[j]):int(at[j]) + m].tobytes()))
    assert (back[int(at[k]):] == 0xEE).all()
    return got


@pytest.mark.parametrize("fmt", ["frame", "raw"])
@pytest.mark.parametrize("zipf", [False, True])
def test_gather_equals_range_calls_and_batch_decode(snap, readers, datas, fmt, zipf):
    fr, rr, _, _ = readers
    reader = fr if fmt == "frame" else rr
    rng = random.Random(2 + zipf)
    ranges = random_ranges([len(d) for d in datas], 100000, rng, zipf)
    got = run(snap, reader, fmt, ranges, True)
    want = run(snap, reader, fmt, ranges, False)
    assert got == want
    for (u, lo, n), (st, m, b) in zip(ranges, got):
        assert st[0] & 0xFFFFFFFF == 0 and b == datas[u][lo:lo + n], (u, lo, n)


@pytest.mark.parametrize("fmt", ["frame", "raw"])
def test_other_bytes_of_the_same_length(snap, readers, datas, fmt):
    """Streams 0 and 1 read over copies with one byte changed: the gather's statuses equal the range calls'."""
    import torch
    fr, rr, frames, raws = readers
    reader = fr if fmt == "frame" else rr
    streams = frames if fmt == "frame" else raws
    bad = []
    for u in (0, 1):
        b = bytearray(streams[u])
        b[len(b) // 3] ^= 0x21
        bad.append(torch.from_numpy(np.frombuffer(bytes(b) + bytes(16), dtype=np.uint8).copy()).cuda())
    ptrs = reader._t_ins.cpu().numpy().copy()
    ptrs[0], ptrs[1] = bad[0].data_ptr(), bad[1].data_ptr()
    ins = torch.from_numpy(ptrs).cuda()
    rng = random.Random(5)
    ranges = [(u, rng.randrange(len(datas[u])), rng.randrange(1, 3000)) for u in (0, 1, 2) for _ in range(600)]
    ranges += [(u, 0, len(datas[u])) for u in (0, 1)] + [(5000, 0, 3)]
    got = run(snap, reader, fmt, ranges, True, ins=ins)
    assert got == run(snap, reader, fmt, ranges, False, ins=ins)
    assert any(st[0] & 0xFFFFFFFF for st, _, _ in got[:-1])


@pytest.mark.parametrize("fmt", ["frame", "raw"])
def test_large_ranges(snap, readers, datas, fmt):
    """Few ranges of many chunks each, most of them interior: one range per call, three in a call, and through the
    reader one range per gather call."""
    fr, rr, _, _ = readers
    reader = fr if fmt == "frame" else rr
    for ranges in ([(7, 0, len(datas[7]))], [(8, 5, len(datas[8])), (9, BLOCK - 1, 3 * BLOCK + 2), (7, 0, len(datas[7]) + 100)]):
        got = run(snap, reader, fmt, ranges, True)
        assert got == run(snap, reader, fmt, ranges, False)
        for (u, lo, n), (st, m, b) in zip(ranges, got):
            assert st[0] & 0xFFFFFFFF == 0 and b == datas[u][lo:lo + n]
    data, offs = reader.gather([(11, 0, len(datas[11]))])
    assert data.cpu().numpy().tobytes() == datas[11] and list(offs) == [0, len(datas[11])]


@pytest.mark.parametrize("fmt", ["frame", "raw"])
def test_one_call_of_2_20_ranges(snap, readers, datas, fmt):
    fr, rr, _, _ = readers
    reader = fr if fmt == "frame" else rr
    L = snap._lib.lib()
    n = 1 << 20
    need = getattr(L, "sb_%s_table_gather_scratch_bytes" % fmt)(n)
    assert need <= 128 * n + (256 << 20) + (64 << 10)
    ranges = random_ranges([len(d) for d in datas], n, random.Random(9), size=128)[:n]
    got = run(snap, reader, fmt, ranges, True)
    for (u, lo, k), (st, m, b) in zip(ranges, got):
        assert st[0] & 0xFFFFFFFF == 0 and b == datas[u][lo:lo + k]


@pytest.mark.parametrize("fmt", ["frame", "raw"])
def test_call_rules(snap, readers, datas, fmt):
    """The same launches for 1, 5,000 and 200,000 ranges, spread or all on one chunk; no allocation once warm; a call on
    a side stream behind pending work; argument errors launch nothing."""
    import torch
    fr, rr, _, _ = readers
    reader = fr if fmt == "frame" else rr
    L = snap._lib.lib()
    lens = [len(d) for d in datas]
    sets = [[(3, 10, 20)], random_ranges(lens, 5000, random.Random(1)), [(0, 100 + i % 900, 50) for i in range(200000)]]
    big = max(getattr(L, "sb_%s_table_gather_scratch_bytes" % fmt)(len(s)) for s in sets)
    run(snap, reader, fmt, sets[2], True, scratch_bytes=big)                 # warm: every pool sized
    deltas, a0 = set(), L.sb_alloc_count()
    for s in sets:
        l0 = L.sb_launch_count()
        run(snap, reader, fmt, s, True)
        deltas.add(L.sb_launch_count() - l0)
    assert deltas == {10} and L.sb_alloc_count() == a0
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        torch.cuda._sleep(20000000)                                          # pending work ahead of the call
        got = run(snap, reader, fmt, sets[1], True, stream=side)
    assert got == run(snap, reader, fmt, sets[1], False)
    fn = getattr(L, "sb_%s_table_gather_device_ws" % fmt)
    nb = getattr(L, "sb_%s_table_gather_scratch_bytes" % fmt)
    scr = torch.empty(nb(4), dtype=torch.uint8, device="cuda")
    p = reader._t_tables.data_ptr()
    e = snap._lib.SbError()
    st = torch.cuda.current_stream().cuda_stream
    l0 = L.sb_launch_count()
    assert fn(p, p, p, 3, p, p, p, p, p, p, 4, scr.data_ptr(), nb(4) - 1, st, C.byref(e)) == 202
    assert fn(p, p, p, 3, p, p, p, p, p, p, (1 << 28) + 1, scr.data_ptr(), 1 << 62, st, C.byref(e)) == 202
    assert fn(p, p, p, 1 << 31, p, p, p, p, p, p, 4, scr.data_ptr(), nb(4), st, C.byref(e)) == 202
    assert fn(p, p, p, 3, None, p, p, p, p, p, 4, scr.data_ptr(), nb(4), st, C.byref(e)) == 202
    assert fn(p, p, p, 3, p, p, p, p, p, p, 4, None, nb(4), st, C.byref(e)) == 202
    assert fn(p, p, p, 3, p, p, p, p, p, p, 0, None, 0, st, C.byref(e)) == 0
    assert L.sb_launch_count() == l0


def test_table_reader_gather(snap, oracle, readers, datas):
    """gather equals read_ranges: both readers over stored tables, fresh builds with a raw stream that is not
    seekable, and the first failing range's error."""
    import torch
    fr, rr, frames, raws = readers
    rng = random.Random(11)
    ranges = random_ranges([len(d) for d in datas], 20000, rng, True)
    for reader in (fr, rr):
        data, offs = reader.gather(ranges)
        assert isinstance(data, torch.Tensor) and data.is_cuda and len(offs) == len(ranges) + 1
        back = data.cpu().numpy().tobytes()
        want = reader.read_ranges(ranges)
        assert [back[int(offs[j]):int(offs[j + 1])] for j in range(len(ranges))] == want
    # a fresh raw reader: a stream that is not seekable (an unblocked encoder's copies reach across blocks) beside
    # tabled ones, and a stream that does not decode
    import legal_streams as ls
    g = random.Random(3)
    unblocked = next(s for s in (ls.gen_stream(g, 200000, "unblocked") for _ in range(50)) if s.straddles)
    r2 = snap.raw.TableReader([raws[0], unblocked.stream, raws[1]])
    assert r2.seekable == [True, False, True]
    rs = [(1, 5, 100), (0, 7, 300), (1, 150000, 70000), (2, 0, 10), (1, 0, 0), (1, 10 ** 6, 4)] * 3
    data, offs = r2.gather(rs)
    back = data.cpu().numpy().tobytes()
    assert [back[int(offs[j]):int(offs[j + 1])] for j in range(len(rs))] == r2.read_ranges(rs)
    r3 = snap.raw.TableReader([raws[0], b"\x05\x00", raws[1]])
    for rs in ([(0, 5, 10), (1, 0, 1)], [(1, 0, 1), (0, 5, 10)]):
        with pytest.raises(Exception) as want:
            r3.read_ranges(rs)
        with pytest.raises(type(want.value)) as got:
            r3.gather(rs)
        assert str(got.value) == str(want.value)
    f2 = snap.frame.TableReader(frames[:3])
    rs = [(0, 0, 100), (2, BLOCK - 5, 10), (1, 7, 0), (2, len(datas[2]) + 3, 5)]
    data, offs = f2.gather(rs)
    back = data.cpu().numpy().tobytes()
    assert [back[int(offs[j]):int(offs[j + 1])] for j in range(len(rs))] == f2.read_ranges(rs)
    with pytest.raises(IndexError):
        f2.gather([(3, 0, 1)])
