"""Seek tables and ranges over many tabled streams on the GPU (sb_frame_table_build_device_ws,
sb_frame_table_decode_ranges_device_ws and frame.TableReader). Every range must give exactly the status, out_len and
bytes that sb_frame_decode_ranges_device_ws gives it on the same stream with the same index, flags and max_chunks."""
import ctypes as C
import random

import numpy as np
import pytest

import legal_streams as ls
from conftest import CORPUS, corpus
from test_frame_batch_decode_emu import IDENT, _flip, _text, chain
from test_frame_range_decode_emu import OK, boundary_ranges, spans
from test_frame_range_decode_gpu import _status, call, full_decode, upload

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


def build(snap, t_in, n, index=None, fragment=False, max_chunks=None, table_bytes=None, scratch_bytes=None):
    """One sb_frame_table_build_device_ws call; the table and the scratch have 4 KiB of guard bytes behind them.
    Returns rc, the table (table_bytes(max_chunks) bytes) and (status, bytes, nchunks)."""
    import torch
    L = snap._lib.lib()
    if max_chunks is None:
        max_chunks = min(n // 8 + 16, (1 << 22) - 2)
    tb = L.sb_frame_table_bytes(max_chunks) if table_bytes is None else table_bytes
    need = L.sb_frame_table_build_scratch_bytes(max_chunks)
    sb = need if scratch_bytes is None else scratch_bytes
    t_tab = torch.full((tb + 4096,), 0x3C, dtype=torch.uint8, device="cuda")
    t_scr = torch.full((sb + 4096,), 0x5A, dtype=torch.uint8, device="cuda")
    t_res = torch.full((64,), 0x77, dtype=torch.uint8, device="cuda")
    t_ix = torch.from_numpy(np.array(list(index) + [7], dtype=np.uint64).view(np.int64)).cuda() if index is not None else None
    e = snap._lib.SbError()
    rc = L.sb_frame_table_build_device_ws(t_in.data_ptr(), n, t_ix.data_ptr() if t_ix is not None else None,
                                          len(index) - 1 if index is not None else 0, 1 if fragment else 0,
                                          t_tab.data_ptr(), tb, max_chunks, t_res.data_ptr(), t_scr.data_ptr(), sb,
                                          torch.cuda.current_stream().cuda_stream, C.byref(e))
    torch.cuda.synchronize()
    assert bool((t_tab[tb:] == 0x3C).all()) and bool((t_scr[sb:] == 0x5A).all()), "table or scratch overrun"
    if rc:
        assert bool((t_tab == 0x3C).all()) and bool((t_res == 0x77).all())
        return rc, None, None
    r = snap._lib.SbFrameResult.from_buffer_copy(t_res.cpu().numpy().tobytes()[:C.sizeof(snap._lib.SbFrameResult)])
    return 0, t_tab[:tb], (_status([r.status.code, r.status.a, r.status.b, r.status.c]), r.bytes, r.nchunks)


def read(snap, units, ranges, in_lens=None, scratch_bytes=None, stream=None, sync=True):
    """One sb_frame_table_decode_ranges_device_ws call over units [(input tensor, n, table tensor)] and ranges
    [(unit, lo, len)]; every output has 16 guard bytes behind it and the scratch 4 KiB. Returns rc, [(status, bytes)]."""
    import torch
    L = snap._lib.lib()
    k = len(ranges)
    lens = [ln for _, _, ln in ranges]
    offs, at = [], 3
    for ln in lens:
        offs.append(at)
        at += ln + 16 + 1 - ln % 2
    t_out = torch.full((at + 16,), 0xEE, dtype=torch.uint8, device="cuda")
    to64 = lambda v: torch.from_numpy(np.array(v, dtype=np.uint64).view(np.int64)).cuda()
    t_tabs = to64([t.data_ptr() for _, _, t in units] + [0])
    t_ins = to64([i.data_ptr() for i, _, _ in units] + [0])
    t_ns = to64((in_lens if in_lens is not None else [n for _, n, _ in units]) + [0])
    t_unit = torch.from_numpy(np.array([u for u, _, _ in ranges] + [0], dtype=np.uint32).view(np.int32)).cuda()
    t_lo, t_len = to64([lo for _, lo, _ in ranges] + [0]), to64(lens + [0])
    t_ptr = to64([t_out.data_ptr() + o for o in offs] + [0])
    t_ol = torch.full((k + 1,), -1, dtype=torch.int64, device="cuda")
    t_st = torch.full((max(k, 1) * 32,), 0x77, dtype=torch.uint8, device="cuda")
    need = L.sb_frame_table_ranges_scratch_bytes(k)
    sb = need if scratch_bytes is None else scratch_bytes
    t_scr = torch.full((sb + 4096,), 0x5A, dtype=torch.uint8, device="cuda")
    e = snap._lib.SbError()
    st = (stream or torch.cuda.current_stream()).cuda_stream
    rc = L.sb_frame_table_decode_ranges_device_ws(t_tabs.data_ptr(), t_ins.data_ptr(), t_ns.data_ptr(), len(units),
                                                  t_unit.data_ptr(), t_lo.data_ptr(), t_len.data_ptr(), t_ptr.data_ptr(),
                                                  t_ol.data_ptr(), t_st.data_ptr(), k, t_scr.data_ptr(), sb, st, C.byref(e))
    if not sync:
        return rc, (t_out, t_ol, t_st, t_tabs, t_ins, t_ns, t_unit, t_lo, t_len, t_ptr, t_scr)
    torch.cuda.synchronize()
    if rc:
        assert bool((t_ol == -1).all()) and bool((t_out == 0xEE).all())
        return rc, None
    assert bool((t_scr[sb:] == 0x5A).all()), "scratch overrun"
    back, ols = t_out.cpu().numpy(), t_ol.cpu().numpy()
    sts = t_st.cpu().numpy().view(np.uint64).reshape(-1, 4)
    assert (back[:3] == 0xEE).all() and int(ols[k]) == -1
    got = []
    for i, (o, ln) in enumerate(zip(offs, lens)):
        assert (back[o + ln:o + ln + 16] == 0xEE).all(), ("output overrun", i)
        m = int(ols[i])
        assert 0 <= m <= ln
        got.append((_status(sts[i]), back[o:o + m].tobytes()))
    return 0, got


def against_k12(snap, streams, ranges):
    """streams: [(stream, kwargs of the build)]. One table per stream, every range in one read, each stream's ranges
    compared with sb_frame_decode_ranges_device_ws on that stream. Returns the results and the builds' results."""
    units, results = [], []
    for s, kw in streams:
        t_in = upload(s)
        rc, table, res = build(snap, t_in, len(s), **kw)
        assert rc == 0
        units.append((t_in, len(s), table))
        results.append(res)
    rc, got = read(snap, units, ranges)
    assert rc == 0
    for u, (s, kw) in enumerate(streams):
        mine = [(lo, n) for v, lo, n in ranges if v == u]
        if mine:
            rc, want, res = call(snap, units[u][0], len(s), mine, **kw)
            assert rc == 0 and res == results[u], u
            assert [g for (v, _, _), g in zip(ranges, got) if v == u] == want, u
    return got, results


def test_corpus_in_one_table_set(snap, oracle):
    """Every corpus file as one stream, all tabled, random ranges spread over all of them in one call."""
    rng = random.Random(1)
    streams = [(oracle.frame_encode(corpus(name)), {}) for name in CORPUS]
    fulls = [full_decode(snap, s) for s, _ in streams]
    assert all(st == OK for st, _ in fulls)
    ranges = []
    for u, (_, full) in enumerate(fulls):
        ranges += [(u, rng.randrange(len(full) + 1), rng.randrange(0, 200000)) for _ in range(25)]
    rng.shuffle(ranges)
    got, _ = against_k12(snap, streams, ranges)
    assert all(g == (OK, fulls[u][1][lo:lo + n]) for (u, lo, n), g in zip(ranges, got))


def test_multi_mib_walked_damaged_and_fragments(snap, oracle):
    rng = random.Random(2)
    big = oracle.frame_encode(_text(8 * MIB, 3))
    mid = oracle.frame_encode(_text(3 * MIB + 5, 4))
    noise = oracle.frame_encode(np.random.default_rng(2).integers(0, 256, 3 * MIB, dtype=np.uint8).tobytes())
    g = ls.gen_frame(rng, oracle.crc32c_masked, 30)
    walked = g.stream + IDENT + g.stream[10:]                            # a repeated identifier: walked
    cix = chain(mid)
    damaged = _flip(_flip(mid, cix[5] + 40), cix[20] + 5)
    streams = [(big, {}), (big, {"index": chain(big)}), (mid, {}), (noise, {}), (walked, {}), (damaged, {}),
               (damaged, {"index": cix}), (mid[:-7], {}), (big[10:], {"fragment": True}),
               (mid[10:], {"fragment": True, "index": chain(mid[10:], True)}), (mid, {"max_chunks": 40})]
    ranges = []
    for u, (s, kw) in enumerate(streams):
        sp, total = spans(s, kw.get("fragment", False))
        ranges += [(u, lo, n) for lo, n in boundary_ranges([o for o, _ in sp], total)[:30]]
        ranges += [(u, rng.randrange(total + 2), rng.randrange(1, 2 * MIB)) for _ in range(10)]
    rng.shuffle(ranges)
    got, res = against_k12(snap, streams, ranges)
    assert res[-1][0] == ("Invalid", 40, 1, 0)
    assert any(g[0][0] == "Checksum" for (u, _, _), g in zip(ranges, got) if u == 5)


def test_decoded_length_over_4_gib(snap, oracle):
    """A stream of 4.2 GiB decoded, tiled from one encoded fragment: ranges straddling 2^32 and at the ends."""
    import torch
    unit = _text(64 * MIB, 11)
    frag = snap.frame.encode_chunks(unit, include_ident=False)
    reps = 67
    t_in = torch.cat([upload(frag)[:len(frag)].repeat(reps), torch.zeros(16, dtype=torch.uint8, device="cuda")])
    n, D = len(frag) * reps, len(unit)
    total = D * reps
    ranges = [((1 << 32) - 100, 200), ((1 << 32) - 3 * BLOCK - 1, 5 * BLOCK + 7), ((1 << 32) + 5, 1), (0, 10),
              (total - 50, 100), (total - 3 * MIB, 3 * MIB), (D - 1, 2), (total + 1, 5)]
    tile = unit + unit
    for index in (None, [len(frag) * (k // 1024) + chain(frag, True)[k % 1024] for k in range(1024 * reps)] + [n]):
        kw = {"fragment": True, "index": index, "max_chunks": 1024 * reps + 1}
        rc, table, res = build(snap, t_in, n, **kw)
        assert rc == 0 and res == (OK, total, 1024 * reps)
        rc, got = read(snap, [(t_in, n, table)], [(0, lo, ln) for lo, ln in ranges])
        for (lo, ln), g in zip(ranges, got):
            m = max(0, min(ln, total - lo))
            assert g == (OK, tile[lo % D:lo % D + m]), (lo, ln)
        assert call(snap, t_in, n, ranges, **kw)[1] == got
        del table
    del t_in
    torch.cuda.empty_cache()


def test_mismatch_statuses(snap, oracle):
    """Unit out of range (1), and a table of another length or with a wrong magic (2), beside a good unit."""
    s = oracle.frame_encode(_text(BLOCK + 100, 13))
    data = oracle.frame_decode(s)
    n = len(s)
    t_in = upload(s)
    rc, table, _ = build(snap, t_in, n)
    bad = table.clone()
    bad[0] ^= 1
    units = [(t_in, n, table), (t_in, n, table), (t_in, n, bad)]
    rc, got = read(snap, units, [(0, 0, 10), (1, 0, 10), (2, 0, 10), (3, 0, 10), (9, 1, 0)], in_lens=[n, n + 1, n])
    assert got[0] == (OK, data[:10])
    assert got[1] == (("Invalid", n + 1, n, 2), b"")
    assert got[2] == (("Invalid", n, 0, 2), b"")
    assert got[3] == (("Invalid", 3, 3, 1), b"") and got[4] == (("Invalid", 9, 3, 1), b"")


def test_side_stream_no_allocation_and_fixed_launches(snap, oracle):
    import torch
    L = snap._lib.lib()
    s = oracle.frame_encode(_text(6 * BLOCK + 9, 12))
    data = oracle.frame_decode(s)
    ix = chain(s)
    t_in = upload(s)
    rc, table, _ = build(snap, t_in, len(s))                            # first use of the device
    read(snap, [(t_in, len(s), table)], [(0, 0, 5)])
    allocs = L.sb_alloc_count()
    builds = {}
    for index in (None, ix):
        before = L.sb_launch_count()
        assert build(snap, t_in, len(s), index=index)[0] == 0
        builds[index is None] = L.sb_launch_count() - before
    assert builds == {True: 8, False: 5}
    deltas = set()
    for count in (1, 64):
        for k in (1, 1000):
            ranges = [(i % count, i * 997 % len(data), 5000) for i in range(k)]
            before = L.sb_launch_count()
            rc, got = read(snap, [(t_in, len(s), table)] * count, ranges)
            deltas.add(L.sb_launch_count() - before)
            assert rc == 0 and all(g == (OK, data[lo:lo + n]) for (_, lo, n), g in zip(ranges, got))
    assert deltas == {4}
    assert L.sb_alloc_count() == allocs
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        t2 = upload(s)
        busy = torch.randn(4096, 4096, device="cuda")
        for _ in range(4):
            busy = busy @ busy                                           # pending work ahead of the call
        rc, keep = read(snap, [(t2, len(s), table)], [(0, 100, 3 * BLOCK)], stream=side, sync=False)
        assert rc == 0
    side.synchronize()
    t_out, t_ol = keep[0], keep[1]
    assert int(t_ol[0]) == 3 * BLOCK and t_out[3:3 + 3 * BLOCK].cpu().numpy().tobytes() == data[100:100 + 3 * BLOCK]
    assert L.sb_alloc_count() == allocs


def test_argument_errors_launch_nothing(snap, oracle):
    import torch
    L = snap._lib.lib()
    s = oracle.frame_encode(_text(BLOCK + 1, 13))
    n = len(s)
    t_in = upload(s)
    rc, table, _ = build(snap, t_in, n)
    before = L.sb_launch_count()
    assert build(snap, t_in, n, max_chunks=64, table_bytes=L.sb_frame_table_bytes(64) - 1)[0] == INVALID
    assert build(snap, t_in, n, max_chunks=64, scratch_bytes=L.sb_frame_table_build_scratch_bytes(64) - 1)[0] == INVALID
    assert build(snap, t_in, n, max_chunks=0)[0] == INVALID
    assert build(snap, t_in, n, max_chunks=(1 << 22) - 1)[0] == INVALID
    assert build(snap, t_in, n, index=chain(s), max_chunks=1)[0] == INVALID
    units = [(t_in, n, table)]
    assert read(snap, units, [(0, 0, 5), (0, 9, 9)], scratch_bytes=L.sb_frame_table_ranges_scratch_bytes(2) - 1)[0] == INVALID
    e = snap._lib.SbError()
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()

    def raw_build(d_in=p, tab=p, res=p, scr=p):
        return L.sb_frame_table_build_device_ws(d_in, 16, None, 0, 0, tab, 1 << 19, 8, res, scr, 1 << 19, None, C.byref(e))
    assert raw_build(d_in=None) == INVALID and raw_build(tab=None) == INVALID
    assert raw_build(res=None) == INVALID and raw_build(scr=None) == INVALID

    def raw_read(count=1, nr=1, arrays=(p,) * 10):
        return L.sb_frame_table_decode_ranges_device_ws(*arrays[:3], count, *arrays[3:9], nr, arrays[9], 1 << 20, None,
                                                        C.byref(e))
    for k in range(10):
        assert raw_read(arrays=tuple(None if m == k else p for m in range(10))) == INVALID
    assert raw_read(count=1 << 31) == INVALID and raw_read(nr=1 << 31) == INVALID
    assert raw_read(nr=0, arrays=(None,) * 10) == 0
    assert L.sb_launch_count() == before
    torch.cuda.synchronize()


def test_table_reader(snap, oracle):
    import torch
    rng = random.Random(5)
    data = _text(5 * MIB + 3, 14)
    s = oracle.frame_encode(data)
    g = ls.gen_frame(rng, oracle.crc32c_masked, 30)
    srcs = [s, upload(s)[:len(s)].clone(), g.stream, oracle.frame_encode(b""), oracle.frame_encode(b"x" * 70000)]
    wants = [data, data, g.data, b"", b"x" * 70000]
    rd = snap.frame.TableReader(srcs)
    assert len(rd) == len(srcs) and rd.lengths == [len(w) for w in wants]
    assert rd.read(0, 0, len(data) + 10) == data
    ranges = [(i, rng.randrange(len(wants[i]) + 2), rng.randrange(0, 300000)) for i in (rng.randrange(5) for _ in range(80))]
    assert rd.read_ranges(ranges) == [wants[i][lo:lo + n] for i, lo, n in ranges]
    assert rd.read_ranges([]) == []
    rd.RANGES_PER_CALL = 7                                               # several calls per read_ranges
    ranges = [(i % 3, i * 4099, 4096) for i in range(40)]
    assert rd.read_ranges(ranges) == [wants[i][lo:lo + n] for i, lo, n in ranges]
    with pytest.raises(IndexError):
        rd.read(5, 0, 1)
    frag = snap.frame.TableReader([g.stream[10:]], fragment=True)
    assert frag.read(0, 0, len(g.data)) == g.data
    bad = _flip(s, chain(s)[3] + 5)
    rd = snap.frame.TableReader([s, bad])
    assert rd.read(1, 0, 2 * BLOCK) == data[:2 * BLOCK]
    with pytest.raises(snap.Error) as ei:
        rd.read_ranges([(0, 0, 4 * BLOCK), (1, 0, 4 * BLOCK)])
    assert ei.value.as_tuple()[0] == "Checksum"
    tiny = IDENT + ls.chunk(0x01, b"a", oracle.crc32c_masked(b"a")) * 100   # more chunks than n // 1024 + 16
    small = snap.frame.TableReader([tiny])
    assert small.lengths == [100] and small.read(0, 0, 200) == b"a" * 100
    torch.cuda.synchronize()
