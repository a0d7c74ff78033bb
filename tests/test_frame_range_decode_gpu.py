"""Range decode of one frame stream on the GPU (sb_frame_decode_ranges_device_ws and frame.RangeReader): K5's index
phase, then only the chunks the ranges cover are decoded and checksummed. Every range must give what the oracle's
frame_decode gives for those bytes (or, for a damaged stream, the error the rule of include/snapb200.h names), and agree
with sb_frame_decode_device_ws's output."""
import ctypes as C
import random

import numpy as np
import pytest

import legal_streams as ls
from conftest import CORPUS, corpus
from test_frame_batch_decode_emu import IDENT, _flip, _text, chain, oracle_decode
from test_frame_batch_decode_gpu import NAMES
from test_frame_range_decode_emu import OK, boundary_ranges, spans, verifies

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


def _status(row):
    code = int(row[0] & 0xFFFFFFFF)
    return (NAMES.get(code, str(code)), int(row[1]), int(row[2]), int(row[3]))


def upload(stream):
    import torch
    return torch.from_numpy(np.frombuffer(bytes(stream) + bytes(16), dtype=np.uint8).copy()).cuda()


def call(snap, t_in, n, ranges, index=None, fragment=False, max_chunks=None, scratch_bytes=None, stream=None, sync=True):
    """One sb_frame_decode_ranges_device_ws call; every buffer has 16 guard bytes behind it and the scratch 4 KiB.
    Returns rc, [(status, bytes)], (status, bytes, nchunks)."""
    import torch
    L = snap._lib.lib()
    k = len(ranges)
    if max_chunks is None:
        max_chunks = min(n // 8 + 16, (1 << 22) - 2)
    lens = [ln for _, ln in ranges]
    offs, at = [], 3
    for ln in lens:
        offs.append(at)
        at += ln + 16 + 1 - ln % 2
    t_out = torch.full((at + 16,), 0xEE, dtype=torch.uint8, device="cuda")
    to64 = lambda v: torch.from_numpy(np.array(v, dtype=np.uint64).view(np.int64)).cuda()
    t_lo, t_len = to64([lo for lo, _ in ranges] + [0]), to64(lens + [0])
    t_ptr = to64([t_out.data_ptr() + o for o in offs] + [0])
    t_ol = torch.full((k + 1,), -1, dtype=torch.int64, device="cuda")
    t_st = torch.full((max(k, 1) * 32,), 0x77, dtype=torch.uint8, device="cuda")
    t_res = torch.full((64,), 0x77, dtype=torch.uint8, device="cuda")
    t_ix = to64(list(index) + [7]) if index is not None else None
    need = L.sb_frame_decode_ranges_scratch_bytes(max_chunks, k)
    sb = need if scratch_bytes is None else scratch_bytes
    t_scr = torch.full((sb + 4096,), 0x5A, dtype=torch.uint8, device="cuda")
    e = snap._lib.SbError()
    st = (stream or torch.cuda.current_stream()).cuda_stream
    rc = L.sb_frame_decode_ranges_device_ws(t_in.data_ptr(), n, t_ix.data_ptr() if t_ix is not None else None,
                                            len(index) - 1 if index is not None else 0, 1 if fragment else 0,
                                            t_lo.data_ptr(), t_len.data_ptr(), t_ptr.data_ptr(), t_ol.data_ptr(),
                                            t_st.data_ptr(), k, t_res.data_ptr(), t_scr.data_ptr(), sb, max_chunks, st,
                                            C.byref(e))
    if not sync:
        return rc, (t_out, t_lo, t_len, t_ptr, t_ol, t_st, t_res, t_ix, t_scr)
    torch.cuda.synchronize()
    if rc:
        assert bool((t_ol == -1).all()) and bool((t_out == 0xEE).all()) and bool((t_res == 0x77).all())
        return rc, None, None
    assert bool((t_scr[sb:] == 0x5A).all()), "scratch overrun"
    back = t_out.cpu().numpy()
    ols = t_ol.cpu().numpy()
    sts = t_st.cpu().numpy().view(np.uint64).reshape(-1, 4)
    got = []
    for i, (o, ln) in enumerate(zip(offs, lens)):
        assert (back[o + ln:o + ln + 16] == 0xEE).all(), ("output overrun", i)
        m = int(ols[i])
        assert 0 <= m <= ln
        got.append((_status(sts[i]), back[o:o + m].tobytes()))
    assert int(ols[k]) == -1
    r = snap._lib.SbFrameResult.from_buffer_copy(t_res.cpu().numpy().tobytes()[:C.sizeof(snap._lib.SbFrameResult)])
    return 0, got, (_status([r.status.code, r.status.a, r.status.b, r.status.c]), r.bytes, r.nchunks)


def check_valid(snap, data, stream, ranges, fragment=False, **kw):
    rc, got, res = call(snap, upload(stream), len(stream), ranges, fragment=fragment, **kw)
    assert rc == 0
    for (lo, n), g in zip(ranges, got):
        assert g == (OK, data[lo:lo + n]), (lo, n, g[0])
    assert res[0] == OK and res[1] == len(data)
    return res


def full_decode(snap, stream, fragment=False):
    """sb_frame_decode_device_ws of the whole stream: (status, bytes)."""
    import gpu_helpers
    return gpu_helpers.frame_decode_device(stream, max(len(stream) * 30, 1 << 20), fragment=fragment, ws=True)


@pytest.mark.parametrize("how", ["k7", "index", "walk"])
def test_encoder_output(snap, oracle, how):
    s = oracle.frame_encode(_text(5 * BLOCK + 777, 1))
    ix = chain(s)
    sp, total = spans(s)
    kw = {"index": ix} if how == "index" else {"index": ix[:2] + [ix[-1]]} if how == "walk" else {}
    res = check_valid(snap, oracle.frame_decode(s), s, boundary_ranges([o for o, _ in sp], total), **kw)
    assert res[2] == len(sp)


def test_generated_streams_and_fragments(snap, oracle):
    rng = random.Random(3)
    empty = ls.chunk(0x01, b"", oracle.crc32c_masked(b"")) + ls.chunk(0x00, b"\x00", oracle.crc32c_masked(b""))
    for k in range(4):
        g = ls.gen_frame(rng, oracle.crc32c_masked, 14)
        s = g.stream + empty + (IDENT if k % 2 else b"") + ls.gen_frame(rng, oracle.crc32c_masked, 5).stream[10:]
        sp, total = spans(s)
        ranges = boundary_ranges([o for o, _ in sp], total) + [(o, 0) for o, d in sp if d == 0]
        check_valid(snap, oracle.frame_decode(s), s, ranges)
        frag = s[10:]
        check_valid(snap, oracle.frame_decode(s), frag, ranges, fragment=True)


@pytest.mark.parametrize("where", ["crc", "body"])
@pytest.mark.parametrize("indexed", [False, True])
def test_one_corrupted_chunk(snap, oracle, where, indexed):
    clean = oracle.frame_encode(_text(4 * BLOCK + 999, 5))
    ix = chain(clean)
    data = oracle.frame_decode(clean)
    sp, total = spans(clean)
    j = 2
    s = _flip(clean, ix[j] + (5 if where == "crc" else 40))
    err = oracle_decode(oracle, s[:ix[j + 1]])[0]
    ranges = boundary_ranges([o for o, _ in sp], total)
    rc, got, res = call(snap, upload(s), len(s), ranges, index=ix if indexed else None)
    assert rc == 0 and res == (OK, total, len(sp))
    for (lo, n), g in zip(ranges, got):
        if verifies(sp[j][0], sp[j][1], lo, n, total):
            assert g == (err, data[lo:max(sp[j][0], lo)]), (lo, n)
        else:
            assert g == (OK, data[lo:lo + n]), (lo, n)


def test_truncated_stream_and_short_table(snap, oracle):
    clean = oracle.frame_encode(_text(3 * BLOCK + 100, 7))
    ix = chain(clean)
    s = clean[:-5]
    err = oracle_decode(oracle, s)[0]
    data = oracle.frame_decode(clean[:ix[-2]])
    total = len(data)
    ranges = [(0, total), (0, total + 1), (total - 1, 1), (total - 1, 2), (total, 1), (total + 9, 1), (5, 10), (total, 0)]
    rc, got, res = call(snap, upload(s), len(s), ranges)
    assert rc == 0 and res == (err, total, 3)
    for (lo, n), g in zip(ranges, got):
        assert g == (err if lo + n > total else OK, data[lo:lo + n]), (lo, n)
    rc, got, res = call(snap, upload(clean), len(clean), ranges, max_chunks=3)
    assert rc == 0 and res[0] == ("Invalid", 3, 1, 0)
    assert all(g == (("Invalid", 3, 1, 0), b"") for g in got)


def test_corpus_against_full_decode(snap, oracle):
    """Every corpus file and multi-MiB generated streams: random ranges equal slices of sb_frame_decode_device_ws."""
    rng = random.Random(1)
    streams = [oracle.frame_encode(corpus(name)) for name in CORPUS]
    streams += [oracle.frame_encode(_text(n, n)) for n in (3 * MIB + 5, 8 * MIB)]
    streams.append(oracle.frame_encode(np.random.default_rng(2).integers(0, 256, 3 * MIB, dtype=np.uint8).tobytes()))
    for s in streams:
        st, full = full_decode(snap, s)
        assert st == OK
        sp, total = spans(s)
        ranges = boundary_ranges([o for o, _ in sp], total)[:40]
        ranges += [(rng.randrange(total + 1), rng.randrange(1, 2 * MIB)) for _ in range(20)]
        check_valid(snap, full, s, ranges)
        check_valid(snap, full, s, ranges, index=chain(s))


def test_decoded_length_over_4_gib(snap, oracle):
    """A stream of 4.2 GiB decoded, tiled from one encoded fragment (frame chunks are independent): ranges straddling
    2^32 and at the ends."""
    import torch
    unit = _text(64 * MIB, 11)
    frag = snap.frame.encode_chunks(unit, include_ident=False)
    reps = 67
    t_in = torch.cat([upload(frag)[:len(frag)].repeat(reps), torch.zeros(16, dtype=torch.uint8, device="cuda")])
    n, D = len(frag) * reps, len(unit)
    total = D * reps
    assert total > (1 << 32) + 64 * MIB
    ranges = [((1 << 32) - 100, 200), ((1 << 32) - 3 * BLOCK - 1, 5 * BLOCK + 7), ((1 << 32) + 5, 1), (0, 10),
              (total - 50, 100), (total - 3 * MIB, 3 * MIB), (D - 1, 2), (total + 1, 5)]
    tile = unit + unit
    for index in (None, [len(frag) * (k // 1024) + chain(frag, True)[k % 1024] for k in range(1024 * reps)] + [n]):
        rc, got, res = call(snap, t_in, n, ranges, fragment=True, index=index, max_chunks=1024 * reps + 1)
        assert rc == 0 and res == (OK, total, 1024 * reps)
        for (lo, ln), g in zip(ranges, got):
            m = max(0, min(ln, total - lo))
            assert g == (OK, tile[lo % D:lo % D + m]), (lo, ln)
    del t_in
    torch.cuda.empty_cache()


def test_side_stream_no_allocation_and_fixed_launches(snap, oracle):
    import torch
    L = snap._lib.lib()
    s = oracle.frame_encode(_text(6 * BLOCK + 9, 12))
    data = oracle.frame_decode(s)
    ix = chain(s)
    t_in = upload(s)
    call(snap, t_in, len(s), [(0, 5)])                                   # first use of the device
    allocs = L.sb_alloc_count()
    deltas = {}
    for index in (None, ix):
        for k in (0, 1, 1000):
            ranges = [(i * 997 % len(data), 5000) for i in range(k)]
            before = L.sb_launch_count()
            rc, got, _ = call(snap, t_in, len(s), ranges, index=index)
            deltas[(index is None, k)] = L.sb_launch_count() - before
            assert rc == 0 and all(g == (OK, data[lo:lo + n]) for (lo, n), g in zip(ranges, got))
    assert deltas[(True, 0)] == deltas[(True, 1)] == deltas[(True, 1000)] == 11
    assert deltas[(False, 0)] == deltas[(False, 1)] == deltas[(False, 1000)] == 8
    assert L.sb_alloc_count() == allocs
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        t2 = upload(s)
        busy = torch.randn(4096, 4096, device="cuda")
        for _ in range(4):
            busy = busy @ busy                                           # pending work ahead of the call
        rc, keep = call(snap, t2, len(s), [(100, 3 * BLOCK)], stream=side, sync=False)
        assert rc == 0
    side.synchronize()
    t_out, t_ol = keep[0], keep[4]
    assert int(t_ol[0]) == 3 * BLOCK and t_out[3:3 + 3 * BLOCK].cpu().numpy().tobytes() == data[100:100 + 3 * BLOCK]
    assert L.sb_alloc_count() == allocs


def test_argument_errors_launch_nothing(snap, oracle):
    import torch
    L = snap._lib.lib()
    s = oracle.frame_encode(_text(BLOCK + 1, 13))
    t_in = upload(s)
    call(snap, t_in, len(s), [(0, 5)])
    before = L.sb_launch_count()
    need = L.sb_frame_decode_ranges_scratch_bytes(64, 2)
    assert call(snap, t_in, len(s), [(0, 5), (9, 9)], max_chunks=64, scratch_bytes=need - 1)[0] == INVALID
    assert call(snap, t_in, len(s), [(0, 5)], max_chunks=0)[0] == INVALID
    assert call(snap, t_in, len(s), [(0, 5)], max_chunks=(1 << 22) - 1)[0] == INVALID
    assert call(snap, t_in, len(s), [(0, 5)], index=chain(s), max_chunks=1)[0] == INVALID
    e = snap._lib.SbError()
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()

    def raw(d_in=p, res=p, scr=p, nr=0, arrays=(None,) * 5):
        return L.sb_frame_decode_ranges_device_ws(d_in, 16, None, 0, 0, *arrays, nr, res, scr, 1 << 20, 8, None,
                                                  C.byref(e))
    assert raw(d_in=None) == INVALID and raw(res=None) == INVALID and raw(scr=None) == INVALID
    for k in range(5):
        assert raw(nr=1, arrays=tuple(None if m == k else p for m in range(5))) == INVALID
    assert raw(nr=1 << 31, arrays=(p,) * 5) == INVALID
    assert L.sb_launch_count() == before
    torch.cuda.synchronize()


def test_range_reader(snap, oracle):
    import torch
    rng = random.Random(5)
    data = _text(5 * MIB + 3, 14)
    s = oracle.frame_encode(data)
    g = ls.gen_frame(rng, oracle.crc32c_masked, 30)
    for src, want, frag in ((s, data, False), (upload(s)[:len(s)].clone(), data, False), (g.stream, g.data, False),
                            (g.stream[10:], g.data, True)):
        rd = snap.frame.RangeReader(src, fragment=frag)
        assert len(rd) == len(want)
        assert rd.read(0, len(want) + 10) == want
        ranges = [(rng.randrange(len(want) + 2), rng.randrange(0, 300000)) for _ in range(50)]
        assert rd.read_ranges(ranges) == [want[lo:lo + n] for lo, n in ranges]
        assert rd.read_ranges([]) == []
    rd = snap.frame.RangeReader(s)
    rd.RANGES_PER_CALL = 7                                               # several calls per read_ranges
    ranges = [(i * 4099, 4096) for i in range(40)]
    assert rd.read_ranges(ranges) == [data[lo:lo + n] for lo, n in ranges]
    bad = _flip(s, chain(s)[3] + 5)
    rd = snap.frame.RangeReader(bad)
    assert rd.read(0, 2 * BLOCK) == data[:2 * BLOCK]
    with pytest.raises(snap.Error) as ei:
        rd.read(0, 4 * BLOCK)
    assert ei.value.as_tuple()[0] == "Checksum"
    torch.cuda.synchronize()
