"""Seek tables of a batch of frame streams on the GPU (sb_frame_table_build_batch_device_ws and frame.TableReader built
on it). Every unit that fits the chunk table must get the table bytes and result sb_frame_table_build_device_ws gives
that stream alone; the first unit that does not fit and every unit after it get the 64-byte too-small header."""
import ctypes as C
import random

import numpy as np
import pytest

import legal_streams as ls
from conftest import CORPUS, corpus
from test_frame_batch_decode_emu import IDENT, _flip, _text, chain
from test_frame_range_decode_gpu import _status, upload
from test_frame_table_gpu import build

pytestmark = pytest.mark.gpu

BLOCK = 65536
HEAD = 64
REC = 32
INVALID = 202


@pytest.fixture(scope="module")
def snap():
    import torch
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)
    import gpu_helpers
    return gpu_helpers.snap()


def batch_build(snap, ins, flags=0, index=None, max_chunks=None, tables_bytes=None, scratch_bytes=None, stream=None,
                sync=True):
    """One sb_frame_table_build_batch_device_ws call over device inputs [(tensor, n)]. The tables, offsets, results and
    scratch have 4 KiB of guard bytes behind them. Returns rc and (tables tensor, offsets, [(status, bytes, nchunks)])."""
    import torch
    L = snap._lib.lib()
    k = len(ins)
    if max_chunks is None:
        max_chunks = min(sum(n // 8 + 2 for _, n in ins), (1 << 22) - 2)
    in_bytes = sum(n for _, n in ins)
    to64 = lambda v: torch.from_numpy(np.array(v, dtype=np.uint64).view(np.int64)).cuda()
    t_ptrs = to64([t.data_ptr() for t, _ in ins] + [0])
    t_lens = torch.from_numpy(np.array([n for _, n in ins] + [0], dtype=np.uint32).view(np.int32)).cuda()
    tb = L.sb_frame_table_batch_bytes(k, max_chunks) if tables_bytes is None else tables_bytes
    sb = L.sb_frame_table_build_batch_scratch_bytes(k, in_bytes, max_chunks) if scratch_bytes is None else scratch_bytes
    t_tab = torch.full((tb + 4096,), 0x3C, dtype=torch.uint8, device="cuda")
    t_offs = torch.full((k + 1 + 512,), -1, dtype=torch.int64, device="cuda")
    rsz = C.sizeof(snap._lib.SbFrameResult)
    t_res = torch.full((k * rsz + 4096,), 0x77, dtype=torch.uint8, device="cuda")
    t_scr = torch.full((sb + 4096,), 0x5A, dtype=torch.uint8, device="cuda")
    t_ix = t_at = None
    if index is not None:
        at, flat = [], []
        for ix in index:
            at.append(len(flat))
            flat += list(ix)
        at.append(len(flat))
        t_ix, t_at = to64(flat + [7]), to64(at)
    b = snap._lib.SbBatch()
    b.in_ptrs, b.in_lens, b.count = t_ptrs.data_ptr(), t_lens.data_ptr(), k
    e = snap._lib.SbError()
    st = (stream or torch.cuda.current_stream()).cuda_stream
    rc = L.sb_frame_table_build_batch_device_ws(C.byref(b), in_bytes, flags, t_ix.data_ptr() if t_ix is not None else None,
                                                t_at.data_ptr() if t_at is not None else None, max_chunks, t_tab.data_ptr(),
                                                tb, t_offs.data_ptr(), t_res.data_ptr(), t_scr.data_ptr(), sb, st,
                                                C.byref(e))
    keep = (t_tab, t_offs, t_res, t_scr, t_ptrs, t_lens, t_ix, t_at)
    if not sync:
        return rc, keep
    torch.cuda.synchronize()
    assert bool((t_scr[sb:] == 0x5A).all()) and bool((t_res[k * rsz:] == 0x77).all()), "scratch or results overrun"
    if rc or k == 0:
        assert bool((t_tab == 0x3C).all()) and bool((t_offs == -1).all()) and bool((t_res == 0x77).all())
        return rc, None
    offs = t_offs.cpu().numpy()
    assert (offs[k + 1:] == -1).all() and offs[0] == 0 and offs[k] <= tb
    assert bool((t_tab[int(offs[k]):] == 0x3C).all()), "written past the packed tables"
    raw = t_res[:k * rsz].cpu().numpy().view(np.uint64).reshape(k, rsz // 8)
    res = [(_status(r[:4]), int(r[4]), int(r[5]) & 0xFFFFFFFF) for r in raw]
    assert all(int(r[5]) >> 32 == 0 and int(r[0]) >> 32 == 0 for r in raw)   # the padding is written as zeros
    assert all(int(offs[i + 1] - offs[i]) == HEAD + REC * res[i][2] for i in range(k))
    return 0, (t_tab, [int(x) for x in offs[:k + 1]], res)


def single(snap, t, n, fragment=False, index=None):
    """sb_frame_table_build_device_ws alone: (table bytes cut to its chunks, result)."""
    rc, table, res = build(snap, t, n, fragment=fragment, index=index,
                           max_chunks=max(min(n // 8 + 16, (1 << 22) - 2), len(index or []) + 1))
    assert rc == 0
    return table[:HEAD + REC * res[2]].cpu().numpy().tobytes(), res


def check(snap, streams, **kw):
    ins = [(upload(s), len(s)) for s in streams]
    rc, (tab, offs, res) = batch_build(snap, ins, **kw)
    assert rc == 0
    back = tab.cpu().numpy()
    ix = kw.get("index")
    for i, (t, n) in enumerate(ins):
        want_t, want_r = single(snap, t, n, fragment=bool(kw.get("flags", 0) & 1), index=ix[i] if ix else None)
        assert res[i] == want_r, (i, res[i], want_r)
        assert back[offs[i]:offs[i + 1]].tobytes() == want_t, i
    return tab, offs, res


def corpus_and_generated(oracle):
    rng = random.Random(31)
    ss = [oracle.frame_encode(corpus(name)) for name in CORPUS]
    ss += [ls.gen_frame(rng, oracle.crc32c_masked, k).stream for k in (1, 5, 12, 30)]
    three = oracle.frame_encode(_text(3 * BLOCK - 7, 5))
    c3 = chain(three)
    ss += [_flip(three, c3[1] + 6), three[:-3], three[:c3[2] + 2], oracle.frame_encode(b""), b"",
           oracle.frame_encode(_text(5000, 1)) + oracle.frame_encode(_text(300, 2))]   # a repeated identifier
    return ss


def test_corpus_and_generated_streams(snap, oracle):
    streams = corpus_and_generated(oracle)
    check(snap, streams)
    check(snap, streams, index=[chain(s) if s else [0] for s in streams])
    frags = [oracle.frame_encode(corpus(name))[10:] for name in CORPUS[:5]]
    check(snap, frags, flags=1)


def test_unit_over_4_gib_decoded(snap, oracle):
    """A long run of zeros: compressed far below 2^32, decoded past it. K11 could not decode it into a 32-bit cap; its
    table has the exact 64-bit total."""
    import torch
    chunk = oracle.frame_encode(bytes(BLOCK))[10:]
    reps = (1 << 32) // BLOCK + 300
    t_chunk = torch.from_numpy(np.frombuffer(chunk, dtype=np.uint8).copy()).cuda()
    big = torch.cat([torch.from_numpy(np.frombuffer(IDENT, dtype=np.uint8).copy()).cuda(), t_chunk.repeat(reps),
                     torch.zeros(16, dtype=torch.uint8, device="cuda")])
    n = big.numel() - 16
    small = oracle.frame_encode(_text(70000, 3))
    t_small = upload(small)
    rc, (tab, offs, res) = batch_build(snap, [(t_small, len(small)), (big, n)], max_chunks=reps + 2 + 16)
    assert rc == 0
    assert res[1] == (("Ok", 0, 0, 0), reps * BLOCK, reps) and reps * BLOCK > 1 << 32
    want_t, want_r = single(snap, big, n)
    assert want_r == res[1] and torch.equal(tab[offs[1]:offs[2]].cpu(), torch.from_numpy(np.frombuffer(want_t, np.uint8).copy()))
    assert res[0] == single(snap, t_small, len(small))[1]
    del big, tab
    torch.cuda.empty_cache()


def test_many_small_streams(snap, oracle):
    """10,000 small streams in one call; every table equals its single build (made without a wait in between)."""
    import torch
    L = snap._lib.lib()
    rng = random.Random(7)
    pool = _text(3 * BLOCK + 100000, 1)
    streams = []
    for i in range(10000):
        if i % 10 == 3:
            streams.append(ls.gen_frame(rng, oracle.crc32c_masked, rng.randrange(1, 6)).stream)
        else:
            at = rng.randrange(100000)
            streams.append(oracle.frame_encode(pool[at:at + rng.randrange(0, 3 * BLOCK)]))
    ins = [(upload(s), len(s)) for s in streams]
    rc, (tab, offs, res) = batch_build(snap, ins)
    assert rc == 0
    caps = [n // 1024 + 16 for _, n in ins]                               # a generated chunk is at least 1 KiB
    slot = [L.sb_frame_table_bytes(c) for c in caps]
    at = np.cumsum([0] + slot)
    t_single = torch.empty(int(at[-1]), dtype=torch.uint8, device="cuda")
    rsz = C.sizeof(snap._lib.SbFrameResult)
    t_res = torch.zeros(len(ins) * rsz, dtype=torch.uint8, device="cuda")
    need = max(L.sb_frame_table_build_scratch_bytes(c) for c in caps)
    scr = torch.empty(need, dtype=torch.uint8, device="cuda")
    e = snap._lib.SbError()
    for i, ((t, n), c) in enumerate(zip(ins, caps)):
        assert L.sb_frame_table_build_device_ws(t.data_ptr(), n, None, 0, 0, t_single.data_ptr() + int(at[i]), slot[i], c,
                                                t_res.data_ptr() + i * rsz, scr.data_ptr(), need,
                                                torch.cuda.current_stream().cuda_stream, C.byref(e)) == 0
    mine, theirs = tab.cpu().numpy(), t_single.cpu().numpy()
    raw = t_res.cpu().numpy().view(np.uint64).reshape(len(ins), rsz // 8)
    for i in range(len(ins)):
        want = (_status(raw[i][:4]), int(raw[i][4]), int(raw[i][5]) & 0xFFFFFFFF)
        assert res[i] == want, i
        assert mine[offs[i]:offs[i + 1]].tobytes() == theirs[int(at[i]):int(at[i]) + offs[i + 1] - offs[i]].tobytes(), i


def test_too_small_chunk_table(snap, oracle):
    enc = oracle.frame_encode
    streams = [enc(_text(n, n)) for n in (100000, 5000, 200000, 70000)]
    ins = [(upload(s), len(s)) for s in streams]
    rc, (tab, offs, res) = batch_build(snap, ins, max_chunks=2 + 1 + 3)   # the third unit is one chunk short
    assert rc == 0
    for i in (0, 1):
        assert res[i] == single(snap, *ins[i])[1]
    back = tab.cpu().numpy()
    for i in (2, 3):
        assert res[i] == (("Invalid", 6, 1, 0), 0, 0)
        h = back[offs[i]:offs[i + 1]].view(np.uint64)
        assert len(h) == 8 and [int(x) for x in h[1:4]] == [len(streams[i]), 0, 1 << 32]
        assert [int(x) for x in h[4:]] == [INVALID, 6, 1, 0]


def test_fixed_launches_no_allocation_side_stream(snap, oracle):
    import torch
    L = snap._lib.lib()
    streams = [oracle.frame_encode(_text(n, n)) for n in (1000, 200000, 70000, 5 * BLOCK)]
    ins = [(upload(s), len(s)) for s in streams]
    index = [chain(s) for s in streams]
    batch_build(snap, ins)
    allocs = L.sb_alloc_count()
    deltas = {False: set(), True: set()}
    for count in (1, 4, 64):
        for indexed in (False, True):
            u = (ins * 16)[:count]
            before = L.sb_launch_count()
            rc, _ = batch_build(snap, u, index=(index * 16)[:count] if indexed else None)
            assert rc == 0
            deltas[indexed].add(L.sb_launch_count() - before)
    assert len(deltas[False]) == 1 and len(deltas[True]) == 1, deltas
    assert L.sb_alloc_count() == allocs
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        t2 = upload(streams[3])
        busy = torch.randn(4096, 4096, device="cuda")
        for _ in range(4):
            busy = busy @ busy                                           # pending work ahead of the call
        rc, keep = batch_build(snap, [(t2, len(streams[3]))], stream=side, sync=False)
        assert rc == 0
    side.synchronize()
    t_tab, t_offs = keep[0], keep[1]
    want_t, _ = single(snap, t2, len(streams[3]))
    assert int(t_offs[1]) == len(want_t) and t_tab[:len(want_t)].cpu().numpy().tobytes() == want_t
    assert L.sb_alloc_count() == allocs


def test_argument_errors_launch_nothing(snap, oracle):
    import torch
    L = snap._lib.lib()
    s = oracle.frame_encode(_text(BLOCK + 1, 13))
    ins = [(upload(s), len(s))]
    before = L.sb_launch_count()
    assert batch_build(snap, ins, max_chunks=64, tables_bytes=L.sb_frame_table_batch_bytes(1, 64) - 1)[0] == INVALID
    assert batch_build(snap, ins, max_chunks=64,
                       scratch_bytes=L.sb_frame_table_build_batch_scratch_bytes(1, len(s), 64) - 1)[0] == INVALID
    assert batch_build(snap, ins, max_chunks=0)[0] == INVALID
    assert batch_build(snap, ins, max_chunks=(1 << 22) - 1)[0] == INVALID
    assert batch_build(snap, [], max_chunks=8)[0] == 0                    # count == 0: nothing launched or written
    e = snap._lib.SbError()
    buf = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    p = buf.data_ptr()
    b = snap._lib.SbBatch()
    b.in_ptrs, b.in_lens, b.count = p, p, 1

    def raw(bb=C.byref(b), a=None, c=None, t=p, o=p, r=p, sc=p):
        return L.sb_frame_table_build_batch_device_ws(bb, 0, 0, a, c, 8, t, 1 << 12, o, r, sc, 1 << 16, None, C.byref(e))
    for kw in ({"bb": None}, {"t": None}, {"o": None}, {"r": None}, {"sc": None}, {"a": p}, {"c": p}):
        assert raw(**kw) == INVALID, kw
    b.count = 1 << 31
    assert raw() == INVALID
    assert L.sb_launch_count() == before
    torch.cuda.synchronize()


def test_table_reader_over_many_small_streams(snap, oracle):
    """2,000 streams, bytes-like and CUDA tensors mixed: reads equal the oracle's decode, and construction makes the same
    library launches for 20 streams as for 2,000 (one group each)."""
    import torch
    L = snap._lib.lib()
    rng = random.Random(12)
    pool = _text(2 * BLOCK + 100000, 2)
    datas = []
    for _ in range(2000):
        at = rng.randrange(100000)
        datas.append(pool[at:at + rng.randrange(0, 2 * BLOCK)])
    streams = [oracle.frame_encode(d) for d in datas]
    mixed = [upload(s)[:len(s)].clone() if i % 3 == 0 else s for i, s in enumerate(streams)]
    launches = []
    for k in (20, 2000):
        before = L.sb_launch_count()
        rd = snap.frame.TableReader(mixed[:k])
        launches.append(L.sb_launch_count() - before)
    assert launches[0] == launches[1]
    assert rd.lengths == [len(d) for d in datas]
    ranges = [(i, rng.randrange(len(datas[i]) + 2), rng.randrange(0, 3 * BLOCK)) for i in (rng.randrange(2000) for _ in range(3000))]
    assert rd.read_ranges(ranges) == [datas[i][lo:lo + n] for i, lo, n in ranges]
    good = oracle.frame_encode(_text(5000, 3))
    rd = snap.frame.TableReader([good, _flip(good, chain(good)[0] + 9)])
    with pytest.raises(snap.Error):
        rd.read(1, 0, 10)
    assert rd.read(0, 0, 100) == _text(5000, 3)[:100]
    torch.cuda.synchronize()
