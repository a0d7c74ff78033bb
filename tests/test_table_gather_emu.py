"""Gathers over tabled frame and raw streams on CPU: the k17_* bodies of rust-snappy_b200/csrc/k17_table_gather.cuh with
the K13 and K15 bodies they run, compiled by g++ against the fiber warp emulator with small grids and 4 decoding warps.
Every range must get exactly the status, out_len and bytes the range call (sb_*_table_decode_ranges_device_ws, under
the emulator harnesses of tests/test_frame_table_emu.py and tests/test_raw_table_emu.py) gives it, and the oracle's
bytes where Ok; nothing may be written outside a range's buffer or the scratch; and the call must decode each edge chunk
once per work item of at most K17_GROUP ranges and each interior pair once. Test tooling only."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import emu_helpers as emu
import legal_streams as ls
import test_frame_table_emu as ft
import test_raw_table_emu as rt
from test_frame_batch_decode_emu import _flip, _text

INVALID = 202
GUARD = 512
BLOCK = 65536
OK = ("Ok", 0, 0, 0)

_HERE = os.path.dirname(os.path.abspath(__file__))
_EMU = os.path.join(_HERE, "emu")
_SO = os.path.join(_EMU, "_build", "libemu_table_gather.so")
_lib = None


def glib():
    """The emulator build of K17 (tests/emu/emu_table_gather.cpp), rebuilt when a source is newer."""
    global _lib
    if _lib is None:
        csrc = os.path.join(os.path.dirname(_HERE), "rust-snappy_b200", "csrc")
        srcs = [os.path.join(_EMU, f) for f in ("emu_table_gather.cpp", "simt_emu.cpp", "simt_emu.h")]
        srcs += [os.path.join(csrc, f) for f in os.listdir(csrc)]
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            tmp = "%s.%d.tmp" % (_SO, os.getpid())
            subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unused-function",
                                   "-Wno-unknown-pragmas", "-Wl,-Bsymbolic", "-o", tmp,
                                   os.path.join(_EMU, "emu_table_gather.cpp"), os.path.join(_EMU, "simt_emu.cpp")])
            os.replace(tmp, _SO)
        _lib = C.CDLL(_SO)
        for f in ("emu_frame_table_gather_scratch_bytes", "emu_raw_table_gather_scratch_bytes"):
            getattr(_lib, f).restype = C.c_uint64
            getattr(_lib, f).argtypes = [C.c_uint32]
        _lib.emu_gather_group.restype = C.c_uint32
        for f in ("emu_frame_table_gather", "emu_raw_table_gather"):
            getattr(_lib, f).argtypes = [C.c_void_p] * 3 + [C.c_uint32] + [C.c_void_p] * 6 + \
                [C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p]
    return _lib


def gather(fmt, units, ranges, rooms, scratch_short=0, in_lens=None, count=None):
    """sb_{fmt}_table_gather_device_ws under the emulator. units: [(input array, table array)], ranges: [(unit, lo, n)],
    rooms: each range's buffer size. Returns rc, [(status, bytes)] and the call's decode count; checks the guard bytes
    around every buffer and the scratch, and that the inputs and tables are unchanged."""
    L = glib()
    k = len(ranges)
    count = len(units) if count is None else count
    before = [(bytes(i), bytes(t)) for i, t in units]
    outs = [np.full(r + 2 * GUARD, 0xEE, dtype=np.uint8) for r in rooms]
    t_tab = np.array([t.ctypes.data for _, t in units] + [0], dtype=np.uint64)
    t_in = np.array([i.ctypes.data for i, _ in units] + [0], dtype=np.uint64)
    t_n = np.array((in_lens if in_lens is not None else [len(i) - 16 for i, _ in units]) + [0], dtype=np.uint64)
    t_unit = np.array([u for u, _, _ in ranges] + [0], dtype=np.uint32)
    t_lo = np.array([lo for _, lo, _ in ranges] + [0], dtype=np.uint64)
    t_len = np.array([n for _, _, n in ranges] + [0], dtype=np.uint64)
    t_ptr = np.array([o.ctypes.data + GUARD for o in outs] + [0], dtype=np.uint64)
    out_lens = np.full(k + 1, 0xDEADBEEF, dtype=np.uint64)
    st = (emu.SbError * (k + 1))()
    size = getattr(L, "emu_%s_table_gather_scratch_bytes" % fmt)(k)
    scratch = np.full(size + 2 * GUARD, 0xCD, dtype=np.uint8)
    dec = C.c_uint64(0xFFFF)
    rc = getattr(L, "emu_%s_table_gather" % fmt)(t_tab.ctypes.data, t_in.ctypes.data, t_n.ctypes.data, count,
                                                 t_unit.ctypes.data, t_lo.ctypes.data, t_len.ctypes.data,
                                                 t_ptr.ctypes.data, out_lens.ctypes.data, C.addressof(st), k,
                                                 scratch.ctypes.data + GUARD, size - scratch_short, C.byref(dec))
    assert [(bytes(i), bytes(t)) for i, t in units] == before
    assert (scratch[:GUARD] == 0xCD).all() and (scratch[GUARD + size:] == 0xCD).all()
    if rc or k == 0:
        assert (out_lens == 0xDEADBEEF).all() and all((o == 0xEE).all() for o in outs) and (scratch == 0xCD).all()
        return rc, None if rc else [], 0
    assert int(out_lens[k]) == 0xDEADBEEF
    got = []
    for i, (o, r) in enumerate(zip(outs, rooms)):
        assert (o[:GUARD] == 0xEE).all() and (o[GUARD + r:] == 0xEE).all(), i
        m = int(out_lens[i])
        assert m <= r, i
        got.append(((ft.status_of if fmt == "frame" else rt.status_of)(st[i]), o[GUARD:GUARD + m].tobytes()))
    return 0, got, dec.value


def frame_spans(table):
    """[(off, dlen)] of a frame table's records, and its total."""
    w = np.frombuffer(table[:ft.HEAD].tobytes(), dtype=np.uint64)
    nch = int(w[3]) & 0xFFFFFFFF
    recs = np.frombuffer(table[ft.HEAD:ft.HEAD + nch * ft.REC].tobytes(), dtype=np.uint64).reshape(nch, 4)
    return [(int(r[3]), int(r[1]) >> 32) for r in recs], int(w[2])


def raw_spans(table):
    dn = rt.head_of(table)[2]
    return [(j * BLOCK, min(BLOCK, dn - j * BLOCK)) for j in range((dn + BLOCK - 1) // BLOCK)], dn


def expected_decodes(spans_of, ranges):
    """(edge work items) + (interior pairs) for valid tables: a range verifies the chunks with off < end and
    off + max(dlen, 1) > lo; its first and last are edges unless inside [lo, end)."""
    G = glib().emu_gather_group()
    edges, interior = {}, 0
    for u, lo, n in ranges:
        sp, total = spans_of[u]
        end = min(lo + n, total)
        run = [k for k, (o, d) in enumerate(sp) if o < end and o + max(d, 1) > lo]
        for k in run:
            o, d = sp[k]
            if o >= lo and o + d <= end:
                interior += 1
            elif k in (run[0], run[-1]):
                edges[(u, k)] = edges.get((u, k), 0) + 1
    return sum((c + G - 1) // G for c in edges.values()) + interior


def frame_both(units, ranges, in_lens=None, overlapping=()):
    """The range call and the gather over the same frame tables: identical results. Returns them and the decode count.
    overlapping: units whose tampered records claim overlapping outputs and decodable chunks that are not inside a range
    in the middle of its run. The range call decodes all of those into one staging slot of the range, so what it returns
    there depends on the order of its warps; they are not compared."""
    rc, want = ft.read(units, ranges, in_lens=in_lens)
    assert rc == 0
    rc, got, dec = gather("frame", units, ranges, [n for _, _, n in ranges], in_lens=in_lens)
    assert rc == 0
    for i, (a, b) in enumerate(zip(got, want)):
        if ranges[i][0] not in overlapping:
            assert a == b, (i, ranges[i], a[0], b[0], len(a[1]), len(b[1]))
    return got, dec


def raw_both(units, ranges, count=None):
    rc, want = rt.read(units, ranges, count=count)
    assert rc == 0

    def room(u, lo, n):
        if u >= len(units) or len(units[u][1]) < rt.HEAD:
            return 0
        return max(0, min(n, rt.head_of(units[u][1])[2] - lo))
    rc, got, dec = gather("raw", units, ranges, [room(*r) for r in ranges], count=count)
    assert rc == 0
    for i, (a, b) in enumerate(zip(got, want)):
        assert a == b, (i, ranges[i], a[0], b[0], len(a[1]), len(b[1]))
    return got, dec


def shared_ranges(rng, u, sp, total, hot=None, many=300):
    """Heavy sharing over one stream: many small ranges inside one chunk, more than K17_GROUP on one edge chunk (hot),
    duplicates, empty, overlapping, straddling and past-the-end ranges."""
    out = [(u, 0, 0), (u, total, 5), (u, total + 9, 1), (u, 0, total), (u, max(total - 3, 0), 10)]
    if total == 0:
        return out
    o, d = sp[len(sp) // 2]
    out += [(u, o + rng.randrange(max(d, 1)), rng.randrange(1, 300)) for _ in range(40)]    # inside one chunk
    if hot is not None:
        ho, hd = sp[hot]
        out += [(u, ho + rng.randrange(max(hd - 1, 1)), rng.randrange(1, 64)) for _ in range(many)]
    for k in range(1, len(sp)):                                          # straddling every boundary, twice
        b = sp[k][0]
        out += [(u, b - 5, 10), (u, b - 5, 10), (u, b - 1, BLOCK + 2)]
    out += [(u, rng.randrange(total), rng.randrange(1, 3 * BLOCK)) for _ in range(10)]
    return out


@pytest.fixture(autouse=True)
def _crc(oracle):
    rt._crc_oracle = oracle.crc32c_masked                                # what test_raw_table_emu.check_build checks with


def test_frame_gather_equals_range_call_and_oracle(oracle):
    """Corpus text, walked streams with empty chunks, fragments and a stream with one corrupted chunk, in one call with
    their ranges shuffled; more than K17_GROUP ranges on one edge chunk. The decode count is the cost contract."""
    rng = random.Random(1)
    streams, datas = [], []
    for k, n in enumerate((4 * BLOCK + 777, 3 * BLOCK, 1000)):
        s = oracle.frame_encode(_text(n, 20 + k))
        streams.append((s, {}))
        datas.append(oracle.frame_decode(s))
    empty = ls.chunk(0x01, b"", oracle.crc32c_masked(b""))
    g = ls.gen_frame(rng, oracle.crc32c_masked, 10)
    walked = g.stream + empty + ls.gen_frame(rng, oracle.crc32c_masked, 4).stream[10:]
    streams += [(walked, {}), (walked[10:], {"fragment": True})]
    datas += [oracle.frame_decode(walked)] * 2
    units, spans_of = [], []
    for s, kw in streams:
        src = ft.upload(s)
        rc, table, _ = ft.build(s, src=src, **kw)
        assert rc == 0
        units.append((src, table))
        spans_of.append(frame_spans(table))
    ranges = []
    for u in range(len(units)):
        sp, total = spans_of[u]
        ranges += shared_ranges(rng, u, sp, total, hot=1 if u == 0 else None)
    rng.shuffle(ranges)
    got, dec = frame_both(units, ranges)
    for (u, lo, n), (st, b) in zip(ranges, got):
        assert st == OK and b == datas[u][lo:lo + n], (u, lo, n)
    assert dec == expected_decodes(spans_of, ranges)
    # a corrupted chunk: every range that verifies it fails as the range call says, the others are served
    s = streams[0][0]
    bad = _flip(s, ft.chain(s)[2] + 40)
    src = ft.upload(bad)
    rc, table, _ = ft.build(bad, src=src)
    sp, total = frame_spans(table)
    rs = shared_ranges(rng, 0, sp, total, hot=2, many=40) + shared_ranges(rng, 1, *spans_of[0])
    got, _ = frame_both([(src, table), units[0]], rs)
    assert any(st != OK for st, _ in got)


def test_frame_n_ranges_in_one_chunk_cost_one_decode(oracle):
    s = oracle.frame_encode(_text(3 * BLOCK, 5))
    data = oracle.frame_decode(s)
    src = ft.upload(s)
    rc, table, _ = ft.build(s, src=src)
    G = glib().emu_gather_group()
    for n in (1, 7, G, G + 1):
        rng = random.Random(n)
        ranges = [(0, BLOCK + rng.randrange(BLOCK - 300), rng.randrange(1, 300)) for _ in range(n)]
        rc, got, dec = gather("frame", [(src, table)], ranges, [r[2] for r in ranges])
        assert rc == 0 and dec == (n + G - 1) // G
        assert all(g == (OK, data[lo:lo + m]) for (_, lo, m), g in zip(ranges, got))


def test_frame_tampered_tables_and_bad_units(oracle, monkeypatch):
    """Scribbled records, a short chunk table, units out of range and wrong lengths: the range call's statuses and bytes."""
    s = oracle.frame_encode(_text(6 * BLOCK + 5, 14))
    src = ft.upload(s)
    rc, table, res = ft.build(s, src=src, max_chunks=64)
    nch, total = res[2], res[1]
    rng = np.random.default_rng(6)
    scribbled = table.copy()
    recs = scribbled[ft.HEAD:ft.HEAD + nch * ft.REC].view(np.uint64).reshape(nch, 4)
    recs[:, 3] = np.sort(rng.integers(0, total + BLOCK, nch, dtype=np.uint64))
    recs[1, 0] = len(s) + 3
    rc, short, _ = ft.build(s, src=src, max_chunks=3)
    r = random.Random(7)
    ranges = [(u, r.randrange(total + 10), r.randrange(0, 2 * BLOCK)) for u in range(3) for _ in range(30)]
    ranges += [(u, lo, 100) for u in range(3) for lo in (0, BLOCK - 50, total - 20)] + [(9, 0, 5), (3, 0, 5)]
    units = [(src, table), (src, scribbled), (src, short), (src, table)]
    in_lens = [len(s)] * 3 + [len(s) + 1]
    got, _ = frame_both(units, ranges, in_lens=in_lens, overlapping=(1,))
    # the scribbled unit: records outside the build's bounds fail with c=3, the others decode and pass their CRC; the
    # gather's answer does not depend on the order of its lanes and warps
    assert {st for (u, _, _), (st, _) in zip(ranges, got) if u == 1} <= {OK} | {("Invalid", k, 0, 3) for k in range(nch)}
    monkeypatch.setenv("SBEMU_ORDER", "reverse")
    assert gather("frame", units, ranges, [n for _, _, n in ranges], in_lens=in_lens)[1] == got


def test_raw_gather_equals_range_call_and_model(oracle):
    rng = random.Random(1)
    streams = rt.gen_units(rng, oracle)
    streams += [oracle.compress(_text(5 * BLOCK + 99, 3))]
    got, ref = rt.check_build(streams)
    units = [(got.srcs[u], got.table(u)) for u in range(len(streams))]
    seek = [rt.head_of(t)[5] for _, t in units]
    ranges = []
    for u, (_, data) in enumerate(ref):
        if seek[u]:
            sp, dn = raw_spans(units[u][1])
            ranges += shared_ranges(rng, u, sp, dn, hot=1 if u == len(streams) - 1 else None)
    rng.shuffle(ranges)
    out, dec = raw_both(units, ranges)
    for (u, lo, n), (st, b) in zip(ranges, out):
        assert st == OK and b == ref[u][1][lo:lo + n], (u, lo, n)
    assert dec == expected_decodes({u: raw_spans(units[u][1]) for u in range(len(units)) if seek[u]}, ranges)


def test_raw_not_seekable_corrupted_and_tampered(oracle):
    """A stream that is not seekable, a same-length stream with a byte changed, tampered records and headers, units out
    of range and a frame table: the range call's statuses and bytes."""
    rng = random.Random(4)
    good = ls.gen_stream(rng, 5 * BLOCK + 333, "blocked", copy_share=0.3)
    bad = ls.gen_stream(rng, 150000, "unblocked")
    got, ref = rt.check_build([good.stream, bad.stream if bad.straddles else b"\x00\x00"])
    src, table = got.srcs[0], got.table(0).copy()
    e = next(x for x in good.elems if x[2] == 0 and x[6] >= 3 * BLOCK and x[6] + x[3] <= 4 * BLOCK)
    flip = bytearray(good.stream)
    flip[e[0] + e[1]] ^= 0x40
    crc = table.copy()
    crc[rt.HEAD + 8 * 2 + 4] ^= 1
    moved = table.copy()
    moved[rt.HEAD + 8 * 4:rt.HEAD + 8 * 4 + 4] = np.frombuffer(np.uint32(len(good.stream) + 1).tobytes(), dtype=np.uint8)
    head = table.copy()
    head[28:32] = np.frombuffer(np.uint32(7).tobytes(), dtype=np.uint8)
    units = [(src, table), (got.srcs[1], got.table(1)), (rt.upload(flip), table), (src, crc), (src, moved), (src, head)]
    dn = len(ref[0][1])
    sp, _ = raw_spans(table)
    ranges = []
    for u in range(len(units)):
        ranges += shared_ranges(rng, u, sp, dn, hot=3, many=20)
    ranges += [(17, 0, 4), (len(units), 5, 5)]
    rng.shuffle(ranges)
    out, _ = raw_both(units, ranges)
    assert {st[3] for st, _ in out if st != OK} >= {1, 3, 4, 5}


def test_lane_and_warp_order_do_not_change_results(oracle, monkeypatch):
    s = oracle.frame_encode(_text(3 * BLOCK + 10, 8))
    src = ft.upload(s)
    rc, table, _ = ft.build(s, src=src)
    sp, total = frame_spans(table)
    ranges = shared_ranges(random.Random(3), 0, sp, total, hot=1, many=40)
    rc, base, _ = gather("frame", [(src, table)], ranges, [n for _, _, n in ranges])
    for order in ("reverse", "shuffle"):
        monkeypatch.setenv("SBEMU_ORDER", order)
        rc, got, _ = gather("frame", [(src, table)], ranges, [n for _, _, n in ranges])
        assert rc == 0 and got == base, order


def test_scratch_bound_and_call_checks(oracle):
    L = glib()
    for f, g in ((L.emu_frame_table_gather_scratch_bytes, ft.tlib().emu_frame_table_ranges_scratch_bytes),
                 (L.emu_raw_table_gather_scratch_bytes, rt.tlib().emu_raw_table_ranges_scratch_bytes)):
        for n in (1, 4096, 1 << 20):
            assert f(n) <= 128 * n + (256 << 20) + (64 << 10), n
        assert f(1) <= g(1) + 4096
    s = oracle.frame_encode(_text(2 * BLOCK, 2))
    src = ft.upload(s)
    rc, table, _ = ft.build(s, src=src)
    ranges = [(0, 5, 10), (0, BLOCK - 3, 10)]
    for fmt in ("frame", "raw"):
        assert gather(fmt, [(src, table)], ranges, [10, 10], scratch_short=1)[0] == INVALID
        assert gather(fmt, [(src, table)], [], [])[:2] == (0, [])
    p = C.c_void_p(8)
    for fmt in ("frame", "raw"):
        fn = getattr(L, "emu_%s_table_gather" % fmt)
        big = getattr(L, "emu_%s_table_gather_scratch_bytes" % fmt)(1)
        assert fn(p, p, p, 1, p, p, p, p, p, p, (1 << 28) + 1, p, 1 << 62, None) == INVALID
        assert fn(p, p, p, 1 << 31, p, p, p, p, p, p, 1, p, big, None) == INVALID
        for i in range(10):
            a = [p] * 10                                                   # the pointers, the scratch last
            a[i] = None
            assert fn(*a[:3], 1, *a[3:9], 1, a[9], big, None) == INVALID, i
