"""Host-stream gathers on CPU: the HOST instantiations of the K13, K15 and K17 decode bodies
(rust-snappy_b200/csrc/k18_host_gather.cuh) compiled by g++ against the fiber warp emulator with small grids and 4
decoding warps. Every range must get exactly what the device gather (tests/test_table_gather_emu.py's harness) gives it,
and the oracle's bytes where Ok; nothing may be written outside a range's buffer or the scratch; and the call must copy
into its slots exactly the bodies it decodes, once per decode, except a raw block too large for a slot, which decodes in
place. Test tooling only."""
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
import test_table_gather_emu as tg
from test_frame_batch_decode_emu import _flip, _text

INVALID = 202
GUARD = 512
BLOCK = 65536
OK = ("Ok", 0, 0, 0)

_HERE = os.path.dirname(os.path.abspath(__file__))
_EMU = os.path.join(_HERE, "emu")
_SO = os.path.join(_EMU, "_build", "libemu_table_gather_host.so")
_lib = None


def hlib():
    """The emulator build of the host gathers (tests/emu/emu_table_gather_host.cpp), rebuilt when a source is newer."""
    global _lib
    if _lib is None:
        csrc = os.path.join(os.path.dirname(_HERE), "rust-snappy_b200", "csrc")
        srcs = [os.path.join(_EMU, f) for f in ("emu_table_gather_host.cpp", "simt_emu.cpp", "simt_emu.h")]
        srcs += [os.path.join(csrc, f) for f in os.listdir(csrc)]
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            tmp = "%s.%d.tmp" % (_SO, os.getpid())
            subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unused-function",
                                   "-Wno-unknown-pragmas", "-Wl,-Bsymbolic", "-o", tmp,
                                   os.path.join(_EMU, "emu_table_gather_host.cpp"), os.path.join(_EMU, "simt_emu.cpp")])
            os.replace(tmp, _SO)
        _lib = C.CDLL(_SO)
        for f in ("emu_frame_table_gather_host_scratch_bytes", "emu_raw_table_gather_host_scratch_bytes"):
            getattr(_lib, f).restype = C.c_uint64
            getattr(_lib, f).argtypes = [C.c_uint32]
        _lib.emu_cslot_bytes.restype = C.c_uint64
        for f in ("emu_frame_table_gather_host", "emu_raw_table_gather_host"):
            getattr(_lib, f).argtypes = [C.c_void_p] * 3 + [C.c_uint32] + [C.c_void_p] * 6 + \
                [C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p]
    return _lib


def host_gather(fmt, units, ranges, rooms, scratch_short=0, in_lens=None, count=None):
    """sb_{fmt}_table_gather_host_streams_ws under the emulator, as tg.gather calls the device gather. Returns rc,
    [(status, bytes)], the decode count and the bytes fetched into slots."""
    L = hlib()
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
    size = getattr(L, "emu_%s_table_gather_host_scratch_bytes" % fmt)(k)
    scratch = np.full(size + 2 * GUARD, 0xCD, dtype=np.uint8)
    dec, fetched = C.c_uint64(0xFFFF), C.c_uint64(0xFFFF)
    rc = getattr(L, "emu_%s_table_gather_host" % fmt)(t_tab.ctypes.data, t_in.ctypes.data, t_n.ctypes.data, count,
                                                       t_unit.ctypes.data, t_lo.ctypes.data, t_len.ctypes.data,
                                                       t_ptr.ctypes.data, out_lens.ctypes.data, C.addressof(st), k,
                                                       scratch.ctypes.data + GUARD, size - scratch_short, C.byref(dec),
                                                       C.byref(fetched))
    assert [(bytes(i), bytes(t)) for i, t in units] == before
    assert (scratch[:GUARD] == 0xCD).all() and (scratch[GUARD + size:] == 0xCD).all()
    if rc or k == 0:
        assert (out_lens == 0xDEADBEEF).all() and all((o == 0xEE).all() for o in outs) and (scratch == 0xCD).all()
        return rc, None if rc else [], 0, 0
    assert int(out_lens[k]) == 0xDEADBEEF
    got = []
    for i, (o, r) in enumerate(zip(outs, rooms)):
        assert (o[:GUARD] == 0xEE).all() and (o[GUARD + r:] == 0xEE).all(), i
        m = int(out_lens[i])
        assert m <= r, i
        got.append(((ft.status_of if fmt == "frame" else rt.status_of)(st[i]), o[GUARD:GUARD + m].tobytes()))
    return 0, got, dec.value, fetched.value


def frame_bodies(src, table):
    """Per record of a frame table: its body length (every frame body fits a slot)."""
    w = np.frombuffer(table[:ft.HEAD].tobytes(), dtype=np.uint64)
    nch = int(w[3]) & 0xFFFFFFFF
    recs = np.frombuffer(table[ft.HEAD:ft.HEAD + nch * ft.REC].tobytes(), dtype=np.uint64).reshape(nch, 4)
    return [int(r[1]) & 0xFFFFFFFF for r in recs]


def raw_bodies(src, table):
    """Per block of a raw table: its compressed bytes, or 0 when they do not fit a slot (decoded in place)."""
    h = rt.head_of(table)
    offs = np.frombuffer(table[rt.HEAD:rt.HEAD + 8 * h[4]].tobytes(), dtype=np.uint32).reshape(-1, 2)[:, 0]
    ends = list(offs[1:]) + [h[1]]
    cslot = hlib().emu_cslot_bytes()
    out = []
    for a, b in zip(offs, ends):
        n = int(b) - int(a)
        out.append(n if (src.ctypes.data + int(a)) % 16 + n <= cslot else 0)
    return out


def expected_fetch(spans_of, bodies_of, ranges):
    """The bytes fetched for valid tables: each edge's body once per work item of at most K17_GROUP ranges, each
    interior pair's body once (tg.expected_decodes, weighted by body length)."""
    G = tg.glib().emu_gather_group()
    edges, total = {}, 0
    for u, lo, n in ranges:
        sp, size = spans_of[u]
        end = min(lo + n, size)
        run = [k for k, (o, d) in enumerate(sp) if o < end and o + max(d, 1) > lo]
        for k in run:
            o, d = sp[k]
            if o >= lo and o + d <= end:
                total += bodies_of[u][k]
            elif k in (run[0], run[-1]):
                edges[(u, k)] = edges.get((u, k), 0) + 1
    return total + sum((c + G - 1) // G * bodies_of[u][k] for (u, k), c in edges.items())


def both(fmt, units, ranges, rooms, **kw):
    """The device gather and the host gather over the same inputs: identical results. Returns them, the host call's
    decode count and its fetched bytes."""
    rc, want, dec_d = tg.gather(fmt, units, ranges, rooms, **kw)
    assert rc == 0
    rc, got, dec, fetched = host_gather(fmt, units, ranges, rooms, **kw)
    assert rc == 0
    for i, (a, b) in enumerate(zip(got, want)):
        assert a == b, (i, ranges[i], a[0], b[0], len(a[1]), len(b[1]))
    assert dec == dec_d
    return got, dec, fetched


def shifted(src, by):
    """The same stream bytes at another address alignment (a view `by` bytes into a larger array)."""
    a = np.zeros(src.size + by, dtype=np.uint8)
    a[by:] = src
    return a[by:]


@pytest.fixture(autouse=True)
def _crc(oracle):
    rt._crc_oracle = oracle.crc32c_masked


def test_frame_host_equals_device_and_oracle(oracle):
    """Corpus text, walked streams with empty chunks and fragments, at four address alignments, ranges shuffled; more
    than K17_GROUP ranges on one edge chunk. Fetched bytes are the cost contract."""
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
    units, spans_of, bodies_of = [], [], []
    for j, (s, kw) in enumerate(streams):
        src = ft.upload(s)
        rc, table, _ = ft.build(s, src=src, **kw)
        assert rc == 0
        src = shifted(src, (0, 3, 8, 13, 1)[j])
        units.append((src, table))
        spans_of.append(tg.frame_spans(table))
        bodies_of.append(frame_bodies(src, table))
    ranges = []
    for u in range(len(units)):
        sp, total = spans_of[u]
        ranges += tg.shared_ranges(rng, u, sp, total, hot=1 if u == 0 else None)
    rng.shuffle(ranges)
    got, dec, fetched = both("frame", units, ranges, [n for _, _, n in ranges])
    for (u, lo, n), (st, b) in zip(ranges, got):
        assert st == OK and b == datas[u][lo:lo + n], (u, lo, n)
    assert dec == tg.expected_decodes(spans_of, ranges)
    assert fetched == expected_fetch(spans_of, bodies_of, ranges)
    # a corrupted chunk: every range that verifies it fails as the device gather says
    s = streams[0][0]
    bad = _flip(s, ft.chain(s)[2] + 40)
    src = ft.upload(bad)
    rc, table, _ = ft.build(bad, src=src)
    sp, total = tg.frame_spans(table)
    rs = tg.shared_ranges(rng, 0, sp, total, hot=2, many=40) + tg.shared_ranges(rng, 1, *spans_of[0])
    got, _, _ = both("frame", [(src, table), units[0]], rs, [n for _, _, n in rs])
    assert any(st != OK for st, _ in got)


def test_frame_tampered_tables_and_bad_units(oracle):
    """Scribbled records, a short chunk table, units out of range and wrong lengths: the device gather's statuses and
    bytes, under two lane orders."""
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
    got, _, _ = both("frame", units, ranges, [n for _, _, n in ranges], in_lens=in_lens)
    assert {st[0] for st, _ in got} >= {"Ok", "Invalid"}


def test_raw_host_equals_device_and_model(oracle):
    rng = random.Random(1)
    streams = rt.gen_units(rng, oracle)
    streams += [oracle.compress(_text(5 * BLOCK + 99, 3))]
    built, ref = rt.check_build(streams)
    units = [(shifted(built.srcs[u], u % 16), built.table(u)) for u in range(len(streams))]
    seek = [rt.head_of(t)[5] for _, t in units]
    ranges = []
    for u, (_, data) in enumerate(ref):
        if seek[u]:
            sp, dn = tg.raw_spans(units[u][1])
            ranges += tg.shared_ranges(rng, u, sp, dn, hot=1 if u == len(streams) - 1 else None)
    rng.shuffle(ranges)
    rooms = [max(0, min(n, rt.head_of(units[u][1])[2] - lo)) for u, lo, n in ranges]
    out, dec, fetched = both("raw", units, ranges, rooms)
    for (u, lo, n), (st, b) in zip(ranges, out):
        assert st == OK and b == ref[u][1][lo:lo + n], (u, lo, n)
    spans = {u: tg.raw_spans(units[u][1]) for u in range(len(units)) if seek[u]}
    bodies = {u: raw_bodies(units[u][0], units[u][1]) for u in spans}
    assert dec == tg.expected_decodes(spans, ranges)
    assert fetched == expected_fetch(spans, bodies, ranges)


def test_raw_not_seekable_corrupted_and_tampered(oracle):
    """A stream that is not seekable, a same-length stream with a byte changed, tampered records and headers and units
    out of range: the device gather's statuses and bytes."""
    rng = random.Random(4)
    good = ls.gen_stream(rng, 5 * BLOCK + 333, "blocked", copy_share=0.3)
    bad = ls.gen_stream(rng, 150000, "unblocked")
    built, ref = rt.check_build([good.stream, bad.stream if bad.straddles else b"\x00\x00"])
    src, table = built.srcs[0], built.table(0).copy()
    e = next(x for x in good.elems if x[2] == 0 and x[6] >= 3 * BLOCK and x[6] + x[3] <= 4 * BLOCK)
    flip = bytearray(good.stream)
    flip[e[0] + e[1]] ^= 0x40
    crc = table.copy()
    crc[rt.HEAD + 8 * 2 + 4] ^= 1
    moved = table.copy()
    moved[rt.HEAD + 8 * 4:rt.HEAD + 8 * 4 + 4] = np.frombuffer(np.uint32(len(good.stream) + 1).tobytes(), dtype=np.uint8)
    head = table.copy()
    head[28:32] = np.frombuffer(np.uint32(7).tobytes(), dtype=np.uint8)
    units = [(src, table), (built.srcs[1], built.table(1)), (rt.upload(flip), table), (src, crc), (src, moved),
             (src, head)]
    dn = len(ref[0][1])
    sp, _ = tg.raw_spans(table)
    ranges = []
    for u in range(len(units)):
        ranges += tg.shared_ranges(rng, u, sp, dn, hot=3, many=20)
    ranges += [(17, 0, 4), (len(units), 5, 5)]
    rng.shuffle(ranges)

    def room(u, lo, n):
        if u >= len(units):
            return 0
        return max(0, min(n, rt.head_of(units[u][1])[2] - lo))
    out, _, _ = both("raw", units, ranges, [room(*r) for r in ranges])
    assert {st[3] for st, _ in out if st != OK} >= {1, 3, 4, 5}


def oversized_raw(oracle):
    """A legal two-block raw stream whose first block spends 5 bytes per output byte: one literal byte, then 65,535
    one-byte copy-4 elements, 327,677 compressed bytes; then a block of text. Returns (stream, its seek table, data)."""
    tail = _text(BLOCK // 2 + 17, 9)
    data = b"a" * BLOCK + tail
    hdr = ls.varint(len(data))
    body0 = ls.literal_header(1, "lit1") + b"a" + ls.copy_elem(1, 1, "copy4") * (BLOCK - 1)
    body1 = ls.literal_header(len(tail), ls.lit_forms(len(tail))[0]) + tail
    stream = hdr + body0 + body1
    assert len(body0) == 5 * BLOCK - 3
    head = np.array([rt.MAGIC, len(stream), len(data), len(hdr) | (2 << 32), 1, 0, 0, 0], dtype=np.uint64)
    recs = np.array([len(hdr), oracle.crc32c_masked(data[:BLOCK]), len(hdr) + len(body0),
                     oracle.crc32c_masked(data[BLOCK:])], dtype=np.uint32)
    return stream, np.concatenate([head.view(np.uint8), recs.view(np.uint8)]), data


def test_raw_oversized_block_decodes_in_place(oracle):
    stream, table, data = oversized_raw(oracle)
    assert rt.model(stream)[1] == data
    src = rt.upload(stream)
    ranges = [(0, 5, 10), (0, BLOCK - 7, 20), (0, 0, len(data)), (0, BLOCK + 3, 100), (0, 0, BLOCK)]
    rooms = [min(n, len(data) - lo) for _, lo, n in ranges]
    got, dec, fetched = both("raw", [(src, table)], ranges, rooms)
    assert all(g == (OK, data[lo:lo + n]) for (_, lo, n), g in zip(ranges, got))
    bodies = raw_bodies(src, table)
    assert bodies[0] == 0 and bodies[1] > 0
    assert fetched == expected_fetch({0: tg.raw_spans(table)}, {0: bodies}, ranges)


def test_lane_and_warp_order_do_not_change_results(oracle, monkeypatch):
    s = oracle.frame_encode(_text(3 * BLOCK + 10, 8))
    src = ft.upload(s)
    rc, table, _ = ft.build(s, src=src)
    sp, total = tg.frame_spans(table)
    ranges = tg.shared_ranges(random.Random(3), 0, sp, total, hot=1, many=40)
    stream, rtable, _ = oversized_raw(oracle)
    units = [(shifted(src, 5), table), (rt.upload(stream), rtable)]
    rranges = [(1, 9, 70000), (1, BLOCK - 1, 2), (1, 100, 5)]
    base = (host_gather("frame", units[:1], ranges, [n for _, _, n in ranges]),
            host_gather("raw", units[1:], [(0, lo, n) for _, lo, n in rranges], [n for _, _, n in rranges]))
    for order in ("reverse", "shuffle"):
        monkeypatch.setenv("SBEMU_ORDER", order)
        got = (host_gather("frame", units[:1], ranges, [n for _, _, n in ranges]),
               host_gather("raw", units[1:], [(0, lo, n) for _, lo, n in rranges], [n for _, _, n in rranges]))
        assert got == base, order


def test_scratch_formula_and_call_checks(oracle):
    L, D = hlib(), tg.glib()
    cslot = L.emu_cslot_bytes()
    assert cslot == (76490 + 255) // 256 * 256 == 76544
    for fmt in ("frame", "raw"):
        for n in (1, 7, 2048, 4096, 1 << 20):
            host = getattr(L, "emu_%s_table_gather_host_scratch_bytes" % fmt)(n)
            dev = getattr(D, "emu_%s_table_gather_scratch_bytes" % fmt)(n)
            assert host == dev + min(2 * n, 4096) * cslot, (fmt, n)
            assert host <= 128 * n + 4096 * (65536 + cslot) + (64 << 10), (fmt, n)
    s = oracle.frame_encode(_text(2 * BLOCK, 2))
    src = ft.upload(s)
    rc, table, _ = ft.build(s, src=src)
    ranges = [(0, 5, 10), (0, BLOCK - 3, 10)]
    for fmt in ("frame", "raw"):
        assert host_gather(fmt, [(src, table)], ranges, [10, 10], scratch_short=1)[0] == INVALID
        assert host_gather(fmt, [(src, table)], [], [])[:2] == (0, [])
    p = C.c_void_p(8)
    for fmt in ("frame", "raw"):
        fn = getattr(L, "emu_%s_table_gather_host" % fmt)
        big = getattr(L, "emu_%s_table_gather_host_scratch_bytes" % fmt)(1)
        assert fn(p, p, p, 1, p, p, p, p, p, p, (1 << 28) + 1, p, 1 << 62, None, None) == INVALID
        assert fn(p, p, p, 1 << 31, p, p, p, p, p, p, 1, p, big, None, None) == INVALID
        for i in range(10):
            a = [p] * 10                                                   # the pointers, the scratch last
            a[i] = None
            assert fn(*a[:3], 1, *a[3:9], 1, a[9], big, None, None) == INVALID, i
