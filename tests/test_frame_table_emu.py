"""Seek tables and ranges over many tabled streams on CPU: K5's index phase plus k13_export (the build), and the k13_*
read bodies of rust-snappy_b200/csrc/k13_frame_table.cuh (plan, pair scan, decode + CRC, finish), compiled by g++ against
the fiber warp emulator with small grids. Every range must give exactly what K12 (sb_frame_decode_ranges_device_ws,
under the emulator) gives it on the same stream with the same index, flags and max_chunks, and the oracle's bytes for
a valid stream. Nothing may be written outside a range's buffer, the staging, the scratch or the table. Test tooling
only, like tests/test_frame_range_decode_emu.py."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import emu_helpers as emu
import legal_streams as ls
from test_frame_batch_decode_emu import IDENT, _flip, _text, chain
from test_frame_range_decode_emu import OK, SEG, boundary_ranges, run_ranges, spans, status_of, verifies

INVALID = 202
GUARD = 512
BLOCK = 65536
SLOT = 65536
HEAD = 64
REC = 32

_HERE = os.path.dirname(os.path.abspath(__file__))
_EMU = os.path.join(_HERE, "emu")
_SO = os.path.join(_EMU, "_build", "libemu_frame_table.so")
_lib = None


def tlib():
    """The emulator build of K13's bodies (tests/emu/emu_frame_table.cpp), rebuilt when a source is newer."""
    global _lib
    if _lib is None:
        csrc = os.path.join(os.path.dirname(_HERE), "rust-snappy_b200", "csrc")
        srcs = [os.path.join(_EMU, f) for f in ("emu_frame_table.cpp", "simt_emu.cpp", "simt_emu.h")]
        srcs += [os.path.join(csrc, f) for f in os.listdir(csrc)]
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            tmp = "%s.%d.tmp" % (_SO, os.getpid())
            subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unused-function",
                                   "-Wno-unknown-pragmas", "-Wl,-Bsymbolic", "-o", tmp,
                                   os.path.join(_EMU, "emu_frame_table.cpp"), os.path.join(_EMU, "simt_emu.cpp")])
            os.replace(tmp, _SO)
        _lib = C.CDLL(_SO)
        for f in ("emu_frame_table_bytes", "emu_frame_table_build_scratch_bytes", "emu_frame_table_ranges_scratch_bytes"):
            getattr(_lib, f).restype = C.c_uint64
            getattr(_lib, f).argtypes = [C.c_uint32]
        _lib.emu_frame_table_build.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p,
                                               C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64]
        _lib.emu_frame_table_decode_ranges.argtypes = [C.c_void_p] * 3 + [C.c_uint32] + [C.c_void_p] * 6 + \
            [C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p]
    return _lib


def upload(stream):
    """A stream as the device would hold it: 16 bytes of slack behind it, as the K12 tests give theirs."""
    return np.frombuffer(bytes(stream) + bytes(16), dtype=np.uint8).copy()


def build(stream, fragment=False, index=None, max_chunks=None, seg=SEG, table_short=0, scratch_short=0, src=None):
    """sb_frame_table_build_device_ws under the emulator. Returns rc, the table (exactly table_bytes(max_chunks)
    bytes) and the stream's (status, bytes, nchunks); checks the guard bytes around the table and the scratch."""
    n = len(stream)
    src = upload(stream) if src is None else src
    if max_chunks is None:
        max_chunks = n // 8 + 16
    L = tlib()
    tb = L.emu_frame_table_bytes(max_chunks)
    table = np.full(tb + 2 * GUARD, 0xAB, dtype=np.uint8)
    size = L.emu_frame_table_build_scratch_bytes(max_chunks)
    scratch = np.full(size + 2 * GUARD, 0xCD, dtype=np.uint8)
    idx = np.array(list(index) + [0xCDCD], dtype=np.uint64) if index is not None else None
    res = emu.SbFrameResult()
    rc = L.emu_frame_table_build(src.ctypes.data, n, idx.ctypes.data if idx is not None else None,
                                 len(index) - 1 if index is not None else 0, 1 if fragment else 0,
                                 table.ctypes.data + GUARD, tb - table_short, max_chunks, C.byref(res),
                                 scratch.ctypes.data + GUARD, size - scratch_short, seg)
    assert (table[:GUARD] == 0xAB).all() and (table[GUARD + tb:] == 0xAB).all()
    assert (scratch[:GUARD] == 0xCD).all() and (scratch[GUARD + size:] == 0xCD).all()
    if rc:
        assert (table == 0xAB).all()
        return rc, None, None
    return 0, table[GUARD:GUARD + tb].copy(), (status_of(res.status), res.bytes, res.nchunks)


def read(units, ranges, scratch_short=0, in_lens=None):
    """sb_frame_table_decode_ranges_device_ws under the emulator. units: [(input array, table array)], ranges:
    [(unit, lo, n)]. Returns rc and [(status, bytes)]; checks the guard bytes around every range's buffer, the scratch
    (past the staging) and that the inputs and tables are unchanged."""
    L = tlib()
    count, k = len(units), len(ranges)
    before = [(bytes(i), bytes(t)) for i, t in units]
    lens = [n for _, _, n in ranges]
    offs, at = [], 3
    for ln in lens:
        offs.append(at)
        at += ln + 16 + 1 - ln % 2
    out = np.full(at + 16, 0xEE, dtype=np.uint8)
    t_tab = np.array([t.ctypes.data for _, t in units] + [0], dtype=np.uint64)
    t_in = np.array([i.ctypes.data for i, _ in units] + [0], dtype=np.uint64)
    t_n = np.array((in_lens if in_lens is not None else [len(i) - 16 for i, _ in units]) + [0], dtype=np.uint64)
    t_unit = np.array([u for u, _, _ in ranges] + [0], dtype=np.uint32)
    t_lo = np.array([lo for _, lo, _ in ranges] + [0], dtype=np.uint64)
    t_len = np.array(lens + [0], dtype=np.uint64)
    t_ptr = np.array([out.ctypes.data + o for o in offs] + [0], dtype=np.uint64)
    out_lens = np.full(k + 1, 0xDEADBEEF, dtype=np.uint64)
    st = (emu.SbError * max(k, 1))()
    size = L.emu_frame_table_ranges_scratch_bytes(k)
    scratch = np.full(size + 2 * GUARD, 0xCD, dtype=np.uint8)
    sat = C.c_uint64(0)
    rc = L.emu_frame_table_decode_ranges(t_tab.ctypes.data, t_in.ctypes.data, t_n.ctypes.data, count, t_unit.ctypes.data,
                                         t_lo.ctypes.data, t_len.ctypes.data, t_ptr.ctypes.data, out_lens.ctypes.data,
                                         C.addressof(st), k, scratch.ctypes.data + GUARD, size - scratch_short,
                                         C.byref(sat))
    assert [(bytes(i), bytes(t)) for i, t in units] == before                # inputs and tables are read-only
    assert (scratch[:GUARD] == 0xCD).all()
    if rc or k == 0:
        assert (out_lens == 0xDEADBEEF).all() and (out == 0xEE).all() and (scratch == 0xCD).all()
        return rc, [] if not rc else None
    assert (scratch[GUARD + sat.value + 2 * SLOT * k:] == 0xCD).all()      # nothing past the staging or the scratch
    assert int(out_lens[k]) == 0xDEADBEEF and (out[:3] == 0xEE).all()
    got = []
    for i, (o, ln) in enumerate(zip(offs, lens)):
        assert bytes(out[o + ln:o + ln + 16]) == b"\xee" * 16, i         # nothing written past the range's buffer
        m = int(out_lens[i])
        assert m <= ln, i
        got.append((status_of(st[i]), bytes(out[o:o + m])))
    return 0, got


def against_k12(streams, ranges):
    """Build a table per stream (streams: [(stream, kwargs)]), read all ranges in one call and compare every range
    with K12's answer on its own stream. Returns the per-range results and the builds' results."""
    units, results = [], []
    for s, kw in streams:
        src = upload(s)
        rc, table, res = build(s, src=src, **kw)
        assert rc == 0
        units.append((src, table))
        results.append(res)
    rc, got = read(units, ranges)
    assert rc == 0
    for u, (s, kw) in enumerate(streams):
        mine = [(lo, n) for v, lo, n in ranges if v == u]
        if not mine:
            continue
        k12kw = {k: v for k, v in kw.items() if k in ("fragment", "index", "max_chunks")}
        rc, want, res = run_ranges(s, mine, **k12kw)
        assert rc == 0 and res == results[u], u
        assert [g for (v, _, _), g in zip(ranges, got) if v == u] == want, u
    return got, results


def _encoded(oracle, n, seed):
    s = oracle.frame_encode(_text(n, seed))
    return s, chain(s)


def _all(u, stream, fragment=False):
    sp, total = spans(stream, fragment)
    return [(u, lo, n) for lo, n in boundary_ranges([o for o, _ in sp], total)]


@pytest.mark.parametrize("how", ["k7", "index", "walk"])
def test_encoder_output(oracle, how):
    """Encoder output tabled through K7, through the encoder's own index, and walked: the oracle's bytes, K12's answers."""
    s, ix = _encoded(oracle, 5 * BLOCK + 777, 1)
    kw = {"index": ix} if how == "index" else {"index": ix[:2] + [ix[-1]]} if how == "walk" else {}
    ranges = _all(0, s)
    got, res = against_k12([(s, kw)], ranges)
    data = oracle.frame_decode(s)
    assert all(g == (OK, data[lo:lo + n]) for (_, lo, n), g in zip(ranges, got))
    assert res[0] == (OK, len(data), len(spans(s)[0]))


def test_walked_streams_and_fragments_in_one_call(oracle):
    """Padding, skippable and empty chunks, a repeated identifier (all walked at build time) and fragments, several
    streams per call with their ranges interleaved."""
    rng = random.Random(3)
    empty = ls.chunk(0x01, b"", oracle.crc32c_masked(b"")) + ls.chunk(0x00, b"\x00", oracle.crc32c_masked(b""))
    streams, datas = [], []
    for k in range(4):
        g = ls.gen_frame(rng, oracle.crc32c_masked, 14)
        s = g.stream + empty + (IDENT if k % 2 else b"") + ls.gen_frame(rng, oracle.crc32c_masked, 5).stream[10:]
        streams.append((s, {}))
        datas.append(oracle.frame_decode(s))
        streams.append((s[10:], {"fragment": True}))
        datas.append(datas[-1])
    ranges = []
    for u, (s, kw) in enumerate(streams):
        sp, total = spans(s, kw.get("fragment", False))
        ranges += _all(u, s, kw.get("fragment", False)) + [(u, o, 0) for o, d in sp if d == 0]
    rng.shuffle(ranges)
    got, _ = against_k12(streams, ranges)
    assert all(g == (OK, datas[u][lo:lo + n]) for (u, lo, n), g in zip(ranges, got))
    s, _ = _encoded(oracle, 3 * BLOCK + 5, 4)
    frag = s[10:]
    against_k12([(frag, {"fragment": True}), (frag, {"fragment": True, "index": chain(frag, True)})],
                _all(0, frag, True) + _all(1, frag, True))


@pytest.mark.parametrize("indexed", [False, True])
def test_corrupted_chunks(oracle, indexed):
    """One and two corrupted chunks: ranges that verify one get the first failing chunk's status and the bytes before
    it, the same as K12; the clean stream beside them in the same call is unaffected."""
    clean, ix = _encoded(oracle, 4 * BLOCK + 999, 5)
    data = oracle.frame_decode(clean)
    one = _flip(clean, ix[2] + 40)
    two = _flip(_flip(clean, ix[1] + 5), ix[3] + 6)
    kw = {"index": ix} if indexed else {}
    ranges = _all(0, clean) + _all(1, clean) + _all(2, clean)
    random.Random(1).shuffle(ranges)
    got, _ = against_k12([(one, kw), (two, kw), (clean, kw)], ranges)
    sp, total = spans(clean)
    assert any(g[0] != OK for (u, _, _), g in zip(ranges, got) if u == 0)
    assert any(g[0][0] == "Checksum" for (u, _, _), g in zip(ranges, got) if u == 1)
    for (u, lo, n), g in zip(ranges, got):
        if u == 2 or (u == 0 and not verifies(sp[2][0], sp[2][1], lo, n, total)):
            assert g == (OK, data[lo:lo + n])


def test_truncated_stream_and_short_table(oracle):
    clean, ix = _encoded(oracle, 3 * BLOCK + 100, 7)
    s = clean[:-5]
    total = len(oracle.frame_decode(clean[:ix[-2]]))
    ranges = [(0, total), (0, total + 1), (total - 1, 1), (total - 1, 2), (total, 1), (total + 9, 1), (5, 10), (total, 0)]
    got, res = against_k12([(s, {}), (clean, {"max_chunks": 3}), (clean, {"max_chunks": 4})],
                           [(u, lo, n) for u in range(3) for lo, n in ranges])
    assert res[0][0][0] != "Ok" and res[1][0] == ("Invalid", 3, 1, 0) and res[2][0] == OK
    assert all(g == (("Invalid", 3, 1, 0), b"") for g in got[len(ranges):2 * len(ranges)])
    assert build(clean, index=ix, max_chunks=3)[0] == INVALID          # nchunks > max_chunks: an argument error


def test_segments_and_random_ranges_over_many_streams(oracle):
    """Streams over several K7 segments and short ones, many straddling ranges in one call, units in any order."""
    rng = random.Random(2)
    streams = []
    for k, n in enumerate((9 * BLOCK + 12345, 1, 0, 2 * BLOCK, 70000)):
        s, ix = _encoded(oracle, n, 10 + k)
        streams.append((s, {"index": ix} if k % 2 else {}))
    totals = [len(oracle.frame_decode(s)) for s, _ in streams]
    ranges = [(u, rng.randrange(totals[u] + 2), rng.randrange(0, 3 * BLOCK)) for u in (rng.randrange(5) for _ in range(60))]
    against_k12(streams, ranges)


def test_same_stream_under_two_units_and_units_out_of_range(oracle):
    s, _ = _encoded(oracle, 2 * BLOCK + 3, 9)
    data = oracle.frame_decode(s)
    src = upload(s)
    rc, table, _ = build(s, src=src)
    ranges = [(1, 5, 100), (0, 5, 100), (2, 0, 10), (7, 0, 0), (1, BLOCK - 1, 3)]
    rc, got = read([(src, table), (src, table)], ranges)
    assert rc == 0
    assert got[0] == got[1] == (OK, data[5:105]) and got[4] == (OK, data[BLOCK - 1:BLOCK + 2])
    assert got[2] == (("Invalid", 2, 2, 1), b"") and got[3] == (("Invalid", 7, 2, 1), b"")
    rc, got = read([], [(0, 0, 5)])                                        # no streams at all: every unit is out of range
    assert rc == 0 and got == [(("Invalid", 0, 0, 1), b"")]


def test_table_cut_to_its_chunks_and_moved(oracle):
    s, _ = _encoded(oracle, 4 * BLOCK + 17, 12)
    data = oracle.frame_decode(s)
    src = upload(s)
    rc, table, res = build(s, src=src, max_chunks=1000)
    assert rc == 0 and res == (OK, len(data), 5)
    exact = tlib().emu_frame_table_bytes(res[2])
    assert exact == HEAD + 5 * REC
    moved = np.frombuffer(bytes(7) + table[:exact].tobytes(), dtype=np.uint8).copy()
    moved = np.frombuffer(moved[7:].tobytes(), dtype=np.uint8).copy()        # a fresh buffer holding just the table
    sp, total = spans(s)
    ranges = _all(0, s) + _all(1, s)
    rc, got = read([(src, table), (src, moved)], ranges)
    assert rc == 0 and all(g == (OK, data[lo:lo + n]) for (_, lo, n), g in zip(ranges, got))


def test_header_mismatches(oracle):
    """A table read with another stream length, a wrong magic and an empty buffer give status 2; the other units of
    the call are unaffected."""
    s, _ = _encoded(oracle, BLOCK + 100, 13)
    data = oracle.frame_decode(s)
    src = upload(s)
    rc, table, _ = build(s, src=src)
    bad = table.copy()
    bad[0] ^= 1
    zero = np.zeros(HEAD, dtype=np.uint8)
    n = len(s)
    units = [(src, table), (src, table), (src, bad), (src, zero)]
    rc, got = read(units, [(0, 0, 10), (1, 0, 10), (2, 0, 10), (3, 0, 10), (1, 5, 0)], in_lens=[n, n + 1, n, n])
    assert got[0] == (OK, data[:10])
    assert got[1] == (("Invalid", n + 1, n, 2), b"") and got[4] == got[1]
    assert got[2] == (("Invalid", n, 0, 2), b"") and got[3] == (("Invalid", n, 0, 2), b"")
    other = _flip(s, chain(s)[1] + 30)                                     # other bytes of the same length
    assert len(other) == n
    rc, got = read([(upload(other), table)], [(0, 0, 2 * BLOCK)])
    assert got[0][0][0] != "Ok" and got[0][1] == data[:BLOCK]          # the first chunk still checks out


def test_decodable_record_claimed_past_total(oracle):
    """A record that still decodes and passes its CRC, moved to just below total (the offsets stay sorted): a range that
    starts past total finds it verified, and it must fail as its chunk (Invalid{k, 0, 3}, no bytes) instead of giving
    a slice of negative length. A range inside the stream that reaches it stays within its buffer."""
    s, _ = _encoded(oracle, 2 * BLOCK + 777, 15)
    src = upload(s)
    rc, table, res = build(s, src=src, max_chunks=16)
    assert rc == 0 and res[2] == 3
    total = res[1]
    recs = table[HEAD:HEAD + 3 * REC].view(np.uint64).reshape(3, 4)
    assert int(recs[2, 3]) == 2 * BLOCK
    recs[2, 3] = total - 10
    rc, got = read([(src, table)], [(0, total + 5, 10), (0, total + 5, 0), (0, total - 20, 100), (0, 0, 10)])
    assert rc == 0
    assert got[0] == (("Invalid", 2, 0, 3), b"") and got[1] == got[0]
    assert got[2][0] == OK and len(got[2][1]) == 20
    assert got[3] == (OK, oracle.frame_decode(s)[:10])


@pytest.mark.parametrize("how", ["bytes", "fields"])
def test_scribbled_records_stay_inside_their_buffers(oracle, how):
    """Records overwritten with random bytes, or with random but plausible field values: every range ends with some
    status, and nothing is read or written outside the stream, the ranges' buffers, the staging or the scratch (the
    guard bytes of read() and the unchanged inputs)."""
    rng = np.random.default_rng(5 if how == "bytes" else 6)
    s, _ = _encoded(oracle, 6 * BLOCK + 5, 14)
    src = upload(s)
    rc, table, res = build(s, src=src, max_chunks=64)
    nch, total = res[2], res[1]
    recs = table[HEAD:HEAD + nch * REC].view(np.uint64).reshape(nch, 4).copy()
    if how == "bytes":
        recs[:] = rng.integers(0, 1 << 63, recs.shape, dtype=np.uint64) * 2 + 1
    else:
        body = rng.integers(0, len(s) + 100, nch, dtype=np.uint64)
        blen = rng.integers(0, 80000, nch, dtype=np.uint64)
        dlen = rng.integers(0, 70000, nch, dtype=np.uint64)
        crc = rng.integers(0, 1 << 32, nch, dtype=np.uint64)
        ty = rng.integers(0, 3, nch, dtype=np.uint64)
        off = np.sort(rng.integers(0, total + BLOCK, nch, dtype=np.uint64))
        recs[:, 0], recs[:, 1], recs[:, 2], recs[:, 3] = body, blen | (dlen << 32), crc | (ty << 32), off
        recs[::3, 1] = recs[::3, 1] & 0xFFFFFFFF | ((recs[::3, 1] & 0xFFFFFFFF) << 32)   # stored bodies as long as output
        recs[::3, 2] = recs[::3, 2] & 0xFFFFFFFF | (1 << 32)
    table[HEAD:HEAD + nch * REC] = recs.reshape(-1).view(np.uint8)
    r = random.Random(7)
    ranges = [(0, r.randrange(total + 10), r.randrange(0, 2 * BLOCK)) for _ in range(40)] + [(0, 0, total)]
    rc, got = read([(src, table)], ranges)
    assert rc == 0
    codes = [g[0] for g in got]
    if how == "fields":                                                    # offsets in range: records are used and refused
        assert any(c[0] == "Invalid" and c[3] == 3 for c in codes)
    for (_, lo, n), (stt, b) in zip(ranges, got):
        assert len(b) <= n


def test_no_ranges_and_call_checks(oracle):
    L = tlib()
    assert L.emu_frame_table_bytes(0) == HEAD and L.emu_frame_table_bytes(7) == HEAD + 7 * REC
    f = L.emu_frame_table_ranges_scratch_bytes
    assert f(0) < f(1) < f(2) and f(2) - f(1) >= 2 * SLOT
    g = L.emu_frame_table_build_scratch_bytes
    assert g(10) < g(1000) < g(100000)
    s, ix = _encoded(oracle, BLOCK + 1, 11)
    assert build(s, table_short=1)[0] == INVALID and build(s, scratch_short=1)[0] == INVALID
    assert build(s, max_chunks=0)[0] == INVALID and build(s, max_chunks=(1 << 22) - 1)[0] == INVALID
    assert build(s, index=ix, max_chunks=1)[0] == INVALID
    assert build(s, max_chunks=(1 << 22) - 2)[0] == 0
    src = upload(s)
    rc, table, _ = build(s, src=src)
    assert read([(src, table)], [])[0] == 0
    assert read([(src, table)], [(0, 0, 5)], scratch_short=1)[0] == INVALID
    buf = np.zeros(1 << 20, dtype=np.uint8)
    p = buf.ctypes.data
    sat = C.c_uint64(0)
    res = emu.SbFrameResult()

    def call(count=1, nr=1, arrays=(p,) * 10):
        return L.emu_frame_table_decode_ranges(*arrays[:3], count, *arrays[3:9], nr, arrays[9], 1 << 20, C.byref(sat))
    for k in range(10):                                                    # one of the needed pointers missing
        assert call(arrays=tuple(None if m == k else p for m in range(10))) == INVALID
    for k in range(3):                                                     # no streams: their arrays are not needed
        assert call(count=0, arrays=tuple(None if m == k else p for m in range(10))) == 0
    assert call(count=1 << 31) == INVALID and call(nr=1 << 31) == INVALID
    assert call(nr=0, arrays=(None,) * 10) == 0
    t = np.zeros(1 << 16, dtype=np.uint8)
    args = [src.ctypes.data, len(s), None, 0, 0, t.ctypes.data, 1 << 16, 64, C.byref(res), buf.ctypes.data, 1 << 20, 0]
    assert L.emu_frame_table_build(*args) == 0
    for m in (0, 5, 8, 9):                                                 # the build's pointers: input, table, result, scratch
        bad = list(args)
        bad[m] = None
        assert L.emu_frame_table_build(*bad) == INVALID
