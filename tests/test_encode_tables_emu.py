"""Tabled batch encodes on CPU: K9's or K10's bodies around the K1 body with its CRC array, then the k16_* bodies of
rust-snappy_b200/csrc/k16_encode_tables.cuh, compiled by g++ against the fiber warp emulator with small grids. Every
unit's output must equal the untabled harness's (tests/emu/emu_raw_batch_compress.cpp, emu_frame_batch_encode.cpp);
every unit's table, offset and result must be byte-identical to the batch builds over those outputs
(tests/emu/emu_raw_table.cpp, emu_frame_table_batch.cpp); reads over the encoder's tables must equal slices of the
input; and nothing may be written past the tables, the offsets, the results or the scratch. Test tooling only, like
tests/test_raw_table_emu.py."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import emu_helpers as emu
import test_frame_batch_encode_emu as fenc
import test_frame_table_batch_emu as fbuild
import test_frame_table_emu as fread
import test_raw_batch_compress_emu as renc
import test_raw_table_emu as rtab
from conftest import corpus

BLOCK = 65536
INVALID = 202
GUARD = 512
HEAD = 64

_HERE = os.path.dirname(os.path.abspath(__file__))
_EMU = os.path.join(_HERE, "emu")
_SO = os.path.join(_EMU, "_build", "libemu_encode_tables.so")
_lib = None


def elib():
    """The emulator build of the tabled encodes (tests/emu/emu_encode_tables.cpp), rebuilt when a source is newer."""
    global _lib
    if _lib is None:
        csrc = os.path.join(os.path.dirname(_HERE), "rust-snappy_b200", "csrc")
        srcs = [os.path.join(_EMU, f) for f in ("emu_encode_tables.cpp", "simt_emu.cpp", "simt_emu.h")]
        srcs += [os.path.join(csrc, f) for f in os.listdir(csrc)]
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            tmp = "%s.%d.tmp" % (_SO, os.getpid())
            subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unused-function",
                                   "-Wno-unknown-pragmas", "-Wl,-Bsymbolic", "-o", tmp,
                                   os.path.join(_EMU, "emu_encode_tables.cpp"), os.path.join(_EMU, "simt_emu.cpp")])
            os.replace(tmp, _SO)
        _lib = C.CDLL(_SO)
        for name in ("emu_compress_tables_bytes", "emu_frame_encode_tables_bytes"):
            getattr(_lib, name).restype = C.c_uint64
            getattr(_lib, name).argtypes = [C.c_uint32, C.c_uint64]
        _lib.emu_encode_tabled_scratch_bytes.restype = C.c_uint64
        _lib.emu_encode_tabled_scratch_bytes.argtypes = [C.c_int, C.c_uint32, C.c_uint64]
    return _lib


def tables_bytes(frame, count, in_bytes):
    """The documented bound: 64 per unit plus a record (8 raw, 32 frame) per single-block unit or K9 slot."""
    units = in_bytes // (BLOCK + 1)
    slots = in_bytes // BLOCK + min(units, count)
    return 64 * count + (32 if frame else 8) * (count + slots)


def run(frame, units, addressing="ptrs", in_bytes=None, index=False, tables_short=0, scratch_short=0):
    """The tabled call under the emulator, addressed as the untabled harnesses address it (odd addresses, or bases with
    odd strides). Returns rc and ([(status, bytes or None, index entries or None)], [table bytes], [result bytes]);
    checks every guard."""
    mod = fenc if frame else renc
    n = len(units)
    if in_bytes is None:
        in_bytes = mod.multi_bytes(units)
    if addressing == "ptrs":
        ioffs, at = [], 1
        for u in units:
            ioffs.append(at)
            at += len(u.data) + 3 + (at + len(u.data)) % 2
        ooffs, oat = [], 3
        for u in units:
            ooffs.append(oat)
            oat += u.room + 16 + 1 - (u.room % 2)
        inbuf = np.zeros(at + 16, dtype=np.uint8)
    else:
        in_stride = max([len(u.data) for u in units] + [1]) | 1
        out_stride = (max([u.room for u in units] + [1]) + 16) | 1
        ioffs = [1 + i * in_stride for i in range(n)]
        ooffs = [3 + i * out_stride for i in range(n)]
        inbuf = np.zeros(1 + n * in_stride + 16, dtype=np.uint8)
        oat = 3 + n * out_stride
    for o, u in zip(ioffs, units):
        inbuf[o:o + len(u.data)] = np.frombuffer(u.data, dtype=np.uint8)
    out = np.full(oat + 16, 0xEE, dtype=np.uint8)
    lens = np.array([u.n for u in units] + [0], dtype=np.uint32)
    caps = np.array([u.cap for u in units] + [0], dtype=np.uint32)
    in_ptrs = np.array([inbuf.ctypes.data + o for o in ioffs] + [0], dtype=np.uint64)
    out_ptrs = np.array([out.ctypes.data + o for o in ooffs] + [0], dtype=np.uint64)
    out_lens = np.full(n + 1, 0xDEADBEEF, dtype=np.uint32)
    ibase, at = [], 0
    for u in units:
        ibase.append(at)
        at += fenc.chunks(u.n) + 1
    idx = np.full(at + 4, fenc.IDX_FILL, dtype=np.uint64)
    st = (emu.SbError * max(n, 1))()
    b = emu.SbBatch()
    if addressing == "ptrs":
        b.in_ptrs, b.out_ptrs = in_ptrs.ctypes.data, out_ptrs.ctypes.data
    else:
        b.in_base, b.in_stride = inbuf.ctypes.data + 1, in_stride
        b.out_base, b.out_stride = out.ctypes.data + 3, out_stride
    b.in_lens, b.out_caps = lens.ctypes.data, caps.ctypes.data
    b.out_lens, b.statuses, b.count = out_lens.ctypes.data, C.addressof(st), n
    L = elib()
    tb = (L.emu_frame_encode_tables_bytes if frame else L.emu_compress_tables_bytes)(n, in_bytes)
    tabs = np.full(tb + GUARD, 0xAB, dtype=np.uint8)
    offs = np.full(n + 2, 0xDEADBEEF, dtype=np.uint64)
    res = (emu.SbFrameResult * (n + 1))()
    C.memset(res, 0xA5, C.sizeof(res))
    size = L.emu_encode_tabled_scratch_bytes(1 if frame else 0, n, in_bytes)
    scratch = np.full(size + 2 * GUARD, 0xCD, dtype=np.uint8)
    rc = L.emu_encode_tabled(1 if frame else 0, C.byref(b), C.c_uint64(in_bytes),
                             C.c_void_p(idx.ctypes.data if index else None), C.c_void_p(tabs.ctypes.data),
                             C.c_uint64(tb - tables_short), C.c_void_p(offs.ctypes.data), C.c_void_p(C.addressof(res)),
                             C.c_void_p(scratch.ctypes.data + GUARD), C.c_uint64(size - scratch_short))
    assert (scratch[:GUARD] == 0xCD).all() and (scratch[GUARD + size:] == 0xCD).all()
    if rc or n == 0:
        assert (out_lens == 0xDEADBEEF).all() and (out == 0xEE).all() and (idx == fenc.IDX_FILL).all()
        assert (tabs == 0xAB).all() and (offs == 0xDEADBEEF).all() and bytes(res) == b"\xa5" * C.sizeof(res)
        return rc, None
    assert tb == tables_bytes(frame, n, in_bytes)
    assert int(out_lens[n]) == 0xDEADBEEF and int(offs[n + 1]) == 0xDEADBEEF
    assert bytes(res)[n * C.sizeof(emu.SbFrameResult):] == b"\xa5" * C.sizeof(emu.SbFrameResult)
    assert int(offs[0]) == 0 and int(offs[n]) <= tb and (tabs[int(offs[n]):] == 0xAB).all()
    assert (idx[len(idx) - 4:] == fenc.IDX_FILL).all()
    if not index:
        assert (idx == fenc.IDX_FILL).all()
    outs, tables, results = [], [], []
    for i, u in enumerate(units):
        e, o, k = st[i], ooffs[i], int(out_lens[i])
        assert bytes(out[o + u.room:o + u.room + 16]) == b"\xee" * 16, i
        status = (emu.ERR.get(e.code, str(e.code)), e.a, e.b)
        ix = [int(x) for x in idx[ibase[i]:ibase[i] + fenc.chunks(u.n) + 1]]
        if e.code:
            assert k == 0 and (out[o:o + u.room] == 0xEE).all(), i
            outs.append((status, None, None))
        else:
            outs.append((status, bytes(out[o:o + k]), ix if index else None))
        tables.append(tabs[int(offs[i]):int(offs[i + 1])].tobytes())
        results.append(bytes(res[i]))
    return 0, (outs, tables, results)


def check(frame, units, **kw):
    """The tabled call against the untabled harness and the batch build over its outputs. Returns the tabled outputs and
    tables."""
    mod = fenc if frame else renc
    rc, got = run(frame, units, **kw)
    assert rc == 0
    outs, tables, results = got
    ukw = {k: v for k, v in kw.items() if k in ("addressing", "in_bytes")}
    if frame:
        ukw["index"] = kw.get("index", False)
    rc, want = mod.run_batch(units, **ukw)
    assert rc == 0
    assert (outs if frame else [o[:2] for o in outs]) == want
    streams = [o[1] or b"" for o in outs]
    if frame:
        rc, built = fbuild.run(streams)
    else:
        rc, built = rtab.build(streams)
    assert rc == 0
    for i, s in enumerate(streams):
        assert tables[i] == built.table(i).tobytes(), (i, len(s), units[i].n)
        assert results[i] == bytes(built.res[i]), (i, built.result(i))
    return streams, tables


def raw_units(rng):
    U = renc.Unit
    units = [U(renc._text(n, i)) for i, n in enumerate((0, 1, BLOCK - 1, BLOCK, BLOCK + 1))]
    units += [U(renc._text(3 * BLOCK, 4)), U(renc._text(2 * BLOCK + 1, 5)), U(renc._text(2 * BLOCK + BLOCK - 1, 6))]
    units += [U(bytes(2 * BLOCK + 17)), U(renc._random(2 * BLOCK + 999, 1)), U(renc._random(700, 2))]
    units += [U(corpus("alice29.txt")), U(corpus("fireworks.jpeg"))]
    units += [U(renc._text(2 * BLOCK + 3, 9), cap=renc.max_compress_len(2 * BLOCK + 3) - 1),
              U(renc._text(100, 9), cap=renc.max_compress_len(100) - 1),
              U(b"", n=renc.MAX_OK + 1, cap=0xFFFFFFFF)]
    rng.shuffle(units)
    return units


def frame_units(rng):
    U = fenc.Unit
    units = [U(fenc._text(n, i)) for i, n in enumerate((0, 1, BLOCK - 1, BLOCK, BLOCK + 1))]
    units += [U(fenc._text(3 * BLOCK, 4)), U(fenc._text(2 * BLOCK + 1, 5)), U(fenc._text(2 * BLOCK + BLOCK - 1, 6))]
    units += [U(bytes(2 * BLOCK + 17)), U(fenc._random(2 * BLOCK + 999, 1)), U(fenc._random(700, 2))]
    units += [U(corpus("alice29.txt")), U(corpus("fireworks.jpeg"))]
    units += [U(fenc._text(2 * BLOCK + 3, 9), cap=fenc.frame_max_len(2 * BLOCK + 3) - 1),
              U(fenc._text(100, 9), cap=fenc.frame_max_len(100) - 1), U(b"")]
    rng.shuffle(units)
    return units


@pytest.mark.parametrize("addressing", ["ptrs", "base"])
def test_raw_tables_equal_the_build(addressing):
    units = raw_units(random.Random(1))
    streams, tables = check(False, units, addressing=addressing)
    for i, u in enumerate(units):
        magic, n, dn, hl, nb, seek, reason = rtab.head_of(np.frombuffer(tables[i], dtype=np.uint8))
        assert n == len(streams[i]) and bool(seek) == (n > 0), i


@pytest.mark.parametrize("addressing,index", [("ptrs", True), ("base", True), ("ptrs", False)])
def test_frame_tables_equal_the_build(addressing, index):
    check(True, frame_units(random.Random(2)), addressing=addressing, index=index)


@pytest.mark.parametrize("frame", [False, True])
def test_lengths_over_in_bytes(frame):
    """Multi-block units past in_bytes are Invalid{sum, in_bytes} with no output, so their tables are a 0-byte
    stream's; the others still get theirs."""
    mod = fenc if frame else renc
    units = [mod.Unit(mod._text(2 * BLOCK + 5, 1)), mod.Unit(mod._text(500, 2)), mod.Unit(mod._text(3 * BLOCK, 3)),
             mod.Unit(mod._text(BLOCK, 4))]
    total = mod.multi_bytes(units)
    _, tables = check(frame, units, in_bytes=total - 1)
    assert [len(t) for t in tables] == [HEAD, HEAD + (32 if frame else 8), HEAD, HEAD + (32 if frame else 8)]


def test_reads_over_raw_tables():
    rng = random.Random(3)
    units = [renc.Unit(renc._text(3 * BLOCK + 1, 7)), renc.Unit(renc._random(2 * BLOCK, 8)),
             renc.Unit(renc._text(BLOCK - 1, 9)), renc.Unit(bytes(BLOCK + 1)), renc.Unit(b"")]
    streams, tables = check(False, units)
    pairs = [(rtab.upload(s), np.frombuffer(t, dtype=np.uint8).copy()) for s, t in zip(streams, tables)]
    ranges = []
    for i, u in enumerate(units):
        ranges += [(i, lo, ln) for lo, ln in rtab.boundary_ranges(u.n, rng, extra=4)]
    rc, got = rtab.read(pairs, ranges)
    assert rc == 0
    for (i, lo, ln), (st, data) in zip(ranges, got):
        assert st == rtab.OK and data == units[i].data[lo:lo + ln], (i, lo, ln, st)


def test_reads_over_frame_tables():
    rng = random.Random(4)
    units = [fenc.Unit(fenc._text(3 * BLOCK + 1, 7)), fenc.Unit(fenc._random(2 * BLOCK, 8)),
             fenc.Unit(fenc._text(BLOCK - 1, 9)), fenc.Unit(bytes(BLOCK + 1))]
    streams, tables = check(True, units, index=True)
    pairs = [(fread.upload(s), np.frombuffer(t, dtype=np.uint8).copy()) for s, t in zip(streams, tables)]
    ranges = []
    for i, u in enumerate(units):
        ranges += [(i, lo, ln) for lo, ln in rtab.boundary_ranges(u.n, rng, extra=4) if lo + ln <= u.n]
    rc, got = fread.read(pairs, ranges)
    assert rc == 0
    for (i, lo, ln), (st, data) in zip(ranges, got):
        assert st[0] == "Ok" and data == units[i].data[lo:lo + ln], (i, lo, ln, st)


@pytest.mark.parametrize("frame", [False, True])
def test_short_tables_or_scratch_and_call_checks(frame):
    mod = fenc if frame else renc
    units = [mod.Unit(mod._text(2 * BLOCK + 1, 5)), mod.Unit(mod._text(10, 6))]
    assert run(frame, units, tables_short=1)[0] == INVALID
    assert run(frame, units, scratch_short=1)[0] == INVALID
    assert run(frame, [])[0] == 0
    L = elib()
    f = 1 if frame else 0
    assert L.emu_encode_tabled_scratch_bytes(f, 0xFFFFFFFF >> 1, 1 << 48) == 2 ** 64 - 1
    b = emu.SbBatch()
    lens = np.zeros(4, dtype=np.uint32)
    buf = np.zeros(1 << 16, dtype=np.uint8)
    p = C.c_void_p(buf.ctypes.data)
    b.out_lens, b.count = lens.ctypes.data, 1
    assert L.emu_encode_tabled(f, None, C.c_uint64(0), None, p, C.c_uint64(1 << 12), p, p, p, C.c_uint64(1 << 15)) == INVALID
    for k in range(4):
        args = [p, p, p, p]
        args[k] = None
        assert L.emu_encode_tabled(f, C.byref(b), C.c_uint64(0), None, args[0], C.c_uint64(1 << 12), args[1], args[2],
                                   args[3], C.c_uint64(1 << 15)) == INVALID, k
    b.count = 1 << 31
    assert L.emu_encode_tabled(f, C.byref(b), C.c_uint64(0), None, p, C.c_uint64(1 << 12), p, p, p,
                               C.c_uint64(1 << 15)) == INVALID
    assert (buf == 0).all() and (lens == 0).all()
