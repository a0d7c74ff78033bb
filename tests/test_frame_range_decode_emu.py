"""Range decode of one frame stream on CPU: K5's index phase (K7 or the caller's index, parse, walk, scan) and the k12_*
kernel bodies of rust-snappy_b200/csrc/k12_frame_range_decode.cuh (plan, pair scan, decode + CRC, finish) compiled by
g++ against the fiber warp emulator with small grids. Every range's (status, out_len, bytes) must be what the oracle's
frame_decode gives for those bytes; nothing may be written past a range's buffer, the staging or the scratch. Test
tooling only, like tests/test_frame_batch_decode_emu.py."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import emu_helpers as emu
import legal_streams as ls
from test_frame_batch_decode_emu import IDENT, NAMES, _flip, _text, chain, oracle_decode

INVALID = 202
GUARD = 512
SEG = 128 << 10
BLOCK = 65536
SLOT = 65536

_HERE = os.path.dirname(os.path.abspath(__file__))
_EMU = os.path.join(_HERE, "emu")
_SO = os.path.join(_EMU, "_build", "libemu_frame_range_decode.so")
_lib = None


def rdlib():
    """The emulator build of K12's bodies (tests/emu/emu_frame_range_decode.cpp), rebuilt when a source is newer."""
    global _lib
    if _lib is None:
        csrc = os.path.join(os.path.dirname(_HERE), "rust-snappy_b200", "csrc")
        srcs = [os.path.join(_EMU, f) for f in ("emu_frame_range_decode.cpp", "simt_emu.cpp", "simt_emu.h")]
        srcs += [os.path.join(csrc, f) for f in os.listdir(csrc)]
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            tmp = "%s.%d.tmp" % (_SO, os.getpid())
            subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unused-function",
                                   "-Wno-unknown-pragmas", "-Wl,-Bsymbolic", "-o", tmp,
                                   os.path.join(_EMU, "emu_frame_range_decode.cpp"), os.path.join(_EMU, "simt_emu.cpp")])
            os.replace(tmp, _SO)
        _lib = C.CDLL(_SO)
        _lib.emu_frame_decode_ranges_scratch_bytes.restype = C.c_uint64
        _lib.emu_frame_decode_ranges_scratch_bytes.argtypes = [C.c_uint32, C.c_uint32]
        _lib.emu_frame_decode_ranges.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_uint32, C.c_uint32, C.c_void_p,
                                                 C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p,
                                                 C.c_void_p, C.c_uint64, C.c_uint32, C.c_uint64, C.c_void_p]
    return _lib


def status_of(e):
    return (emu.ERR.get(e.code, NAMES.get(e.code, str(e.code))), e.a, e.b, e.c)


def run_ranges(stream, ranges, fragment=False, index=None, max_chunks=None, scratch_short=0, seg=SEG):
    """sb_frame_decode_ranges_device_ws under the emulator. Returns rc, [(status, bytes)] and the stream's
    (status, bytes, nchunks); checks the guard bytes after every range's buffer, after the staging and after the scratch."""
    n = len(stream)
    src = np.frombuffer(bytes(stream) + bytes(16), dtype=np.uint8).copy()
    if max_chunks is None:
        max_chunks = n // 8 + 16
    count = len(ranges)
    lens = [ln for _, ln in ranges]
    # every range's buffer is its length plus 16 guard bytes, at odd offsets
    offs, at = [], 3
    for ln in lens:
        offs.append(at)
        at += ln + 16 + 1 - ln % 2
    out = np.full(at + 16, 0xEE, dtype=np.uint8)
    t_lo = np.array([lo for lo, _ in ranges] + [0], dtype=np.uint64)
    t_len = np.array(lens + [0], dtype=np.uint64)
    t_ptr = np.array([out.ctypes.data + o for o in offs] + [0], dtype=np.uint64)
    out_lens = np.full(count + 1, 0xDEADBEEF, dtype=np.uint64)
    st = (emu.SbError * max(count, 1))()
    res = emu.SbFrameResult()
    idx = np.array(list(index) + [0xCDCD], dtype=np.uint64) if index is not None else None
    L = rdlib()
    size = L.emu_frame_decode_ranges_scratch_bytes(max_chunks, count)
    scratch = np.full(size + GUARD, 0xCD, dtype=np.uint8)
    sat = C.c_uint64(0)
    rc = L.emu_frame_decode_ranges(src.ctypes.data, n, idx.ctypes.data if idx is not None else None,
                                   len(index) - 1 if index is not None else 0, 1 if fragment else 0, t_lo.ctypes.data,
                                   t_len.ctypes.data, t_ptr.ctypes.data, out_lens.ctypes.data, C.addressof(st), count,
                                   C.byref(res), scratch.ctypes.data, size - scratch_short, max_chunks, seg, C.byref(sat))
    if rc:
        assert (out_lens == 0xDEADBEEF).all() and (out == 0xEE).all()
        return rc, None, None
    assert (scratch[sat.value + 2 * SLOT * count:] == 0xCD).all()       # nothing past the staging or the scratch
    assert int(out_lens[count]) == 0xDEADBEEF
    got = []
    for i, (o, ln) in enumerate(zip(offs, lens)):
        assert bytes(out[o + ln:o + ln + 16]) == b"\xee" * 16, i         # nothing written past the range's buffer
        k = int(out_lens[i])
        assert k <= ln, i
        got.append((status_of(st[i]), bytes(out[o:o + k])))
    return 0, got, (status_of(res.status), res.bytes, res.nchunks)


OK = ("Ok", 0, 0, 0)


def spans(stream, fragment=False):
    """(output offset, decoded length) of every data chunk of a stream's header chain, and the total."""
    out, at = [], 0
    for o in chain(stream, fragment)[:-1]:
        ln = int.from_bytes(stream[o + 1:o + 4], "little")
        if stream[o] == 1:
            d = ln - 4
        elif stream[o] == 0:
            d = emu_len(stream[o + 8:o + 4 + ln])
        else:
            continue
        out.append((at, d))
        at += d
    return out, at


def emu_len(body):
    v, shift = 0, 0
    for b in body[:10]:
        v |= (b & 0x7F) << shift
        if b < 0x80:
            return v
        shift += 7
    raise AssertionError("no varint")


def verifies(off, dlen, lo, n, total):
    end = min(lo + n, total)
    return off < end and off + max(dlen, 1) > lo


def boundary_ranges(offsets, total):
    """Empty ranges, ranges from 0, to total, past total and past it entirely, one byte at every chunk boundary +-1,
    inside one chunk, across two and over all -- shuffled, with duplicates."""
    r = [(0, 0), (7, 0), (total, 0), (0, total), (0, total + 100), (total, 10), (total + 5, 3), (0, 1), (max(total - 1, 0), 1)]
    for b in offsets[1:]:
        r += [(b - 1, 1), (b, 1), (b + 1, 1), (b - 3, 7)]
    if total > 3000:
        r += [(1000, 2000), (total // 2, 1), (total // 3, total // 3), (5, total - 10)]
    r += r[:4]
    random.Random(total).shuffle(r)
    return [(lo, n) for lo, n in r if lo >= 0]


def check_valid(oracle, stream, ranges, fragment=False, **kw):
    data = oracle.frame_decode(IDENT + stream if fragment else stream)
    rc, got, res = run_ranges(stream, ranges, fragment=fragment, **kw)
    assert rc == 0
    for (lo, n), g in zip(ranges, got):
        assert g == (OK, data[lo:lo + n]), (lo, n, g[0])
    assert res[0] == OK and res[1] == len(data)
    return got, res


def _encoded(oracle, n, seed):
    s = oracle.frame_encode(_text(n, seed))
    return s, chain(s)


@pytest.mark.parametrize("how", ["k7", "index", "walk"])
def test_encoder_output(oracle, how):
    """Encoder output indexed by K7, by the encoder's own index, and walked (an index that does not describe the
    stream): every path gives the oracle's bytes."""
    s, ix = _encoded(oracle, 5 * BLOCK + 777, 1)
    sp, total = spans(s)
    ranges = boundary_ranges([o for o, _ in sp], total)
    kw = {"index": ix} if how == "index" else {}
    if how == "walk":
        kw["index"] = ix[:2] + [ix[-1]]                                   # an index that does not describe it: walked
    _, res = check_valid(oracle, s, ranges, **kw)
    assert res[2] == len(sp)


def test_generated_streams_walk(oracle):
    """Stored, compressed, empty, padding and skippable chunks (walked), and a repeated identifier."""
    rng = random.Random(3)
    empty = ls.chunk(0x01, b"", oracle.crc32c_masked(b"")) + ls.chunk(0x00, b"\x00", oracle.crc32c_masked(b""))
    for k in range(4):
        g = ls.gen_frame(rng, oracle.crc32c_masked, 14)
        s = g.stream + empty + (IDENT if k % 2 else b"") + ls.gen_frame(rng, oracle.crc32c_masked, 5).stream[10:]
        sp, total = spans(s)
        assert sum(1 for _, d in sp if d == 0) >= 2
        ranges = boundary_ranges([o for o, _ in sp], total)
        ranges += [(o, 0) for o, d in sp if d == 0]
        check_valid(oracle, s, ranges)


def test_fragments(oracle):
    s, _ = _encoded(oracle, 3 * BLOCK + 5, 4)
    frag = s[10:]
    sp, total = spans(frag, True)
    ranges = boundary_ranges([o for o, _ in sp], total)
    check_valid(oracle, frag, ranges, fragment=True)
    check_valid(oracle, frag, ranges, fragment=True, index=chain(frag, True))
    g = ls.gen_frame(random.Random(9), oracle.crc32c_masked, 8)
    sp, total = spans(g.stream[10:], True)
    check_valid(oracle, g.stream[10:], boundary_ranges([o for o, _ in sp], total), fragment=True)


@pytest.mark.parametrize("where", ["crc", "body"])
@pytest.mark.parametrize("indexed", [False, True])
def test_one_corrupted_chunk(oracle, where, indexed):
    """Ranges that verify the corrupted chunk get the oracle's error for the stream up to that chunk, with the bytes
    before it; every other range is Ok."""
    clean, ix = _encoded(oracle, 4 * BLOCK + 999, 5)
    data = oracle.frame_decode(clean)
    sp, total = spans(clean)
    j = 2
    s = _flip(clean, ix[j] + (5 if where == "crc" else 40))
    err = oracle_decode(oracle, s[:ix[j + 1]])[0]
    assert err[0] != "Ok"
    ranges = boundary_ranges([o for o, _ in sp], total)
    rc, got, res = run_ranges(s, ranges, index=ix if indexed else None)
    assert rc == 0 and res == (OK, total, len(sp))
    off = sp[j][0]
    hits = 0
    for (lo, n), g in zip(ranges, got):
        if verifies(off, sp[j][1], lo, n, total):
            hits += 1
            assert g == (err, data[lo:max(off, lo)]), (lo, n)
        else:
            assert g == (OK, data[lo:lo + n]), (lo, n)
    assert 0 < hits < len(ranges)


def test_two_corrupted_chunks_first_in_stream_order(oracle):
    clean, ix = _encoded(oracle, 4 * BLOCK, 6)
    data = oracle.frame_decode(clean)
    s = _flip(_flip(clean, ix[1] + 5), ix[3] + 6)
    err = oracle_decode(oracle, s[:ix[2]])[0]
    rc, got, _ = run_ranges(s, [(0, 4 * BLOCK), (BLOCK + 3, 3 * BLOCK), (3 * BLOCK + 1, 10), (10, 10)])
    assert got[0] == (err, data[:BLOCK]) and got[1] == (err, b"")
    assert got[2][0][0] == "Checksum" and got[2][1] == b"" and got[3] == (OK, data[10:20])


def test_truncated_stream(oracle):
    """Ranges past the decoded total of a truncated stream get the walk's error; the rest are Ok."""
    clean, ix = _encoded(oracle, 3 * BLOCK + 100, 7)
    s = clean[:-5]
    err = oracle_decode(oracle, s)[0]
    data = oracle.frame_decode(clean[:ix[-2]])
    total = len(data)
    ranges = [(0, total), (0, total + 1), (total - 1, 1), (total - 1, 2), (total, 1), (total + 9, 1), (5, 10), (total, 0)]
    rc, got, res = run_ranges(s, ranges)
    assert rc == 0 and res == (err, total, 3)
    for (lo, n), g in zip(ranges, got):
        want = err if lo + n > total else OK
        assert g == (want, data[lo:lo + n]), (lo, n)


@pytest.mark.parametrize("indexed", [False, True])
def test_chunk_table_one_short(oracle, indexed):
    s, ix = _encoded(oracle, 3 * BLOCK + 1, 8)
    ranges = [(0, 10), (BLOCK, 5), (0, 0)]
    rc, got, res = run_ranges(s, ranges, max_chunks=3, index=ix if indexed else None)
    if indexed:
        assert rc == INVALID                                               # nchunks > max_chunks: an argument error
        return
    assert rc == 0 and res[0] == ("Invalid", 3, 1, 0)
    assert all(g == (("Invalid", 3, 1, 0), b"") for g in got)
    check_valid(oracle, s, ranges, max_chunks=4)


def test_no_ranges_gives_the_decoded_length(oracle):
    s, ix = _encoded(oracle, 2 * BLOCK + 3, 9)
    for index in (None, ix):
        rc, got, res = run_ranges(s, [], index=index)
        assert rc == 0 and got == [] and res == (OK, 2 * BLOCK + 3, 3)
    rc, _, res = run_ranges(b"", [(0, 5)])
    assert rc == 0 and res == (OK, 0, 0)


def test_segments_and_small_ranges(oracle):
    """A stream over several K7 segments, with many one-byte and straddling ranges."""
    s, ix = _encoded(oracle, 9 * BLOCK + 12345, 10)
    sp, total = spans(s)
    rng = random.Random(2)
    ranges = [(rng.randrange(total), rng.randrange(1, 3 * BLOCK)) for _ in range(20)]
    check_valid(oracle, s, ranges)
    check_valid(oracle, s, ranges, index=ix, seg=0)


def test_call_checks_and_scratch(oracle):
    L = rdlib()
    f = L.emu_frame_decode_ranges_scratch_bytes
    assert f(10, 0) < f(1000, 0) < f(1000, 1) < f(1000, 2)
    assert f(1000, 2) - f(1000, 1) >= 2 * SLOT
    s, ix = _encoded(oracle, BLOCK + 1, 11)
    assert run_ranges(s, [(0, 5)], scratch_short=1)[0] == INVALID
    assert run_ranges(s, [(0, 5)], max_chunks=(1 << 22) - 1)[0] == INVALID
    assert run_ranges(s, [(0, 5)], max_chunks=0)[0] == INVALID
    assert run_ranges(s, [(0, 5)], index=ix, max_chunks=1)[0] == INVALID
    res = emu.SbFrameResult()
    scratch = np.zeros(1 << 20, dtype=np.uint8)
    sat = C.c_uint64(0)
    arr = np.zeros(8, dtype=np.uint64).ctypes.data

    def call(inp=1, nr=0, r=C.byref(res), sc=scratch.ctypes.data, arrays=(None,) * 5):
        return L.emu_frame_decode_ranges(None if not inp else scratch.ctypes.data, 16, None, 0, 0, *arrays[:3], arrays[3],
                                         arrays[4], nr, r, sc, 1 << 20, 8, 0, C.byref(sat))
    assert call() == 0
    assert call(inp=0) == INVALID and call(r=None) == INVALID and call(sc=None) == INVALID
    for k in range(5):                                                     # ranges with one of their arrays missing
        assert call(nr=1, arrays=tuple(None if m == k else arr for m in range(5))) == INVALID
    assert call(nr=1 << 31, arrays=(arr,) * 5) == INVALID
