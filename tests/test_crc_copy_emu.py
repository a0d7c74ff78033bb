"""K3's warp CRC-32C, the warp copy and the K4/K5 two-level scan at their alignment, length and count edges, on CPU: the
kernel bodies compiled by g++ against the fiber warp emulator (tests/emu/emu_crc_copy.cpp) and compared with the C oracle,
a bitwise CRC that shares no table code with the kernels, and numpy. Also K5's chunk-table overflow status and its
decode at scan-tile edges through the existing emulator build. Test tooling only, like tests/test_emu_kernels.py."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import emu_helpers as emu
from conftest import corpus
from test_frame_index_emu import IDENT, frame_decode_indexed, oracle_decode

_HERE = os.path.dirname(os.path.abspath(__file__))
_EMU = os.path.join(_HERE, "emu")
_SO = os.path.join(_EMU, "_build", "libemu_crc_copy.so")
_lib = None

# lengths around the slice, vector and block sizes of both CRC variants and the warp copy
EDGE_LENS = [1023, 1024, 1025, 2047, 2048, 2049, 2050, 2111, 2112, 2113, 4095, 4096, 4097, 65535, 65536, 65537]
K4_TILE = 1024


def lib():
    """The emulator build of K3, the warp copy and the scan (tests/emu/emu_crc_copy.cpp), rebuilt when a source is newer.
    Its own library next to libemu_kernels.so; -Bsymbolic keeps each bound to its own emulator copy."""
    global _lib
    if _lib is None:
        csrc = os.path.join(os.path.dirname(_HERE), "rust-snappy_b200", "csrc")
        srcs = [os.path.join(_EMU, f) for f in ("emu_crc_copy.cpp", "simt_emu.cpp", "simt_emu.h")]
        srcs += [os.path.join(csrc, f) for f in os.listdir(csrc)]
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            tmp = "%s.%d.tmp" % (_SO, os.getpid())
            subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unused-function",
                                   "-Wno-unknown-pragmas", "-Wl,-Bsymbolic", "-o", tmp,
                                   os.path.join(_EMU, "emu_crc_copy.cpp"), os.path.join(_EMU, "simt_emu.cpp")])
            os.replace(tmp, _SO)
        _lib = C.CDLL(_SO)
        _lib.emu_warp_copy_fenced.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p, C.c_int, C.c_int]
    return _lib


def masked(crc):
    return (((crc >> 15) | (crc << 17)) + 0xA282EAD8) & 0xFFFFFFFF


def fill(kind, n, seed=1):
    if kind == "random":
        return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8)
    return np.full(n, 0 if kind == "zeros" else 0xFF, dtype=np.uint8)


def aligned(n, pad=64):
    """uint8 array of n bytes whose first byte sits on a 16-byte boundary (a view into a larger allocation)."""
    raw = np.zeros(n + pad, dtype=np.uint8)
    at = (-raw.ctypes.data) % 16
    return raw[at:at + n]


def crc_units(lens):
    """(offset, length) units: every length at every base offset 0..15 relative to a 16-byte boundary."""
    units, at = [], 0
    for n in lens:
        for a in range(16):
            units.append((at + a, n))
            at += (n + 16 + 15) // 16 * 16
    return units, at


def crc_batch(buf, units, grid=3):
    """k3_crc_body (sb_crc32c_masked_batch_device) over the units, through in_ptrs/in_lens."""
    ptrs = np.array([buf.ctypes.data + o for o, _ in units], dtype=np.uint64)
    lens = np.array([n for _, n in units], dtype=np.uint32)
    out = np.full(len(units), 0xDEADBEEF, dtype=np.uint32)
    b = emu.SbBatch()
    b.in_ptrs = ptrs.ctypes.data
    b.in_lens = lens.ctypes.data
    b.out_lens = out.ctypes.data
    b.count = len(units)
    lib().emu_crc_batch(C.byref(b), grid)
    return [int(x) for x in out]


def crc1(buf, units):
    """k3_warp_crc32c_masked1 (K1's fused chunk checksum) over the units."""
    ptrs = np.array([buf.ctypes.data + o for o, _ in units], dtype=np.uint64)
    lens = np.array([n for _, n in units], dtype=np.uint32)
    out = np.full(len(units), 0xDEADBEEF, dtype=np.uint32)
    lib().emu_crc1(C.c_void_p(ptrs.ctypes.data), C.c_void_p(lens.ctypes.data), C.c_uint32(len(units)), C.c_void_p(out.ctypes.data))
    return [int(x) for x in out]


def _first_diff(got, want, units):
    bad = [(u, hex(g), hex(w)) for g, w, u in zip(got, want, units) if g != w]
    return bad[:8], len(bad)


@pytest.mark.parametrize("kind", ["random", "zeros", "ones"])
def test_crc_variants_every_length_and_offset(oracle, kind):
    """Both warp CRC variants for every n in 0..700 and the edge lengths, each at base offsets 0..15."""
    units, size = crc_units(list(range(701)) + EDGE_LENS)
    buf = aligned(size)
    buf[:] = fill(kind, size, seed=7)
    want = [oracle.crc32c_masked(buf[o:o + n].tobytes()) for o, n in units]
    got = crc_batch(buf, units)
    assert got == want, _first_diff(got, want, units)
    got1 = crc1(buf, units)
    assert got1 == want, _first_diff(got1, want, units)


def test_crc_matches_bitwise_reference(oracle):
    """A subset against a bit-at-a-time CRC that shares no table code with either the kernels or the oracle's table path."""
    rng = random.Random(3)
    units, size = crc_units([0, 1, 3, 4, 31, 32, 63, 64, 65, 127, 128, 129, 255, 511, 700] + EDGE_LENS[:11])
    units = [u for u in units if u[1] < 1000 or rng.random() < 0.25]
    buf = aligned(size)
    buf[:] = fill("random", size, seed=11)
    want = [masked(oracle.lib().orc_crc32c_bitwise(buf[o:o + n].tobytes(), n)) for o, n in units]
    assert crc_batch(buf, units) == want
    assert crc1(buf, units) == want


def _copy_grid(ns, ef, seed):
    """Every (dst mod 16, src mod 16) pair for every n in ns, one warp copy per job; returns (got, want) whole buffers
    plus the jobs, so that any byte written outside [dst, dst + n) shows up as a difference."""
    jobs, spans = [], []
    slot = (max(ns) + 64 + 15) // 16 * 16
    count = 16 * 16 * len(ns)
    src = aligned(slot * count)
    src[:] = fill("random", src.size, seed)
    dst = aligned(slot * count)
    dst[:] = fill("random", dst.size, seed + 1)          # guard bytes: whatever was there must stay
    want = dst.copy()
    k = 0
    for n in ns:
        for d in range(16):
            for s in range(16):
                so, do = k * slot + 16 + s, k * slot + 16 + d
                jobs += [dst.ctypes.data + do, src.ctypes.data + so, n]
                spans.append((d, s, n, do, so))
                want[do:do + n] = src[so:so + n]
                k += 1
    j = np.array(jobs, dtype=np.uint64)
    lib().emu_warp_copy(C.c_void_p(j.ctypes.data), C.c_uint32(len(spans)), 1 if ef else 0)
    return dst, want, spans, slot


@pytest.mark.parametrize("ef", [False, True])
def test_warp_copy_every_alignment_pair(ef):
    for ns in (list(range(201)), [4097, 65536]):
        got, want, spans, slot = _copy_grid(ns, ef, seed=len(ns))
        if not np.array_equal(got, want):
            bad = [(d, s, n) for d, s, n, do, so in spans
                   if not np.array_equal(got[do - 16:do - 16 + slot], want[do - 16:do - 16 + slot])]
            pytest.fail("warp copy wrong for (dst%%16, src%%16, n) in %s (%d jobs)" % (bad[:8], len(bad)))


@pytest.mark.parametrize("at_start", [0, 1])
def test_warp_copy_reads_stay_inside_the_source(at_start):
    """The source ends right before (at_start=0) or begins right after (at_start=1) an inaccessible page: a load past
    either end of [src, src + n) faults. Every destination alignment, every n in 0..200 and two large n."""
    rng = np.random.default_rng(5 + at_start)
    seen = set()
    for n in list(range(201)) + [4097, 65536]:
        data = rng.integers(0, 256, n, dtype=np.uint8)
        for d in range(16):
            for ef in (0, 1):
                out = aligned(n + 64)
                out[:] = 0xEE
                mod = lib().emu_warp_copy_fenced(data.ctypes.data, n, out.ctypes.data + 16 + d, ef, at_start)
                assert mod >= 0
                assert out[16 + d:16 + d + n].tobytes() == data.tobytes(), (n, d, mod, ef)
                assert not (out[:16 + d] != 0xEE).any() and not (out[16 + d + n:] != 0xEE).any(), (n, d, mod, ef)
                if n >= 64:
                    seen.add((d, mod))
    # ending at a page boundary puts the source at every alignment as n varies; starting after one, at 0 only
    assert len(seen) == (256 if at_start == 0 else 16)


@pytest.mark.parametrize("count,threads", [(1, 1024), (1023, 1024), (1024, 1024), (1025, 1024), (2049, 1024),
                                           (32 * K4_TILE + 1, 32), (100000, 32), (64 * K4_TILE, 64)])
def test_two_level_scan(count, threads):
    """scan_local_body + scan_tiles_body against numpy. With fewer scan_tiles threads than tiles, one thread sums several
    tiles (per > 1): the branch a stream of more than 1,048,576 chunks takes in the 1024-thread kernel."""
    vals = np.random.default_rng(count).integers(0, 1 << 17, count, dtype=np.uint32)
    ntiles = (count + K4_TILE - 1) // K4_TILE
    offs = np.full(count, 0xABABABAB, dtype=np.uint64)
    tiles = np.full(ntiles + 1, 0xABABABAB, dtype=np.uint64)
    base = 10
    lib().emu_scan(C.c_uint32(count), C.c_void_p(vals.ctypes.data), C.c_uint64(base), C.c_void_p(offs.ctypes.data),
                   C.c_void_p(tiles.ctypes.data), C.c_uint(threads))
    v = vals.astype(np.uint64)
    absolute = base + np.concatenate([[0], np.cumsum(v)[:-1]])
    starts = np.arange(ntiles) * K4_TILE
    assert np.array_equal(tiles[:ntiles], absolute[starts])
    assert int(tiles[ntiles]) == base + int(v.sum())
    assert np.array_equal(tiles[np.arange(count) // K4_TILE] + offs, absolute)


# ---- K5 through the existing emulator build of the frame decoder

def tiny_chunk_set(oracle):
    """Data chunks of a few bytes, with their decoded bytes: empty type-1 chunks, type-0 chunks of dlen 0 (body b"\\x00"),
    short literals, and compressed chunks whose compressed and decoded lengths differ."""
    forms = [(1, b"", b""), (0, b"\x00", b""), (1, b"z", b"z"), (1, b"abc", b"abc"), (0, b"\x03\x08xyz", b"xyz"),
             (0, b"\x08\x04ab\x09\x02", b"abababab"), (0, b"\x01\x00q", b"q")]
    out = []
    for ty, body, dec in forms:
        assert (oracle.decompress(body) if ty == 0 else body) == dec
        crc = oracle.crc32c_masked(dec)
        out.append((bytes([ty]) + (len(body) + 4).to_bytes(3, "little") + crc.to_bytes(4, "little") + body, dec))
    return out


def tiny_stream(oracle, count, seed, pad=False):
    """Identifier + `count` chunks drawn from tiny_chunk_set: (stream, chunk index, decoded bytes). pad: one padding
    chunk after the identifier, which makes the stream unindexable, so the decoder walks it."""
    forms = tiny_chunk_set(oracle)
    pick = np.random.default_rng(seed).integers(0, len(forms), count)
    lens = np.array([len(f[0]) for f in forms], dtype=np.int64)[pick]
    head = IDENT + (b"\xfe\x02\x00\x00\x00\x00" if pad else b"")
    offs = len(head) + np.concatenate([[0], np.cumsum(lens)])
    stream = head + b"".join([forms[i][0] for i in pick])
    assert int(offs[-1]) == len(stream)
    return stream, offs, b"".join([forms[i][1] for i in pick])


@pytest.mark.parametrize("count", [1023, 1024, 1025, 2049])
def test_k5_decode_at_scan_tile_edges(oracle, count):
    stream, offs, data = tiny_stream(oracle, count, seed=count)
    assert oracle.frame_decode(stream) == data
    for index in ([int(x) for x in offs], None):
        st, out, res = emu.frame_decode(stream, len(data), index=index)
        assert st == ("Ok", 0, 0, 0) and out == data and res.nchunks == count, (index is None, st)
    padded, _, _ = tiny_stream(oracle, count, seed=count, pad=True)
    st, out, res = emu.frame_decode(padded, len(data))
    assert st == ("Ok", 0, 0, 0) and out == data and res.nchunks == count
    # a checksum error in the last tile: the oracle's error and the bytes before it
    bad = bytearray(stream)
    bad[int(offs[count - 2]) + 4] ^= 0x40
    want_st, _ = oracle_decode(oracle, bytes(bad))
    st, out, _ = emu.frame_decode(bytes(bad), len(data))
    assert want_st[0] == "Checksum" and st == want_st and data.startswith(out)


def test_chunk_table_overflow_is_reported_before_the_output_size(oracle):
    """More chunks than max_chunks: Invalid{max_chunks, 1} whatever the output capacity, so a caller grows the table
    before trusting a size -- the walk stopped early and its partial size understates the output."""
    data = corpus("alice29.txt")[:150000]
    stream, offs, _ = emu.frame_encode(data)
    assert len(offs) - 1 == 3 and stream == oracle.frame_encode(data)
    for cap in (1000, len(data)):
        for index in (None, offs):
            st, out, _ = emu.frame_decode(stream, cap, index=index, max_chunks=2)
            assert (st, out) == (("Invalid", 2, 1, 0), b""), (cap, index is None)
        st, out, _ = frame_decode_indexed(stream, cap, max_chunks=2)          # K7 declines, then the walk
        assert (st, out) == (("Invalid", 2, 1, 0), b""), cap
    tiny, _, tdata = tiny_stream(oracle, 300, seed=4)
    for cap in (0, 5, len(tdata)):
        assert emu.frame_decode(tiny, cap, max_chunks=299)[0] == ("Invalid", 299, 1, 0)
    assert emu.frame_decode(tiny, len(tdata), max_chunks=300)[:2] == (("Ok", 0, 0, 0), tdata)
