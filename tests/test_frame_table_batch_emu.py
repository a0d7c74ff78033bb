"""Seek tables of a batch of frame streams on CPU: K11's index-part bodies and the k14_* bodies of
rust-snappy_b200/csrc/k14_frame_table_batch.cuh (size scan, export), compiled by g++ against the fiber warp emulator with
small grids. Every unit that fits the chunk table must get exactly the table bytes and result the emulator's single build
(K5's index phase + k13_export, tests/test_frame_table_emu.py) gives it; the first unit that does not fit and every unit
after it must get the 64-byte too-small header. Nothing may be written outside the packed tables, the offsets, the
results or the scratch, and ranges read through batch-built tables must equal those read through single-built ones.
Test tooling only, like tests/test_frame_table_emu.py."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import emu_helpers as emu
import legal_streams as ls
from test_frame_batch_decode_emu import IDENT, _flip, _random, _text, chain, data_chunks, mixed_streams
from test_frame_range_decode_emu import OK, SEG, boundary_ranges, status_of
from test_frame_table_emu import build, read, upload

INVALID = 202
GUARD = 512
BLOCK = 65536
HEAD = 64
REC = 32
MAGIC = 0x0001000042545342

_HERE = os.path.dirname(os.path.abspath(__file__))
_EMU = os.path.join(_HERE, "emu")
_SO = os.path.join(_EMU, "_build", "libemu_frame_table_batch.so")
_lib = None


def tblib():
    """The emulator build of K11's index part and K14 (tests/emu/emu_frame_table_batch.cpp), rebuilt when a source is
    newer."""
    global _lib
    if _lib is None:
        csrc = os.path.join(os.path.dirname(_HERE), "rust-snappy_b200", "csrc")
        srcs = [os.path.join(_EMU, f) for f in ("emu_frame_table_batch.cpp", "simt_emu.cpp", "simt_emu.h")]
        srcs += [os.path.join(csrc, f) for f in os.listdir(csrc)]
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            tmp = "%s.%d.tmp" % (_SO, os.getpid())
            subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unused-function",
                                   "-Wno-unknown-pragmas", "-Wl,-Bsymbolic", "-o", tmp,
                                   os.path.join(_EMU, "emu_frame_table_batch.cpp"), os.path.join(_EMU, "simt_emu.cpp")])
            os.replace(tmp, _SO)
        _lib = C.CDLL(_SO)
        _lib.emu_frame_table_batch_bytes.restype = C.c_uint64
        _lib.emu_frame_table_batch_bytes.argtypes = [C.c_uint32, C.c_uint32]
        _lib.emu_frame_table_build_batch_scratch_bytes.restype = C.c_uint64
        _lib.emu_frame_table_build_batch_scratch_bytes.argtypes = [C.c_uint32, C.c_uint64, C.c_uint32]
        _lib.emu_frame_table_build_batch.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p,
                                                     C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p,
                                                     C.c_void_p, C.c_uint64, C.c_uint64]
    return _lib


class Built:
    """One batch build: the packed tables buffer, the offsets, the raw results and the inputs."""

    def __init__(self, srcs, buf, offs, res):
        self.srcs, self.buf, self.offs, self.res = srcs, buf, offs, res

    def table(self, i):
        """Unit i's table as a view into the packed buffer (a read then uses it in place)."""
        return self.buf[int(self.offs[i]):int(self.offs[i + 1])]

    def result(self, i):
        r = self.res[i]
        return status_of(r.status), r.bytes, r.nchunks


def run(streams, flags=0, index=None, max_chunks=None, in_bytes=None, addressing="ptrs", tables_short=0, scratch_short=0,
        seg=SEG):
    """sb_frame_table_build_batch_device_ws under the emulator. index: per-unit lists for d_chunk_offs, or None. Returns
    rc and a Built; checks that nothing is written past d_table_offs[count] in the tables, past the offsets, the results
    or the scratch, and that a refused call writes nothing at all."""
    L = tblib()
    n = len(streams)
    if in_bytes is None:
        in_bytes = sum(len(s) for s in streams)
    if max_chunks is None:
        max_chunks = sum(len(s) // 8 + 2 for s in streams)
    srcs = [upload(s) for s in streams]                               # 16 bytes of slack, as the device copies have
    if addressing == "ptrs":
        in_ptrs = np.array([x.ctypes.data for x in srcs] + [0], dtype=np.uint64)
    else:
        stride = max([len(s) for s in streams] + [1]) + 17
        base = np.zeros(n * stride + 16, dtype=np.uint8)
        for i, s in enumerate(streams):
            base[i * stride:i * stride + len(s)] = np.frombuffer(s, dtype=np.uint8)
        srcs = [base[i * stride:i * stride + len(s) + 16] for i, s in enumerate(streams)]
    lens = np.array([len(s) for s in streams] + [0], dtype=np.uint32)
    b = emu.SbBatch()
    if addressing == "ptrs":
        b.in_ptrs = in_ptrs.ctypes.data
    else:
        b.in_base, b.in_stride = base.ctypes.data, stride
    b.in_lens, b.count = lens.ctypes.data, n
    tb = L.emu_frame_table_batch_bytes(n, max_chunks)
    buf = np.full(tb + GUARD, 0xAB, dtype=np.uint8)
    offs = np.full(n + 2, 0xDEADBEEF, dtype=np.uint64)
    res = (emu.SbFrameResult * (n + 1))()
    C.memset(res, 0xA5, C.sizeof(res))
    size = L.emu_frame_table_build_batch_scratch_bytes(n, in_bytes, max_chunks)
    scratch = np.full(size + 2 * GUARD, 0xCD, dtype=np.uint8)
    cidx = cat = None
    if index is not None:
        at_list, flat = [], []
        for ix in index:
            at_list.append(len(flat))
            flat += list(ix)
        at_list.append(len(flat))
        cidx = np.array(flat + [0xCDCD] * 4, dtype=np.uint64)
        cat = np.array(at_list, dtype=np.uint64)
    rc = L.emu_frame_table_build_batch(C.byref(b), in_bytes, flags, cidx.ctypes.data if cidx is not None else None,
                                       cat.ctypes.data if cat is not None else None, max_chunks, buf.ctypes.data,
                                       tb - tables_short, offs.ctypes.data, C.addressof(res),
                                       scratch.ctypes.data + GUARD, size - scratch_short, seg)
    assert (scratch[:GUARD] == 0xCD).all() and (scratch[GUARD + size:] == 0xCD).all()
    if rc or n == 0:
        assert (buf == 0xAB).all() and (offs == 0xDEADBEEF).all()
        assert bytes(res) == b"\xa5" * C.sizeof(res)
        return rc, None
    assert int(offs[n + 1]) == 0xDEADBEEF                               # nothing past the offsets
    assert bytes(res)[n * C.sizeof(emu.SbFrameResult):] == b"\xa5" * C.sizeof(emu.SbFrameResult)
    assert int(offs[0]) == 0 and int(offs[n]) <= tb
    assert (buf[int(offs[n]):] == 0xAB).all()                           # nothing past the packed tables
    for i in range(n):
        assert int(offs[i + 1]) - int(offs[i]) == HEAD + REC * res[i].nchunks, i
        assert res[i]._pad == 0 and res[i].status._pad == 0, i
    return 0, Built(srcs, buf, offs, res)


def single(stream, fragment=False, index=None):
    """The emulator's single build with a chunk table large enough: (table cut to its chunks, result)."""
    rc, table, res = build(stream, fragment=fragment, index=index if index else None,
                           max_chunks=max(len(stream) // 8 + 16, len(index or []) + 1))
    assert rc == 0
    return table[:HEAD + REC * res[2]].tobytes(), res


def check(streams, flags=0, index=None, **kw):
    """Every unit's table and result against its single build; returns the Built."""
    rc, got = run(streams, flags=flags, index=index, **kw)
    assert rc == 0
    for i, s in enumerate(streams):
        want_t, want_r = single(s, bool(flags & 1), index[i] if index is not None else None)
        assert got.result(i) == want_r, (i, len(s), got.result(i), want_r)
        assert got.table(i).tobytes() == want_t, i
    return got


def head_of(t):
    """(magic, n, total, nchunks, full, walk status) of a table's header."""
    w = np.frombuffer(t[:HEAD].tobytes(), dtype=np.uint64)
    return int(w[0]), int(w[1]), int(w[2]), int(w[3]) & 0xFFFFFFFF, int(w[3]) >> 32, \
        (int(w[4]) & 0xFFFFFFFF, int(w[4]) >> 32, int(w[5]), int(w[6]), int(w[7]))


def too_small(t, n, mc):
    return head_of(t) == (MAGIC, n, 0, 0, 1, (INVALID, 0, mc, 1, 0))


def batch_streams(oracle):
    """Encoder output of every size class, generated legal streams, walked, damaged and truncated streams."""
    rng = random.Random(21)
    enc = oracle.frame_encode
    ss = [s for s, _ in mixed_streams(oracle)]
    ss += [enc(b""), enc(b"x"), enc(_text(BLOCK, 2)), enc(_text(9 * BLOCK + 1234, 3)), enc(_random(BLOCK + 1, 4))]
    ss += [ls.gen_frame(rng, oracle.crc32c_masked, k).stream for k in (1, 4, 9, 17)]
    ss += [ls.gen_frame(rng, oracle.crc32c_masked, 8, kinds=("pad", "skip", "raw", "comp")).stream]
    three = enc(_text(3 * BLOCK - 7, 5))
    c3 = chain(three)
    ss += [_flip(three, c3[1] + 6), _flip(_flip(three, c3[0] + 5), c3[2] + 4)]   # flipped CRCs
    ss += [three[:c3[1] + 2], three[:c3[2] + 7], three[:c3[2] + 100], IDENT[:7], three[:-1]]  # truncated header, body
    return ss


@pytest.mark.parametrize("addressing", ["ptrs", "base"])
def test_mixed_batch_equals_single_builds(oracle, addressing):
    check(batch_streams(oracle), addressing=addressing)


def test_caller_index_right_and_wrong(oracle):
    streams = batch_streams(oracle)
    right = [chain(s) if s else [0] for s in streams]
    check(streams, index=right)
    wrong = [list(x) for x in right]
    wrong[2][1] += 1                                                   # a shifted entry
    wrong[3][-1] -= 1                                                  # a wrong last entry
    del wrong[4][1]                                                    # too few chunks
    wrong[5] = [123456789, 5, 77]                                      # garbage
    wrong[6] = []                                                      # no entries at all
    check(streams, index=wrong)


def test_fragments(oracle):
    rng = random.Random(5)
    frags = [oracle.frame_encode(_text(n, n))[10:] for n in (1, BLOCK, 300000)]
    g = ls.gen_frame(rng, oracle.crc32c_masked, 9)
    frags += [b"", g.stream[10:], IDENT + frags[0], frags[2][:-3]]
    check(frags, flags=1)
    check(frags, flags=1, index=[chain(f, True) if f else [0] for f in frags])


def test_in_bytes_below_the_sum(oracle):
    streams = batch_streams(oracle)
    check(streams, in_bytes=sum(len(s) for s in streams) - 1)
    check(streams, in_bytes=0)


@pytest.mark.parametrize("indexed", [False, True])
def test_max_chunks_boundaries(oracle, indexed):
    """max_chunks that unit k fits exactly, then one short: unit k and every unit after it get the too-small header."""
    enc = oracle.frame_encode
    streams = [enc(_text(n, n)) for n in (100000, 5000, 200000, 70000, 0)] + [enc(_text(10, 1))]
    need = [data_chunks(s) for s in streams]
    assert need == [2, 1, 4, 2, 0, 1]
    index = [chain(s) if s else [0] for s in streams] if indexed else None
    for k in (0, 2, 3, 5):
        for mc in (sum(need[:k + 1]), sum(need[:k + 1]) - 1):          # unit k fits exactly, then is one chunk short
            rc, got = run(streams, index=index, max_chunks=mc)
            assert rc == 0
            fit = [sum(need[:i + 1]) <= mc for i in range(len(streams))]
            assert fit[k] == (mc == sum(need[:k + 1]))
            for i, s in enumerate(streams):
                if fit[i]:
                    assert (got.table(i).tobytes(), got.result(i)) == single(s), (k, mc, i)
                else:
                    assert got.result(i) == (("Invalid", mc, 1, 0), 0, 0), (k, mc, i)
                    assert len(got.table(i)) == HEAD and too_small(got.table(i), len(s), mc), (k, mc, i)
            assert int(got.offs[len(streams)]) == HEAD * len(streams) + REC * sum(n for n, f in zip(need, fit) if f)


def test_walked_units_past_the_table(oracle):
    """Walked units take their walk count; the first that does not fit and every unit after it get the header."""
    rng = random.Random(8)
    streams = [ls.gen_frame(rng, oracle.crc32c_masked, 10).stream for _ in range(4)]
    need = [single(s)[1][2] for s in streams]
    mc = need[0] + need[1] - 1
    rc, got = run(streams, max_chunks=mc)
    assert (got.table(0).tobytes(), got.result(0)) == single(streams[0])
    assert all(too_small(got.table(i), len(streams[i]), mc) for i in range(1, 4))


def test_reads_over_batch_tables_equal_single_tables(oracle):
    """Ranges read in place from the packed buffer equal ranges read over single-built tables, for every unit."""
    streams = batch_streams(oracle)
    need = [single(s)[1][2] for s in streams]
    mc = sum(need) - 1                                                   # the last units do not fit
    rc, got = run(streams, max_chunks=mc)
    assert rc == 0
    fit = [got.result(u)[0] != ("Invalid", mc, 1, 0) for u in range(len(streams))]
    k = fit.index(False)
    assert k > 0 and not any(fit[k:])
    units, ranges = [], []
    for u, s in enumerate(streams):
        src = upload(s)
        rc, table, res = build(s, src=src)
        units.append((src, table))
        offs = [int(x) for x in table[HEAD:HEAD + REC * res[2]].view(np.uint64)[3::4]]   # the records' decoded offsets
        ranges += [(u, lo, n) for lo, n in boundary_ranges(offs, res[1])[:12]]
    random.Random(9).shuffle(ranges)
    rc, mine = read([(got.srcs[u], got.table(u)) for u in range(len(streams))], ranges)
    assert rc == 0
    rc, want = read(units, ranges)
    assert rc == 0
    for (u, lo, n), m, w in zip(ranges, mine, want):
        if fit[u]:
            assert m == w, (u, lo, n)
        else:                                                            # what a read over a too-small table gives
            assert m == (("Invalid", mc, 1, 0), b""), (u, lo, n)
    data = oracle.frame_decode(streams[3])
    assert read([(got.srcs[3], got.table(3))], [(0, 5, 100000)])[1] == [(OK, data[5:100005])]


def test_call_checks_write_nothing(oracle):
    L = tblib()
    f = L.emu_frame_table_build_batch_scratch_bytes
    assert f(5, 0, 10) < f(5, 1 << 20, 10) < f(5, 1 << 20, 1000) < f(9, 1 << 20, 1000)
    assert L.emu_frame_table_batch_bytes(3, 10) == 3 * HEAD + 10 * REC
    streams = [oracle.frame_encode(_text(n, 3)) for n in (70000, 10)]
    assert run(streams, tables_short=1)[0] == INVALID
    assert run(streams, scratch_short=1)[0] == INVALID
    assert run(streams, max_chunks=0)[0] == INVALID and run(streams, max_chunks=(1 << 22) - 1)[0] == INVALID
    assert run([], max_chunks=8)[0] == 0                                   # count == 0: nothing written
    check(streams, max_chunks=(1 << 22) - 2)
    b = emu.SbBatch()
    lens = np.zeros(4, dtype=np.uint32)
    b.in_lens, b.count = lens.ctypes.data, 1                              # one empty stream
    bufs = [np.zeros(1 << 14, dtype=np.uint8) for _ in range(4)]        # tables, offsets, results, scratch
    t, o, r, s = (x.ctypes.data for x in bufs)
    ix = np.zeros(4, dtype=np.uint64)

    def call(bb=C.byref(b), a=None, c=None, t=t, o=o, r=r, s=s, mc=8, tb=1 << 12):
        return L.emu_frame_table_build_batch(bb, 0, 0, a, c, mc, t, tb, o, r, s, 1 << 14, 0)
    assert call() == 0
    assert tuple(bufs[1][:16].view(np.uint64)) == (0, HEAD)
    for kw in ({"bb": None}, {"t": None}, {"o": None}, {"r": None}, {"s": None}, {"a": ix.ctypes.data},
               {"c": ix.ctypes.data}, {"mc": 0}, {"mc": (1 << 22) - 1}, {"tb": HEAD + 8 * REC - 1}):
        for x in bufs:
            x[:] = 0x5C
        assert call(**kw) == INVALID, kw
        assert all((x == 0x5C).all() for x in bufs), kw
    b.count = 1 << 31
    assert call() == INVALID and all((x == 0x5C).all() for x in bufs)
