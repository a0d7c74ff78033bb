"""Raw seek tables and ranges over tabled raw streams on CPU: K8b's split-part bodies and the k15_* bodies of
rust-snappy_b200/csrc/k15_raw_table.cuh, compiled by g++ against the fiber warp emulator with small grids and K8's
128 KiB segment. A unit must be seekable exactly when the emulator's batch decode (tests/test_raw_batch_split_emu.py)
splits it and decodes it Ok, or it announces one block at most and decodes Ok; its records must be that decode's cuts and
the blocks' CRCs; every range of a seekable table must equal the model decoder's slice; every table must equal the one a
count == 1 build gives; and nothing may be written outside the tables, the outputs' ranges or the scratch. Test tooling
only, like tests/test_raw_batch_split_emu.py."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import emu_helpers as emu
import legal_streams as ls
from test_raw_batch_split_emu import run_batch

INVALID = 202
GUARD = 512
BLOCK = 65536
HEAD = 64
REC = 8
MAGIC = 0x0001000042545352
FRAME_MAGIC = 0x0001000042545342
SEG = 128 << 10
OK = ("Ok", 0, 0, 0)

_HERE = os.path.dirname(os.path.abspath(__file__))
_EMU = os.path.join(_HERE, "emu")
_SO = os.path.join(_EMU, "_build", "libemu_raw_table.so")
_lib = None


def tlib():
    """The emulator build of K8b's split part and K15 (tests/emu/emu_raw_table.cpp), rebuilt when a source is newer."""
    global _lib
    if _lib is None:
        csrc = os.path.join(os.path.dirname(_HERE), "rust-snappy_b200", "csrc")
        srcs = [os.path.join(_EMU, f) for f in ("emu_raw_table.cpp", "simt_emu.cpp", "simt_emu.h")]
        srcs += [os.path.join(csrc, f) for f in os.listdir(csrc)]
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            tmp = "%s.%d.tmp" % (_SO, os.getpid())
            subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unused-function",
                                   "-Wno-unknown-pragmas", "-Wl,-Bsymbolic", "-o", tmp,
                                   os.path.join(_EMU, "emu_raw_table.cpp"), os.path.join(_EMU, "simt_emu.cpp")])
            os.replace(tmp, _SO)
        _lib = C.CDLL(_SO)
        u64, u32, vp = C.c_uint64, C.c_uint32, C.c_void_p
        for f, args in (("emu_raw_table_bytes", [u32]), ("emu_raw_table_batch_bytes", [u32, u64]),
                        ("emu_raw_table_build_batch_scratch_bytes", [u32, u64]),
                        ("emu_raw_table_ranges_scratch_bytes", [u32])):
            getattr(_lib, f).restype = u64
            getattr(_lib, f).argtypes = args
        _lib.emu_raw_table_build_batch.argtypes = [vp, u64, vp, u64, vp, vp, vp, u64, u64]
        _lib.emu_raw_table_decode_ranges.argtypes = [vp, vp, vp, u32, vp, vp, vp, vp, vp, vp, u32, vp, u64, vp]
    return _lib


def upload(s):
    """A stream as the device holds it: its bytes and 16 bytes of slack."""
    return np.frombuffer(bytes(s) + bytes(16), dtype=np.uint8).copy()


def status_of(e):
    return (emu.ERR.get(e.code, {202: "Invalid", 10: "Checksum"}.get(e.code, str(e.code))), e.a, e.b, e.c)


class Built:
    """One batch build: the packed tables buffer, the offsets, the results and the inputs."""

    def __init__(self, srcs, buf, offs, res):
        self.srcs, self.buf, self.offs, self.res = srcs, buf, offs, res

    def table(self, i):
        return self.buf[int(self.offs[i]):int(self.offs[i + 1])]

    def result(self, i):
        r = self.res[i]
        return status_of(r.status), r.bytes, r.nchunks


def build(streams, in_bytes=None, addressing="ptrs", tables_short=0, scratch_short=0, seg=SEG):
    """sb_raw_table_build_batch_device_ws under the emulator. Returns rc and a Built; checks that nothing is written past
    d_table_offs[count] in the tables, past the offsets, the results or the scratch, and that a refused call writes
    nothing at all."""
    L = tlib()
    n = len(streams)
    if in_bytes is None:
        in_bytes = sum(len(s) for s in streams)
    lens = np.array([len(s) for s in streams] + [0], dtype=np.uint32)
    b = emu.SbBatch()
    if addressing == "ptrs":
        srcs = [upload(s) for s in streams]
        in_ptrs = np.array([x.ctypes.data for x in srcs] + [0], dtype=np.uint64)
        b.in_ptrs = in_ptrs.ctypes.data
    else:
        stride = max([len(s) for s in streams] + [1]) + 17
        base = np.zeros(n * stride + 16, dtype=np.uint8)
        for i, s in enumerate(streams):
            base[i * stride:i * stride + len(s)] = np.frombuffer(s, dtype=np.uint8)
        srcs = [base[i * stride:i * stride + len(s) + 16] for i, s in enumerate(streams)]
        b.in_base, b.in_stride = base.ctypes.data, stride
    b.in_lens, b.count = lens.ctypes.data, n
    tb = L.emu_raw_table_batch_bytes(n, in_bytes)
    buf = np.full(tb + GUARD, 0xAB, dtype=np.uint8)
    offs = np.full(n + 2, 0xDEADBEEF, dtype=np.uint64)
    res = (emu.SbFrameResult * (n + 1))()
    C.memset(res, 0xA5, C.sizeof(res))
    size = L.emu_raw_table_build_batch_scratch_bytes(n, in_bytes)
    scratch = np.full(size + 2 * GUARD, 0xCD, dtype=np.uint8)
    rc = L.emu_raw_table_build_batch(C.byref(b), in_bytes, buf.ctypes.data, tb - tables_short, offs.ctypes.data,
                                     C.addressof(res), scratch.ctypes.data + GUARD, size - scratch_short, seg)
    assert (scratch[:GUARD] == 0xCD).all() and (scratch[GUARD + size:] == 0xCD).all()
    if rc or n == 0:
        assert (buf == 0xAB).all() and (offs == 0xDEADBEEF).all()
        assert bytes(res) == b"\xa5" * C.sizeof(res)
        return rc, None
    assert int(offs[n + 1]) == 0xDEADBEEF
    assert bytes(res)[n * C.sizeof(emu.SbFrameResult):] == b"\xa5" * C.sizeof(emu.SbFrameResult)
    assert int(offs[0]) == 0 and int(offs[n]) <= tb
    assert (buf[int(offs[n]):] == 0xAB).all()
    for i in range(n):
        assert int(offs[i + 1]) - int(offs[i]) == HEAD + REC * res[i].nchunks, i
        assert res[i]._pad == 0 and res[i].status._pad == 0, i
    return 0, Built(srcs, buf, offs, res)


def head_of(t):
    """(magic, n, dn, hl, nblocks, seekable, reason) of a table's header; its padding must be zero."""
    w = np.frombuffer(t[:HEAD].tobytes(), dtype=np.uint64)
    assert not w[5:].any()
    return (int(w[0]), int(w[1]), int(w[2]), int(w[3]) & 0xFFFFFFFF, int(w[3]) >> 32, int(w[4]) & 0xFFFFFFFF,
            int(w[4]) >> 32)


def records(t):
    """[(offset, crc)] of a table's records."""
    r = np.frombuffer(t[HEAD:].tobytes(), dtype=np.uint32)
    return [(int(r[2 * j]), int(r[2 * j + 1])) for j in range(len(r) // 2)]


def read(units, ranges, scratch_short=0, count=None):
    """sb_raw_table_decode_ranges_device_ws under the emulator over units [(src, table)] (numpy arrays; a table may be a
    view into a packed buffer). Every range's buffer holds max(0, min(n, dn - lo)) bytes (dn from its table's header)
    between guard bytes, which must stay untouched, as must the staging's and the scratch's. Returns rc and
    [(status, bytes)]."""
    L = tlib()
    k = len(ranges)
    count = len(units) if count is None else count
    tables = np.array([t.ctypes.data for _, t in units] + [0], dtype=np.uint64)
    ins = np.array([s.ctypes.data for s, _ in units] + [0], dtype=np.uint64)
    in_lens = np.array([len(s) - 16 for s, _ in units] + [0], dtype=np.uint64)

    def room(u, lo, n):
        if u >= len(units) or len(units[u][1]) < HEAD:
            return 0
        dn = head_of(units[u][1])[2]
        return max(0, min(n, dn - lo))
    rooms = [room(u, lo, n) for u, lo, n in ranges]
    outs = [np.full(r + 2 * GUARD, 0xEE, dtype=np.uint8) for r in rooms]
    optrs = np.array([o.ctypes.data + GUARD for o in outs] + [0], dtype=np.uint64)
    unit = np.array([u for u, _, _ in ranges] + [0], dtype=np.uint32)
    lo = np.array([x for _, x, _ in ranges] + [0], dtype=np.uint64)
    ln = np.array([x for _, _, x in ranges] + [0], dtype=np.uint64)
    out_lens = np.full(k + 1, 0xDEADBEEF, dtype=np.uint64)
    st = (emu.SbError * (k + 1))()
    size = L.emu_raw_table_ranges_scratch_bytes(k)
    scratch = np.full(size + GUARD, 0xCD, dtype=np.uint8)
    sat = C.c_uint64(0)
    rc = L.emu_raw_table_decode_ranges(tables.ctypes.data, ins.ctypes.data, in_lens.ctypes.data, count,
                                       unit.ctypes.data, lo.ctypes.data, ln.ctypes.data, optrs.ctypes.data,
                                       out_lens.ctypes.data, C.addressof(st), k, scratch.ctypes.data, size - scratch_short,
                                       C.byref(sat))
    assert (scratch[size:] == 0xCD).all()
    if rc:
        assert (out_lens == 0xDEADBEEF).all()
        return rc, None
    assert int(out_lens[k]) == 0xDEADBEEF
    staging = sat.value
    assert (scratch[staging + 2 * k * BLOCK:size] == 0xCD).all()     # nothing between the staging and the end
    got = []
    for i, (o, r) in enumerate(zip(outs, rooms)):
        assert (o[:GUARD] == 0xEE).all() and (o[GUARD + r:] == 0xEE).all(), i
        m = int(out_lens[i])
        assert m <= r, i
        got.append((status_of(st[i]), o[GUARD:GUARD + m].tobytes()))
    return 0, got


def model(s):
    """The reference's Decoder::decompress(s): (status, bytes or None)."""
    return ls.model_decode(bytes(s), ls.MAX_INPUT)


def boundary_ranges(dn, rng, extra=12):
    """Ranges at and around every block boundary, the whole stream, empty and past-the-end ranges, and random ones."""
    out = [(0, dn), (0, 0), (dn, 5), (dn + 7, 3), (max(dn - 1, 0), 10), (0, 1 << 63)]
    for j in range(0, dn + 1, BLOCK):
        for lo in (j - 1, j, j + 1):
            if 0 <= lo <= dn:
                out += [(lo, 1), (lo, BLOCK), (lo, 2 * BLOCK + 3)]
    for _ in range(extra):
        lo = rng.randrange(dn + 1)
        out.append((lo, rng.randrange(3 * BLOCK)))
    return out


def single(s):
    """(table bytes, result) of a count == 1 build of stream s."""
    rc, got = build([s])
    assert rc == 0
    return got.table(0).tobytes(), got.result(0)


def check_build(streams, want_seekable=None, **kw):
    """Build the batch; every unit is seekable exactly when the emulator's batch decode splits it Ok or it is a
    single-block stream that decodes Ok; seekable records are the decode's cuts with the blocks' CRCs; every table equals
    its count == 1 build. Returns the Built and the model results."""
    rc, got = build(streams, **kw)
    assert rc == 0
    ref = [model(s) for s in streams]
    caps = [len(d) if d is not None else 0 for _, d in ref]
    dres, blocks, cuts = run_batch(streams, caps, in_bytes=kw.get("in_bytes"))
    for i, s in enumerate(streams):
        (st, data), r = ref[i], got.result(i)
        magic, n, dn, hl, nb, seek, reason = head_of(got.table(i))
        assert magic == MAGIC and n == len(s), i
        multi = data is not None and len(data) > BLOCK
        want = st == OK and (blocks[i] > 0 if multi else True)
        if multi:
            assert dres[i][0] == OK, i
        assert bool(seek) == want, (i, len(s), st, blocks[i], reason)
        if want_seekable is not None:
            assert bool(seek) == want_seekable[i], (i, reason)
        if want:
            nblk = (len(data) + BLOCK - 1) // BLOCK
            assert r == (OK, len(data), nblk) and (dn, nb, reason) == (len(data), nblk, 0), i
            offs = cuts[i][:-1] if multi else [hl] * nblk
            crcs = [ls_crc(data[j * BLOCK:(j + 1) * BLOCK]) for j in range(nblk)]
            assert records(got.table(i)) == list(zip(offs, crcs)), i
        else:
            assert r == (("Invalid", i, 0, 5), 0, 0) and (dn, hl, nb) == (0, 0, 0) and reason != 0, (i, r)
            assert len(got.table(i)) == HEAD
    if kw.get("in_bytes") is None or kw["in_bytes"] >= sum(len(s) for s in streams):
        for i, s in enumerate(streams):
            t, r = single(s)
            assert got.table(i).tobytes() == t, i
            assert got.result(i)[1:] == r[1:] and got.result(i)[0] == (r[0] if r[0] == OK else ("Invalid", i, 0, 5)), i
    return got, ref


_crc_oracle = None


def ls_crc(data):
    return _crc_oracle(bytes(data))


@pytest.fixture(autouse=True)
def _crc(oracle):
    global _crc_oracle
    _crc_oracle = oracle.crc32c_masked


def gen_units(rng, oracle):
    """Seekable streams: generated blocked streams over several segments, single-block streams, the encoder's."""
    ss = [ls.gen_stream(rng, n, "blocked", copy_share=c).stream for n, c in ((300000, 0.3), (3 * BLOCK, 0.8),
                                                                             (2 * BLOCK + 1, 0.55))]
    ss += [ls.gen_single(rng).stream for _ in range(4)]
    ss += [ls.gen_stream(rng, BLOCK, "blocked").stream, b"\x00"]
    ss += [oracle.compress(bytes(rng.randrange(4) + 97 for _ in range(200000)))]
    return ss


def test_seekable_batch_reads_equal_the_model(oracle):
    rng = random.Random(1)
    streams = gen_units(rng, oracle)
    got, ref = check_build(streams)
    seek = [head_of(got.table(u))[5] for u in range(len(streams))]
    # a generated block may end in a long-header literal too close to its end to decode alone (the reference checks 4
    # bytes after the tag): such a stream is rightly not seekable
    assert sum(seek) >= len(streams) - 2 and seek[0] and seek[-1] and seek[-2]
    ranges = []
    for u, (_, data) in enumerate(ref):
        if not seek[u]:
            continue
        ranges += [(u, lo, n) for lo, n in boundary_ranges(len(data), rng)]
    ranges += [ranges[3], ranges[7], ranges[3]]                          # repeated
    rng.shuffle(ranges)                                                  # unsorted, mixed units, overlapping
    rc, out = read([(got.srcs[u], got.table(u)) for u in range(len(streams))], ranges)
    assert rc == 0
    for (u, lo, n), (st, b) in zip(ranges, out):
        data = ref[u][1]
        assert st == OK and b == data[lo:lo + n], (u, lo, n)


@pytest.mark.parametrize("addressing", ["ptrs", "base"])
def test_mixed_batch_seekable_exactly_when_split_ok(oracle, addressing):
    rng = random.Random(2)
    good = ls.gen_stream(rng, 200000, "blocked")
    streams = [good.stream]
    while len(streams) < 3:                                              # straddling and reaching back across blocks
        s = ls.gen_stream(rng, 150000, "unblocked")
        if s.straddles:
            streams.append(s.stream)
    streams += [ls.giant_literal(rng, n, f)[0] for n, f in ((70000, "lit62"), (80000, "lit63"))]
    streams += ls.corrupt(rng, good)
    streams += ls.corrupt(rng, ls.gen_single(rng))
    streams += [b"", b"\x00", b"\x00\x00", b"\x80", b"\xff" * 11, ls.varint(1 << 33) + b"\x00",
                ls.varint(BLOCK + 5) + b"\x00abc", ls.varint(3) + b"\x08abc", ls.varint(3) + b"\x08ab"]
    got, ref = check_build(streams, addressing=addressing)
    assert [head_of(got.table(i))[5] for i in (1, 2, 3, 4)] == [0, 0, 0, 0]
    assert [head_of(got.table(i))[5] for i in range(len(streams) - 9, len(streams))] == [0, 1, 0, 0, 0, 0, 0, 1, 0]
    for i, (st, _) in enumerate(ref):
        if st != OK:
            assert head_of(got.table(i))[5] == 0, i


def test_in_bytes_under_the_sum(oracle):
    """Lengths summing past in_bytes: no unit is split, so only single-block units are seekable."""
    rng = random.Random(3)
    streams = gen_units(rng, oracle)
    total = sum(len(s) for s in streams)
    for in_bytes in (total - 1, 0):
        got, ref = check_build(streams, in_bytes=in_bytes)
        for i, (st, d) in enumerate(ref):
            h = head_of(got.table(i))
            if d is None:
                continue
            assert h[5] == (len(d) <= BLOCK), i
            if len(d) > BLOCK:
                assert h[6] == 2, i


def test_read_statuses_and_guards(oracle):
    """Unit out of range, a stream of another length, a frame table, a non-seekable stream, tampered records and
    headers, and a same-length stream with one byte changed."""
    rng = random.Random(4)
    good = ls.gen_stream(rng, 5 * BLOCK + 333, "blocked", copy_share=0.3)
    bad = ls.gen_stream(rng, 150000, "unblocked")
    streams = [good.stream, bad.stream if bad.straddles else b"\x00\x00"]
    got, ref = check_build(streams)
    data = ref[0][1]
    src, table = got.srcs[0], got.table(0).copy()
    assert head_of(table)[5] == 1 and head_of(got.table(1))[5] == 0
    n = len(good.stream)
    frame = np.zeros(HEAD, dtype=np.uint8)
    frame[:16] = np.frombuffer(np.array([FRAME_MAGIC, n], dtype=np.uint64).tobytes(), dtype=np.uint8)
    short = upload(good.stream[:-1])
    rc, out = read([(src, table), (got.srcs[1], got.table(1)), (src, frame), (short, table)],
                   [(0, 5, 10), (7, 0, 10), (1, 0, 10), (2, 0, 10), (3, 0, 10)], count=4)
    assert rc == 0
    assert [s for s, _ in out] == [OK, ("Invalid", 7, 4, 1), ("Invalid", 1, 0, 5), ("Invalid", n, 0, 2),
                                   ("Invalid", n - 1, n, 2)]
    assert out[0][1] == data[5:15] and all(b == b"" for _, b in out[1:])

    def ranges_over(t, s=src):
        rs = [(lo, ln) for lo, ln in boundary_ranges(len(data), rng, 6)]
        rc, out = read([(s, t)], [(0, lo, ln) for lo, ln in rs])
        assert rc == 0
        return rs, out

    # a CRC that does not match: block 2 fails with c=4, for the ranges that cover it only
    t = table.copy()
    t[HEAD + 8 * 2 + 4] ^= 1
    for (lo, ln), (st, b) in zip(*ranges_over(t)):
        end = min(lo + ln, len(data))
        if lo < 3 * BLOCK and end > 2 * BLOCK:
            assert st == ("Invalid", 2, 0, 4) and b == data[lo:max(2 * BLOCK, lo)], (lo, ln)
        else:
            assert st == OK and b == data[lo:lo + ln], (lo, ln)
    # one byte of block 3's literal payload changed, same length: c=4 for ranges covering block 3, Ok elsewhere
    e = next(x for x in good.elems if x[2] == 0 and x[6] >= 3 * BLOCK and x[6] + x[3] <= 4 * BLOCK)
    flip = bytearray(good.stream)
    flip[e[0] + e[1]] ^= 0x40
    for (lo, ln), (st, b) in zip(*ranges_over(table, upload(flip))):
        end = min(lo + ln, len(data))
        if lo < 4 * BLOCK and end > 3 * BLOCK:
            assert st == ("Invalid", 3, 0, 4) and b == data[lo:max(3 * BLOCK, lo)], (lo, ln)
        else:
            assert st == OK and b == data[lo:lo + ln], (lo, ln)
    # records that break the build's bounds: c=3 at the first covered block whose bytes they move
    offs = [o for o, _ in records(table)]
    for j, v in ((3, offs[2] - 1), (4, n + 1), (0, 0), (5, offs[4]), (2, 0xFFFFFFFF)):
        t = table.copy()
        t[HEAD + 8 * j:HEAD + 8 * j + 4] = np.frombuffer(np.uint32(v).tobytes(), dtype=np.uint8)
        moved = {j - 1, j} if j else {0}
        for (lo, ln), (st, b) in zip(*ranges_over(t)):
            end = min(lo + ln, len(data))
            cov = [k for k in range(lo >> 16, ((end - 1) >> 16) + 1)] if end > lo else []
            hit = [k for k in cov if k in moved]
            if hit and st[3] == 3:
                assert st[1] == hit[0] and b == data[lo:max(hit[0] * BLOCK, lo)], (j, v, lo, ln, st)
            elif hit:                                                    # in bounds, but not this block's bytes
                assert st == ("Invalid", hit[0], 0, 4), (j, v, lo, ln, st)
            else:
                assert st == OK and b == data[lo:lo + ln], (j, v, lo, ln)
    # headers that break the bounds: every range that covers a block fails at its first block with c=3
    for at, v in ((28, np.uint32(7)), (16, np.uint64(1 << 33)), (16, np.uint64(len(data) + BLOCK))):   # nblocks, dn
        t = table.copy()
        raw = np.frombuffer(v.tobytes(), dtype=np.uint8)
        t[at:at + raw.size] = raw
        dn = head_of(t)[2]
        for lo, ln in boundary_ranges(len(data), rng, 6):
            rc, out = read([(src, t)], [(0, lo, ln)])
            end = min(lo + ln, dn)
            assert out[0] == ((("Invalid", lo >> 16, 0, 3), b"") if end > lo else (OK, b"")), (at, lo, ln)


def test_moved_tables_and_single_builds_agree(oracle):
    """Tables copied out of the packed buffer read the same, and every table equals its count == 1 build."""
    rng = random.Random(5)
    streams = gen_units(rng, oracle)[:5]
    got, ref = check_build(streams)
    moved = [np.frombuffer(got.table(u).tobytes(), dtype=np.uint8).copy() for u in range(len(streams))]
    ranges = [(u, lo, n) for u, (_, d) in enumerate(ref) for lo, n in boundary_ranges(len(d or b""), rng, 4)]
    rc, a = read([(got.srcs[u], got.table(u)) for u in range(len(streams))], ranges)
    rc2, b = read([(got.srcs[u], moved[u]) for u in range(len(streams))], ranges)
    assert rc == rc2 == 0 and a == b


def test_call_checks_write_nothing(oracle):
    L = tlib()
    f = L.emu_raw_table_build_batch_scratch_bytes
    assert f(5, 0) < f(5, 1 << 20) < f(9, 1 << 20)
    assert L.emu_raw_table_bytes(3) == HEAD + 3 * REC
    assert L.emu_raw_table_batch_bytes(3, 30720) == 3 * HEAD + (10 + 3) * REC
    streams = [oracle.compress(b"ab" * 70000), b"\x00"]
    assert build(streams, tables_short=1)[0] == INVALID
    assert build(streams, scratch_short=1)[0] == INVALID
    assert build([])[0] == 0
    b = emu.SbBatch()
    lens = np.zeros(4, dtype=np.uint32)
    b.in_lens, b.count = lens.ctypes.data, 1
    bufs = [np.zeros(1 << 20, dtype=np.uint8) for _ in range(4)]       # tables, offsets, results, scratch
    t, o, r, s = (x.ctypes.data for x in bufs)

    def call(bb=C.byref(b), t=t, o=o, r=r, s=s):
        return L.emu_raw_table_build_batch(bb, 0, t, 1 << 12, o, r, s, 1 << 20, 0)
    assert call() == 0
    assert tuple(bufs[1][:16].view(np.uint64)) == (0, HEAD)
    for kw in ({"bb": None}, {"t": None}, {"o": None}, {"r": None}, {"s": None}):
        for x in bufs:
            x[:] = 0x5C
        assert call(**kw) == INVALID, kw
        assert all((x == 0x5C).all() for x in bufs), kw
    b.count = 1 << 31
    assert call() == INVALID and all((x == 0x5C).all() for x in bufs)
    # the read's checks
    rc, got = build(streams)
    units = [(got.srcs[u], got.table(u)) for u in range(2)]
    assert read(units, [(0, 0, 10)], scratch_short=1)[0] == INVALID
    assert read(units, [])[0] == 0
