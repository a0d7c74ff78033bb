"""Frame encode of a batch of units of any length on CPU: the k10_* kernel bodies of
rust-snappy_b200/csrc/k10_frame_batch_encode.cuh (plan, slot and index scans, fill, K1 in frame mode over every chunk
of the batch, chunk-size scan, gather, finish) compiled by g++ against the fiber warp emulator. Every unit must equal the
oracle's frame_encode byte for byte, or carry its exact error; every index entry must be the offset of the chunk header
the oracle's stream has there; nothing may be written past a unit's cap, its index entries or the scratch.
Test tooling only, like tests/test_raw_batch_compress_emu.py."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import emu_helpers as emu
from conftest import corpus

BLOCK = 65536
INVALID = 202
GUARD = 512
MAX_OK = 3_679_453_184                 # 56,144 chunks: the largest n whose sb_frame_max_len fits a u32 cap
IDX_FILL = 0xA5A5A5A5A5A5A5A5

_HERE = os.path.dirname(os.path.abspath(__file__))
_EMU = os.path.join(_HERE, "emu")
_SO = os.path.join(_EMU, "_build", "libemu_frame_batch_encode.so")
_lib = None


def kclib():
    """The emulator build of K10's bodies (tests/emu/emu_frame_batch_encode.cpp), rebuilt when a source is newer."""
    global _lib
    if _lib is None:
        csrc = os.path.join(os.path.dirname(_HERE), "rust-snappy_b200", "csrc")
        srcs = [os.path.join(_EMU, f) for f in ("emu_frame_batch_encode.cpp", "simt_emu.cpp", "simt_emu.h")]
        srcs += [os.path.join(csrc, f) for f in os.listdir(csrc)]
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            tmp = "%s.%d.tmp" % (_SO, os.getpid())
            subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unused-function",
                                   "-Wno-unknown-pragmas", "-Wl,-Bsymbolic", "-o", tmp,
                                   os.path.join(_EMU, "emu_frame_batch_encode.cpp"), os.path.join(_EMU, "simt_emu.cpp")])
            os.replace(tmp, _SO)
        _lib = C.CDLL(_SO)
        _lib.emu_frame_batch_scratch_bytes.restype = C.c_uint64
        _lib.emu_frame_batch_scratch_bytes.argtypes = [C.c_uint32, C.c_uint64]
    return _lib


def chunks(n):
    return (n + BLOCK - 1) // BLOCK


def frame_max_len(n):
    return 10 + chunks(n) * (8 + 76490)


def _text(n, seed=0):
    base = corpus("alice29.txt") + corpus("lcet10.txt") + corpus("html_x_4")
    k = seed * 7919 % len(base)
    return ((base[k:] + base) * (n // len(base) + 2))[:n]


def _random(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()


class Unit:
    """A unit: its data, the length the batch announces (a rejected unit may announce more than it holds: it is never
    read) and its cap."""

    def __init__(self, data, cap=None, n=None):
        self.data = data
        self.n = len(data) if n is None else n
        self.cap = min(frame_max_len(self.n), 0xFFFFFFFF) if cap is None else cap
        self.room = self.cap if self.cap <= 1 << 24 else 64      # bytes really behind the output (a rejected unit's cap is a claim)


def expected(oracle, u):
    if u.n == 0:
        return ("Ok", 0, 0), b""
    if u.cap < frame_max_len(u.n):
        return ("BufferTooSmall", u.cap, frame_max_len(u.n)), None
    return ("Ok", 0, 0), oracle.frame_encode(u.data)


def chunk_index(stream):
    """The offset of every chunk header of a frame stream, then its length ([0] for the empty stream)."""
    if not stream:
        return [0]
    offs, at = [], 10
    while at < len(stream):
        offs.append(at)
        at += 4 + int.from_bytes(stream[at + 1:at + 4], "little")
    assert at == len(stream)
    return offs + [at]


def multi_bytes(units):
    """The in_bytes a caller passes: Σ n over the units of more than 65,536 bytes that pass the cap check."""
    return sum(u.n for u in units if u.n > BLOCK and u.cap >= frame_max_len(u.n))


def run_batch(units, addressing="ptrs", in_bytes=None, scratch_short=0, uniform=False, index=True):
    """sb_frame_encode_batch_device_ws under the emulator. addressing "ptrs": in_ptrs/out_ptrs at odd addresses; "base":
    in_base/out_base with odd strides. uniform: in_len_uniform / out_cap_uniform. Returns rc and [(status, bytes,
    index entries or None)]; checks the guard bytes after every cap, after the index and after the scratch."""
    n = len(units)
    if in_bytes is None:
        in_bytes = multi_bytes(units)
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
    for i, u in enumerate(units):
        ibase.append(at)
        at += chunks(u.n) + 1
    idx = np.full(at + 4, IDX_FILL, dtype=np.uint64)
    st = (emu.SbError * max(n, 1))()
    b = emu.SbBatch()
    if addressing == "ptrs":
        b.in_ptrs, b.out_ptrs = in_ptrs.ctypes.data, out_ptrs.ctypes.data
    else:
        b.in_base, b.in_stride = inbuf.ctypes.data + 1, in_stride
        b.out_base, b.out_stride = out.ctypes.data + 3, out_stride
    if uniform:
        assert len({u.n for u in units}) == 1 and len({u.cap for u in units}) == 1
        b.in_len_uniform, b.out_cap_uniform = units[0].n, units[0].cap
    else:
        b.in_lens, b.out_caps = lens.ctypes.data, caps.ctypes.data
    b.out_lens, b.statuses, b.count = out_lens.ctypes.data, C.addressof(st), n
    L = kclib()
    size = L.emu_frame_batch_scratch_bytes(n, in_bytes)
    scratch = np.full(size + GUARD, 0xCD, dtype=np.uint8)
    rc = L.emu_frame_batch_encode(C.byref(b), C.c_uint64(in_bytes), C.c_void_p(idx.ctypes.data if index else None),
                                  C.c_void_p(scratch.ctypes.data), C.c_uint64(size - scratch_short))
    if rc:
        assert (out_lens == 0xDEADBEEF).all() and (out == 0xEE).all() and (idx == IDX_FILL).all()
        return rc, None
    assert bytes(scratch[size:]) == b"\xcd" * GUARD                    # nothing written past the scratch
    assert int(out_lens[n]) == 0xDEADBEEF
    assert (idx[len(idx) - 4:] == IDX_FILL).all()                       # nothing written past the last unit's index
    if not index:
        assert (idx == IDX_FILL).all()
    res = []
    for i, u in enumerate(units):
        e, o, k = st[i], ooffs[i], int(out_lens[i])
        assert bytes(out[o + u.room:o + u.room + 16]) == b"\xee" * 16, i   # nothing written past the cap
        status = (emu.ERR.get(e.code, str(e.code)), e.a, e.b)
        ix = [int(x) for x in idx[ibase[i]:ibase[i] + chunks(u.n) + 1]]
        if e.code:
            assert k == 0 and (out[o:o + u.room] == 0xEE).all(), i      # a rejected unit's output is not touched
            assert all(x == IDX_FILL for x in ix), i                    # nor its index entries
            res.append((status, None, None))
        else:
            assert k <= u.cap, i
            if k == 0:
                assert (out[o:o + u.room] == 0xEE).all(), i             # an empty unit writes nothing
            res.append((status, bytes(out[o:o + k]), ix if index else None))
    return 0, res


def check(oracle, units, **kw):
    rc, res = run_batch(units, **kw)
    assert rc == 0
    for i, u in enumerate(units):
        want = expected(oracle, u)
        assert res[i][0] == want[0], (i, u.n, res[i][0], want[0])
        assert res[i][1] == want[1], (i, u.n)
        if want[1] is not None and res[i][2] is not None:
            assert res[i][2] == chunk_index(want[1]), (i, u.n)
    return res


CORPUS = ("alice29.txt", "lcet10.txt", "urls.10K", "kppkn.gtb", "fireworks.jpeg", "geo.protodata", "html_x_4")
EDGE_LENGTHS = (0, 1, BLOCK - 1, BLOCK, BLOCK + 1, 2 * BLOCK, 3 * BLOCK + 1)


def mixed_units():
    units = [Unit(_text(n, i)) for i, n in enumerate(EDGE_LENGTHS)]
    units += [Unit(corpus(name)) for name in CORPUS]
    # random data: every chunk is stored uncompressed, the single chunk over K1's in-place output
    units += [Unit(_random(2 * BLOCK + 999, 1)), Unit(_random(BLOCK, 2)), Unit(_random(700, 3)), Unit(_random(5, 4))]
    units += [Unit(bytes(3 * BLOCK + 5)), Unit(bytes(BLOCK)), Unit(bytes(17))]
    for n in (5 * BLOCK + 3, BLOCK + 1, BLOCK, 100, 1):
        units.append(Unit(_text(n, 9), cap=frame_max_len(n) - 1))
    units.append(Unit(b"", cap=0))                                     # an empty unit needs no room
    # rejected units announce their length only: they are never read
    units.append(Unit(b"", n=MAX_OK + 1, cap=0xFFFFFFFF))
    units.append(Unit(b"", n=0xFFFFFFFF, cap=0))
    units.append(Unit(b"", n=MAX_OK, cap=frame_max_len(MAX_OK) - 1))
    return units


@pytest.mark.parametrize("addressing", ["ptrs", "base"])
def test_mixed_batch_matches_oracle(oracle, addressing):
    units = mixed_units()
    assert frame_max_len(MAX_OK) == 4_294_903_722 and frame_max_len(MAX_OK + 1) > 0xFFFFFFFF
    res = check(oracle, units, addressing=addressing)
    assert sum(r[0][0] == "Ok" for r in res) == len(units) - 8
    # chunk types: the random units are stored, the zero unit compressed but for its 5-byte tail
    kinds = {i: [r[1][k] for k in r[2][:-1]] for i, r in enumerate(res) if r[1]}
    assert kinds[len(EDGE_LENGTHS) + len(CORPUS)] == [1, 1, 1]
    assert kinds[len(EDGE_LENGTHS) + len(CORPUS) + 1] == [1]
    assert kinds[len(EDGE_LENGTHS) + len(CORPUS) + 4] == [0, 0, 0, 1]


def test_without_index(oracle):
    units = [Unit(_text(2 * BLOCK + 3, 1)), Unit(_text(99, 2)), Unit(b""), Unit(_random(BLOCK + 1, 3))]
    check(oracle, units, index=False)


def test_results_do_not_depend_on_unit_order(oracle):
    units = [u for u in mixed_units() if u.n <= 4 * BLOCK]
    units += [Unit(corpus("alice29.txt")), Unit(corpus("geo.protodata"))]
    perm = list(range(len(units)))
    random.Random(4).shuffle(perm)
    _, res = run_batch(units)
    _, res2 = run_batch([units[i] for i in perm], addressing="base")
    for k, i in enumerate(perm):
        assert res2[k] == res[i], (k, i)
    for i, u in enumerate(units):
        want = expected(oracle, u)
        assert res[i][:2] == want, i


def _threshold_data(n, delta, seed):
    """n bytes whose raw compressed length (varint included) is n - n/8 + delta: a repeated byte, then random bytes (one
    compressed byte each). Found by a seeded search over the length of the random tail."""
    from oracle import oracle as o
    target = n - n // 8 + delta
    rng = np.random.default_rng(seed)
    noise = rng.integers(0, 256, n, dtype=np.uint8).tobytes()
    fill = bytes([int(rng.integers(0, 256))]) * n
    make = lambda r: fill[:n - r] + noise[:r]
    lo, hi = 0, n
    while hi - lo > 1:                                                 # the first r whose length reaches target - 40
        mid = (lo + hi) // 2
        if len(o.compress(make(mid))) >= target - 40:
            hi = mid
        else:
            lo = mid
    for r in range(max(0, hi - 64), min(n, hi + 256)):
        d = make(r)
        if len(o.compress(d)) == target:
            return d
    raise AssertionError("no prefix length gives %d bytes" % target)


@pytest.mark.parametrize("n", [4000, BLOCK])
def test_chunk_type_threshold(oracle, n):
    """Chunks that compress to exactly n - n/8 bytes (stored), one byte less (compressed) and one more (stored), as single
    chunks and as chunks of a multi-chunk unit."""
    datas = {d: _threshold_data(n, d, 10 + d) for d in (-1, 0, 1)}
    for d, x in datas.items():
        assert len(oracle.compress(x)) == n - n // 8 + d
    units = [Unit(datas[d]) for d in (-1, 0, 1)]
    if n == BLOCK:
        units.append(Unit(datas[-1] + datas[0] + datas[1] + datas[-1][:77]))
    res = check(oracle, units)
    for i, d in enumerate((-1, 0, 1)):
        assert res[i][1][10] == (0 if d < 0 else 1), d                 # chunk type of the single chunk
    if n == BLOCK:
        r = res[3]
        assert [r[1][k] for k in r[2][:-1]] == [0, 1, 1, 0]


@pytest.mark.parametrize("addressing", ["ptrs", "base"])
def test_uniform_length_over_64k(oracle, addressing):
    n = 3 * BLOCK + 4097
    units = [Unit(_text(n, s)) for s in range(3)] + [Unit(_random(n, 7))]
    check(oracle, units, addressing=addressing, uniform=True)


def test_uniform_length_past_the_largest_cap():
    """n = 3,679,453,185 needs 56,145 chunks: sb_frame_max_len is over any u32 cap, so every unit is BufferTooSmall."""
    n = MAX_OK + 1
    units = [Unit(b"", n=n, cap=0xFFFFFFFF) for _ in range(3)]
    rc, res = run_batch(units, uniform=True, addressing="base", index=False)
    assert rc == 0
    for r in res:
        assert r == (("BufferTooSmall", 0xFFFFFFFF, frame_max_len(n)), None, None)


def test_lengths_over_in_bytes(oracle):
    """Multi-chunk units whose lengths sum to more than in_bytes are SB_E_INVALID{sum, in_bytes}, untouched, their index
    entries unwritten; single-chunk and empty units are still encoded; rejected units do not count towards the sum."""
    units = [Unit(_text(2 * BLOCK + 5, 1)), Unit(_text(500, 2)), Unit(_text(3 * BLOCK, 3)), Unit(_random(BLOCK, 4)),
             Unit(b"", n=MAX_OK + 1, cap=0xFFFFFFFF), Unit(b""), Unit(_text(2 * BLOCK, 5), cap=frame_max_len(2 * BLOCK) - 1)]
    total = multi_bytes(units)
    assert total == 5 * BLOCK + 5
    rc, res = run_batch(units, in_bytes=total - 1)
    assert rc == 0
    for i, u in enumerate(units):
        if u.n > BLOCK and u.cap >= frame_max_len(u.n):
            assert res[i] == (("202", total, total - 1), None, None), i
        else:
            want = expected(oracle, u)
            assert res[i][:2] == want, i
            if want[1] is not None:
                assert res[i][2] == chunk_index(want[1]), i
    check(oracle, units, in_bytes=total)


def test_scratch_bound_and_call_checks():
    L = kclib()
    f = L.emu_frame_batch_scratch_bytes
    assert f(5, 0) < f(5, BLOCK + 1) < f(5, 3 * BLOCK + 3)
    # K9's slots of 76,544 bytes plus a CRC per slot
    for count, in_bytes, slots in ((5, 10 * BLOCK, 15), (1, 10 * BLOCK + 9, 11), (20, 10 * BLOCK, 19), (3, 7 * (BLOCK + 1), 10)):
        extra = f(count, in_bytes) - f(count, 0)
        assert slots * 76544 <= extra < slots * (76544 + 64) + 2048, (count, in_bytes)
    assert f(0xFFFFFFFF >> 1, 1 << 48) == 2 ** 64 - 1                   # more chunks than one launch takes
    b = emu.SbBatch()
    lens = np.zeros(4, dtype=np.uint32)
    scratch = np.zeros(4096, dtype=np.uint8)
    b.out_lens, b.count = lens.ctypes.data, 0
    assert L.emu_frame_batch_encode(C.byref(b), C.c_uint64(0), None, C.c_void_p(scratch.ctypes.data), C.c_uint64(0)) == 0
    b.count = 1 << 31
    assert L.emu_frame_batch_encode(C.byref(b), C.c_uint64(0), None, C.c_void_p(scratch.ctypes.data), C.c_uint64(4096)) == INVALID


def test_scratch_one_byte_short(oracle):
    units = [Unit(_text(2 * BLOCK + 1, 5)), Unit(_text(10, 6))]
    rc, _ = run_batch(units, scratch_short=1)
    assert rc == INVALID
    check(oracle, units)
