"""Raw compress of a batch of units of any length on CPU: the k9_* kernel bodies of
rust-snappy_b200/csrc/k9_raw_batch_compress.cuh (plan, slot scan, fill, K1 over every block of the batch, body scan,
gather, finish) compiled by g++ against the fiber warp emulator. Every unit must equal the oracle's
Encoder::compress byte for byte, or carry its exact error; nothing may be written past a unit's cap or the scratch.
Test tooling only, like tests/test_raw_batch_split_emu.py."""
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
MAX_OK = 3_681_400_511                 # the largest n with max_compress_len(n) != 0

_HERE = os.path.dirname(os.path.abspath(__file__))
_EMU = os.path.join(_HERE, "emu")
_SO = os.path.join(_EMU, "_build", "libemu_raw_batch_compress.so")
_lib = None


def kclib():
    """The emulator build of K9's bodies (tests/emu/emu_raw_batch_compress.cpp), rebuilt when a source is newer."""
    global _lib
    if _lib is None:
        csrc = os.path.join(os.path.dirname(_HERE), "rust-snappy_b200", "csrc")
        srcs = [os.path.join(_EMU, f) for f in ("emu_raw_batch_compress.cpp", "simt_emu.cpp", "simt_emu.h")]
        srcs += [os.path.join(csrc, f) for f in os.listdir(csrc)]
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            tmp = "%s.%d.tmp" % (_SO, os.getpid())
            subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unused-function",
                                   "-Wno-unknown-pragmas", "-Wl,-Bsymbolic", "-o", tmp,
                                   os.path.join(_EMU, "emu_raw_batch_compress.cpp"), os.path.join(_EMU, "simt_emu.cpp")])
            os.replace(tmp, _SO)
        _lib = C.CDLL(_SO)
        _lib.emu_raw_compress_scratch_bytes.restype = C.c_uint64
        _lib.emu_raw_compress_scratch_bytes.argtypes = [C.c_uint32, C.c_uint64]
    return _lib


def max_compress_len(n):
    m = 32 + n + n // 6
    return 0 if m > 0xFFFFFFFF else m


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
        self.cap = max_compress_len(self.n) if cap is None else cap
        self.room = self.cap if self.cap <= 1 << 24 else 64      # bytes really behind the output (a rejected unit's cap is a claim)


def expected(oracle, u):
    need = max_compress_len(u.n)
    if need == 0:
        return ("TooBig", u.n, 0xFFFFFFFF), None
    if u.cap < need:
        return ("BufferTooSmall", u.cap, need), None
    return ("Ok", 0, 0), oracle.compress(u.data)


def multi_bytes(units):
    """The in_bytes a caller passes: Σ n over the units of more than 65,536 bytes that pass the reference's checks."""
    return sum(u.n for u in units if u.n > BLOCK and 0 < max_compress_len(u.n) <= u.cap)


def run_batch(units, addressing="ptrs", in_bytes=None, scratch_short=0, uniform=False):
    """sb_compress_batch_device_ws under the emulator. addressing "ptrs": in_ptrs/out_ptrs at odd addresses; "base":
    in_base/out_base with odd strides. uniform: in_len_uniform / out_cap_uniform (every unit the same length and cap).
    Returns rc and [(status, bytes)]; checks the guard bytes after every cap and after the scratch."""
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
    size = L.emu_raw_compress_scratch_bytes(n, in_bytes)
    scratch = np.full(size + GUARD, 0xCD, dtype=np.uint8)
    rc = L.emu_raw_batch_compress(C.byref(b), C.c_uint64(in_bytes), C.c_void_p(scratch.ctypes.data),
                                  C.c_uint64(size - scratch_short))
    if rc:
        assert (out_lens == 0xDEADBEEF).all() and (out == 0xEE).all()
        return rc, None
    assert bytes(scratch[size:]) == b"\xcd" * GUARD                    # nothing written past the scratch
    assert int(out_lens[n]) == 0xDEADBEEF
    res = []
    for i, u in enumerate(units):
        e, o, k = st[i], ooffs[i], int(out_lens[i])
        assert bytes(out[o + u.room:o + u.room + 16]) == b"\xee" * 16, i   # nothing written past the cap
        status = (emu.ERR.get(e.code, str(e.code)), e.a, e.b)
        if e.code:
            assert k == 0 and (out[o:o + u.room] == 0xEE).all(), i      # a skipped unit's output is not touched
            res.append((status, None))
        else:
            assert 1 <= k <= u.cap, i
            res.append((status, bytes(out[o:o + k])))
    return 0, res


def check(oracle, units, **kw):
    rc, res = run_batch(units, **kw)
    assert rc == 0
    for i, u in enumerate(units):
        want = expected(oracle, u)
        assert res[i][0] == want[0], (i, u.n, res[i][0], want[0])
        assert res[i][1] == want[1], (i, u.n)
    return res


CORPUS = ("alice29.txt", "lcet10.txt", "urls.10K", "kppkn.gtb", "fireworks.jpeg", "geo.protodata", "html_x_4")
EDGE_LENGTHS = (0, 1, 16, 17, BLOCK - 1, BLOCK, BLOCK + 1, BLOCK + 16, BLOCK + 17, 2 * BLOCK, 3 * BLOCK + 1)


def mixed_units():
    units = [Unit(_text(n, i)) for i, n in enumerate(EDGE_LENGTHS)]
    units += [Unit(corpus(name)) for name in CORPUS]
    units += [Unit(_random(2 * BLOCK + 999, 1)), Unit(bytes(3 * BLOCK + 5)), Unit(_random(700, 2)), Unit(bytes(BLOCK))]
    for n in (5 * BLOCK + 3, BLOCK + 1, BLOCK, 100, 0):
        units.append(Unit(_text(n, 9), cap=max_compress_len(n) - 1))
    # rejected units announce their length only: they are never read
    units.append(Unit(b"", n=MAX_OK + 1, cap=0xFFFFFFFF))
    units.append(Unit(b"", n=0xFFFFFFFF, cap=0))
    units.append(Unit(b"", n=MAX_OK, cap=max_compress_len(MAX_OK) - 1))
    return units


@pytest.mark.parametrize("addressing", ["ptrs", "base"])
def test_mixed_batch_matches_oracle(oracle, addressing):
    units = mixed_units()
    assert max_compress_len(MAX_OK) == 4_294_967_294 and max_compress_len(MAX_OK + 1) == 0
    res = check(oracle, units, addressing=addressing)
    assert sum(r[0][0] == "Ok" for r in res) == len(units) - 8


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
        assert res[i] == expected(oracle, u), i


@pytest.mark.parametrize("addressing", ["ptrs", "base"])
def test_uniform_length_over_64k(oracle, addressing):
    n = 3 * BLOCK + 4097
    units = [Unit(_text(n, s)) for s in range(3)] + [Unit(_random(n, 7))]
    check(oracle, units, addressing=addressing, uniform=True)


def test_lengths_over_in_bytes(oracle):
    """Multi-block units whose lengths sum to more than in_bytes are SB_E_INVALID{sum, in_bytes}, untouched; single-block
    units are still compressed; rejected units do not count towards the sum."""
    units = [Unit(_text(2 * BLOCK + 5, 1)), Unit(_text(500, 2)), Unit(_text(3 * BLOCK, 3)), Unit(_text(BLOCK, 4)),
             Unit(b"", n=MAX_OK + 1, cap=0xFFFFFFFF), Unit(b"")]
    total = multi_bytes(units)
    assert total == 5 * BLOCK + 5
    rc, res = run_batch(units, in_bytes=total - 1)
    assert rc == 0
    for i, u in enumerate(units):
        if u.n > BLOCK and u.n < MAX_OK:
            assert res[i] == (("202", total, total - 1), None), i
        else:
            assert res[i] == expected(oracle, u), i
    check(oracle, units, in_bytes=total)


def test_scratch_bound_and_call_checks():
    L = kclib()
    f = L.emu_raw_compress_scratch_bytes
    assert f(5, 0) < f(5, BLOCK + 1) < f(5, 3 * BLOCK + 3)
    # slots of 76,544 bytes: floor(in / 65536) + min(count, floor(in / 65537)), beside a few arrays per slot
    for count, in_bytes, slots in ((5, 10 * BLOCK, 15), (1, 10 * BLOCK + 9, 11), (20, 10 * BLOCK, 19), (20, BLOCK + 1, 2),
                                   (20, BLOCK, 1), (3, 7 * (BLOCK + 1), 10)):
        extra = f(count, in_bytes) - f(count, 0)
        assert slots * 76544 <= extra < slots * (76544 + 64) + 2048, (count, in_bytes)
    assert f(0xFFFFFFFF >> 1, 1 << 48) == 2 ** 64 - 1                   # more blocks than one launch takes
    b = emu.SbBatch()
    lens = np.zeros(4, dtype=np.uint32)
    scratch = np.zeros(4096, dtype=np.uint8)
    b.out_lens, b.count = lens.ctypes.data, 0
    assert L.emu_raw_batch_compress(C.byref(b), C.c_uint64(0), C.c_void_p(scratch.ctypes.data), C.c_uint64(0)) == 0
    b.count = 1 << 31
    assert L.emu_raw_batch_compress(C.byref(b), C.c_uint64(0), C.c_void_p(scratch.ctypes.data), C.c_uint64(4096)) == INVALID


def test_scratch_one_byte_short(oracle):
    units = [Unit(_text(2 * BLOCK + 1, 5)), Unit(_text(10, 6))]
    rc, _ = run_batch(units, scratch_short=1)
    assert rc == INVALID
    check(oracle, units)
