"""K8 over a batch of raw streams on CPU: the k8b_* kernel bodies of rust-snappy_b200/csrc/k8_raw_split.cuh (plan,
per-unit views of the single-stream segment steps, stitch per unit, block decode over the global block list, the
one-warp pass) compiled by g++ against the fiber warp emulator and compared with the oracle, unit by unit. Split units
must give the single-stream harness's cut table; every other unit the oracle's exact bytes or error. Test tooling only,
like tests/test_raw_split_emu.py."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import emu_helpers as emu
import test_raw_split_emu as single
from conftest import corpus

SEG_MIN = 128 << 10
BLOCK = 65536
INVALID = 202
GUARD = 512

_HERE = os.path.dirname(os.path.abspath(__file__))
_EMU = os.path.join(_HERE, "emu")
_SO = os.path.join(_EMU, "_build", "libemu_raw_batch.so")
_lib = None


def kblib():
    """The emulator build of K8's batch bodies (tests/emu/emu_raw_batch.cpp), rebuilt when a source is newer."""
    global _lib
    if _lib is None:
        csrc = os.path.join(os.path.dirname(_HERE), "rust-snappy_b200", "csrc")
        srcs = [os.path.join(_EMU, f) for f in ("emu_raw_batch.cpp", "simt_emu.cpp", "simt_emu.h")]
        srcs += [os.path.join(csrc, f) for f in os.listdir(csrc)]
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            tmp = "%s.%d.tmp" % (_SO, os.getpid())
            subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unused-function",
                                   "-Wno-unknown-pragmas", "-Wl,-Bsymbolic", "-o", tmp,
                                   os.path.join(_EMU, "emu_raw_batch.cpp"), os.path.join(_EMU, "simt_emu.cpp")])
            os.replace(tmp, _SO)
        _lib = C.CDLL(_SO)
        _lib.emu_raw_batch_scratch_bytes.restype = C.c_uint64
        _lib.emu_raw_batch_scratch_bytes.argtypes = [C.c_uint32, C.c_uint64]
    return _lib


def run_batch(streams, caps, addressing="ptrs", in_bytes=None, seg=SEG_MIN):
    """sb_decompress_batch_device_ws under the emulator. addressing "ptrs": in_ptrs/out_ptrs at odd addresses;
    "base": in_base/out_base with odd strides. Returns [(status, bytes)], unit_blocks, [cut table of unit i]."""
    n = len(streams)
    if in_bytes is None:
        in_bytes = sum(len(s) for s in streams)
    if addressing == "ptrs":
        ioffs, at = [], 1
        for s in streams:
            ioffs.append(at)
            at += len(s) + 3 + (at + len(s)) % 2                  # odd starts, units back to back with small gaps
        inbuf = np.zeros(at + 16, dtype=np.uint8)
        ooffs, oat = [], 3
        for c in caps:
            ooffs.append(oat)
            oat += c + 16 + 1 - (c % 2)
        in_stride = out_stride = 0
    else:
        in_stride = max([len(s) for s in streams] + [1]) | 1
        out_stride = (max(caps + [1]) + 16) | 1
        ioffs = [1 + i * in_stride for i in range(n)]
        ooffs = [3 + i * out_stride for i in range(n)]
        inbuf = np.zeros(1 + n * in_stride + 16, dtype=np.uint8)
        oat = 3 + n * out_stride + 16
    for o, s in zip(ioffs, streams):
        inbuf[o:o + len(s)] = np.frombuffer(s, dtype=np.uint8)
    out = np.full(oat + 16, 0xEE, dtype=np.uint8)
    lens = np.array([len(s) for s in streams] + [0], dtype=np.uint32)
    ocaps = np.array(caps + [0], dtype=np.uint32)
    in_ptrs = np.array([inbuf.ctypes.data + o for o in ioffs] + [0], dtype=np.uint64)
    out_ptrs = np.array([out.ctypes.data + o for o in ooffs] + [0], dtype=np.uint64)
    out_lens = np.full(n + 1, 0xDEADBEEF, dtype=np.uint32)
    st = (emu.SbError * max(n, 1))()
    blocks = np.full(n + 1, 0xDEADBEEF, dtype=np.uint32)
    b = emu.SbBatch()
    if addressing == "ptrs":
        b.in_ptrs, b.out_ptrs = in_ptrs.ctypes.data, out_ptrs.ctypes.data
    else:
        b.in_base, b.in_stride = inbuf.ctypes.data + 1, in_stride
        b.out_base, b.out_stride = out.ctypes.data + 3, out_stride
    b.in_lens, b.out_caps = lens.ctypes.data, ocaps.ctypes.data
    b.out_lens, b.statuses, b.count = out_lens.ctypes.data, C.addressof(st), n
    L = kblib()
    size = L.emu_raw_batch_scratch_bytes(n, in_bytes)
    scratch = np.full(size + GUARD, 0xCD, dtype=np.uint8)
    cuts_cap = (size - 256) // 4
    cut_at = np.zeros(max(n, 1), dtype=np.uint64)
    cuts = np.zeros(cuts_cap, dtype=np.uint32)
    rc = L.emu_raw_batch_decode(C.byref(b), C.c_uint64(in_bytes), C.c_void_p(blocks.ctypes.data),
                                C.c_void_p(scratch.ctypes.data), C.c_uint64(size), C.c_uint64(seg),
                                C.c_void_p(cut_at.ctypes.data), C.c_void_p(cuts.ctypes.data), C.c_uint64(cuts_cap))
    assert rc == 0
    assert bytes(scratch[size:]) == b"\xcd" * GUARD                 # nothing written past the scratch
    assert int(out_lens[n]) == 0xDEADBEEF and int(blocks[n]) == 0xDEADBEEF
    res, tables = [], []
    for i in range(n):
        e = st[i]
        status = (emu.ERR.get(e.code, str(e.code)), e.a, e.b, e.c)
        o = ooffs[i]
        assert bytes(out[o + caps[i]:o + caps[i] + 16]) == b"\xee" * 16, i
        res.append((status, bytes(out[o:o + int(out_lens[i])]) if e.code == 0 else None))
        nb = int(blocks[i])
        tables.append([int(x) for x in cuts[int(cut_at[i]):int(cut_at[i]) + nb + 1]] if nb else None)
    return res, [int(x) for x in blocks[:n]], tables


def oracle_result(oracle, stream, cap):
    st, want = single.oracle_result(oracle, stream, cap)
    return st, want


def check_batch(oracle, streams, caps, split, addressing="ptrs", either=(), **kw):
    """Every unit equals the oracle decoding it alone; units in `split` (indices) were split, with the single-stream
    harness's cut table, and every other unit took the one-warp path -- except those in `either` (a bit flip in a
    literal leaves a clean stream, which may be split)."""
    res, blocks, tables = run_batch(streams, caps, addressing, **kw)
    for i, (s, cap) in enumerate(zip(streams, caps)):
        want_st, want = oracle_result(oracle, s, cap)
        assert res[i][0] == want_st, (i, res[i][0], want_st)
        if want is not None:
            assert res[i][1] == want, i
        if i in split or (i in either and blocks[i]):
            assert blocks[i] == (len(want) + BLOCK - 1) // BLOCK, (i, blocks[i])
            _, _, nchunks, cuts, declined = single.raw_decode(s, cap)
            assert declined == 0 and nchunks == blocks[i]
            assert tables[i] == cuts[:blocks[i] + 1], i
        else:
            assert blocks[i] == 0, (i, blocks[i])
    return res, blocks


def _clean_units(oracle):
    """Multi-block streams of every kind with remainders 1, 65535 and 65536 (split), plus single-block units."""
    units = []
    for kind in ("text", "urls.10K", "geo.protodata", "kppkn.gtb", "fireworks.jpeg", "random", "zeros"):
        for rem in (1, 65535, 65536):
            data = single._data(kind, (3 if kind != "zeros" else 5) * BLOCK + rem)
            units.append(oracle.compress(data))
    return units


def _small_units(oracle):
    return [b"", b"\x00", b"\xff\xff\xff\xff\xff", oracle.compress(corpus("alice29.txt")[:1000]),
            oracle.compress(single._data("text", BLOCK)), oracle.compress(b"")]


def _declined_units():
    rng = random.Random(3)
    head = bytes(rng.getrandbits(8) for _ in range(BLOCK))
    blk0 = single._lit(head)
    far_want = head + head[:10000] + (head + head[:10000])[10000 + BLOCK - 70000:][:40]
    far = single.varint(len(far_want)) + blk0 + single._lit(head[:10000]) + single._copy4(40, 70000)
    near = single.varint(BLOCK + 120) + blk0 + single._lit(head[:100]) + single._copy2(20, 1000)
    d = bytes(rng.getrandbits(8) for _ in range(3 * BLOCK))
    straddle = single.varint(len(d)) + single._lit(d[:65500]) + single._lit(d[65500:65600]) + \
        single._lit(d[65600:2 * BLOCK]) + single._lit(d[2 * BLOCK:])
    big = 140000
    longlit = single.varint(len(d)) + bytes([62 << 2]) + (big - 1).to_bytes(3, "little") + d[:big] + single._lit(d[big:])
    n = 300000
    pdata = bytes(random.Random(5).choice((0, 0, 1)) for _ in range(n))
    parity = single.varint(n) + b"".join(b"\x00" + bytes([c]) for c in pdata)
    return [far, near, straddle, longlit, parity]


def _corrupt_units(oracle):
    good = oracle.compress(single._data("text", 3 * BLOCK + 1234))
    rng = random.Random(6)
    out = []
    for _ in range(4):
        b = bytearray(good)
        b[rng.randrange(3, len(b))] ^= 1 << rng.randrange(8)
        out.append(bytes(b))
    out += [good[:-1], good[:len(good) // 2], good + b"\x00", single.varint(3 * BLOCK + 1235) + good[3:]]
    return out


def _cap(oracle, s):
    """The header's length when it is a sane one, else room for a few blocks."""
    from oracle.oracle import OracleError
    try:
        v = oracle.decompress_len(s)
    except OracleError:
        v = None
    return v if v is not None and v <= 1 << 22 else 4 * BLOCK + 4096


@pytest.mark.parametrize("addressing", ["ptrs", "base"])
def test_mixed_batch_matches_oracle(oracle, addressing):
    clean = _clean_units(oracle)
    streams = _small_units(oracle) + clean + _declined_units() + _corrupt_units(oracle)
    caps = [_cap(oracle, s) for s in streams]
    first = len(_small_units(oracle))
    flips = len(streams) - len(_corrupt_units(oracle))
    check_batch(oracle, streams, caps, set(range(first, first + len(clean))), addressing, either=range(flips, flips + 4))


def test_pyarrow_units(oracle):
    pa = pytest.importorskip("pyarrow")
    streams = []
    for kind, blocks in (("text", 4), ("fireworks.jpeg", 3), ("kppkn.gtb", 5)):
        streams.append(pa.compress(single._data(kind, blocks * BLOCK + 777), codec="snappy", asbytes=True))
    streams.append(oracle.compress(b"x" * 100))
    caps = [_cap(oracle, s) for s in streams]
    check_batch(oracle, streams, caps, {0, 1, 2})


def test_results_do_not_depend_on_unit_order(oracle):
    streams = _small_units(oracle)[:4] + _clean_units(oracle)[::4] + _declined_units()[:3] + _corrupt_units(oracle)[:3]
    caps = [_cap(oracle, s) for s in streams]
    res, blocks, _ = run_batch(streams, caps)
    perm = list(range(len(streams)))
    random.Random(9).shuffle(perm)
    res2, blocks2, _ = run_batch([streams[i] for i in perm], [caps[i] for i in perm], "base")
    for k, i in enumerate(perm):
        assert res2[k] == res[i] and blocks2[k] == blocks[i], (k, i)


def test_adjacent_units_of_many_segments(oracle):
    """Units of 5+ segments each at the 128 KiB floor, back to back, among small ones; and the same at a longer
    segment length."""
    streams, split = [], set()
    for j, kind in enumerate(("text", "kppkn.gtb", "text")):
        data = single._data(kind, (31 + j) * BLOCK + 5 + j)
        s = oracle.compress(data)
        assert len(s) > 3 * SEG_MIN
        split.add(len(streams))
        streams.append(s)
        streams.append(oracle.compress(data[:300 + j]))
    caps = [_cap(oracle, s) for s in streams]
    check_batch(oracle, streams, caps, split)
    res, blocks, tables = run_batch(streams, caps, seg=3 * SEG_MIN + 32)
    res0, blocks0, tables0 = run_batch(streams, caps)
    assert (res, blocks, tables) == (res0, blocks0, tables0)


def test_canonical_restart_and_segment_edges(oracle):
    """The single-stream edge streams (element starts at b_k - 1, b_k, b_k + 1) next to each other in one batch."""
    streams, split = [], set()
    for delta in (-1, 0, 1):
        rng = random.Random(delta + 10)
        hl, pos, firsts = 3, 3, []
        for j in range(8):
            target = next((k * SEG_MIN + delta for k in (1, 2, 3) if pos + 260 <= k * SEG_MIN + delta <= pos + 3 + 65535), None)
            a = target - pos - 3 if target is not None else rng.randint(300, 65000)
            firsts.append(a)
            pos += 3 + a + len(single._lit(b"x" * (BLOCK - a)))
        _, stream = single._two_literal_blocks(rng, firsts)
        assert len(single.varint(8 * BLOCK)) == hl
        split.add(len(streams))
        streams.append(stream)
    caps = [_cap(oracle, s) for s in streams]
    check_batch(oracle, streams, caps, split)


def test_inflated_header_takes_the_one_warp_path(oracle):
    """A header announcing more output than the body can encode (over 64 bytes per 3 compressed bytes) is not split,
    whatever the cap, and gets the oracle's exact error; a unit just under the bound is split."""
    good = oracle.compress(single._data("text", 3 * BLOCK + 9))
    body = good[3:]
    dn = len(body) * 64 // 3 + 1
    inflated = single.varint(dn) + body
    streams = [inflated, good]
    caps = [dn, 3 * BLOCK + 9]
    res, blocks, _ = run_batch(streams, caps)
    assert blocks == [0, 4]
    want_st, _ = oracle_result(oracle, inflated, dn)
    assert want_st[0] != "Ok" and res[0][0] == want_st


def test_lengths_over_in_bytes_take_the_one_warp_path(oracle):
    streams = _clean_units(oracle)[:6] + _small_units(oracle)[:3]
    caps = [_cap(oracle, s) for s in streams]
    total = sum(len(s) for s in streams)
    res, blocks, _ = run_batch(streams, caps, in_bytes=total - 1)
    assert blocks == [0] * len(streams)
    for i, s in enumerate(streams):
        want_st, want = oracle_result(oracle, s, caps[i])
        assert res[i][0] == want_st and (want is None or res[i][1] == want)
    _, blocks, _ = run_batch(streams, caps, in_bytes=total)
    assert blocks[:6] == [(_cap(oracle, s) + BLOCK - 1) // BLOCK for s in streams[:6]]


def test_empty_batch_and_short_scratch():
    L = kblib()
    b = emu.SbBatch()
    lens = np.zeros(1, dtype=np.uint32)
    b.out_lens, b.count = lens.ctypes.data, 0
    scratch = np.zeros(4096, dtype=np.uint8)
    size = L.emu_raw_batch_scratch_bytes(0, 0)
    assert L.emu_raw_batch_decode(C.byref(b), C.c_uint64(0), None, C.c_void_p(scratch.ctypes.data), C.c_uint64(size),
                                  C.c_uint64(0), None, None, C.c_uint64(0)) == 0
    b.count = 3
    size = L.emu_raw_batch_scratch_bytes(3, 1 << 20)
    assert size > L.emu_raw_batch_scratch_bytes(3, 1 << 10) > L.emu_raw_batch_scratch_bytes(0, 1 << 10)
    assert L.emu_raw_batch_decode(C.byref(b), C.c_uint64(1 << 20), None, C.c_void_p(scratch.ctypes.data),
                                  C.c_uint64(size - 1), C.c_uint64(0), None, None, C.c_uint64(0)) == INVALID
