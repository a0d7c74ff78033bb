"""Frame decode of a batch of streams on CPU: the k11_* kernel bodies of rust-snappy_b200/csrc/k11_frame_batch_decode.cuh
(plan, K7's survivors and stitch or the caller index's linkage check, walk count and range scan, K7's emit, parse, walk
fill, output scan, decode + CRC, finish) compiled by g++ against the fiber warp emulator with small grids. Every unit's
(status, out_lens, bytes) must equal the emulator's single-stream decode (K5, tests/emu/emu_kernels.cpp) and the
oracle's frame_decode; d_unit_chunks must show which path ran; nothing may be written past a unit's cap or the scratch.
Test tooling only, like tests/test_frame_batch_encode_emu.py."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import emu_helpers as emu
import legal_streams as ls
from conftest import corpus

INVALID = 202
GUARD = 512
SEG = 128 << 10                       # K7's floor: units over 512 KiB span several segments
IDENT = b"\xff\x06\x00\x00sNaPpY"
NAMES = {10: "StreamHeader", 11: "StreamHeaderMismatch", 12: "UnsupportedChunkType", 13: "UnsupportedChunkLength",
         14: "Checksum", 100: "UnexpectedEof", 202: "Invalid"}

_HERE = os.path.dirname(os.path.abspath(__file__))
_EMU = os.path.join(_HERE, "emu")
_SO = os.path.join(_EMU, "_build", "libemu_frame_batch_decode.so")
_lib = None


def kdlib():
    """The emulator build of K11's bodies (tests/emu/emu_frame_batch_decode.cpp), rebuilt when a source is newer."""
    global _lib
    if _lib is None:
        csrc = os.path.join(os.path.dirname(_HERE), "rust-snappy_b200", "csrc")
        srcs = [os.path.join(_EMU, f) for f in ("emu_frame_batch_decode.cpp", "simt_emu.cpp", "simt_emu.h")]
        srcs += [os.path.join(csrc, f) for f in os.listdir(csrc)]
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            tmp = "%s.%d.tmp" % (_SO, os.getpid())
            subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unused-function",
                                   "-Wno-unknown-pragmas", "-Wl,-Bsymbolic", "-o", tmp,
                                   os.path.join(_EMU, "emu_frame_batch_decode.cpp"), os.path.join(_EMU, "simt_emu.cpp")])
            os.replace(tmp, _SO)
        _lib = C.CDLL(_SO)
        _lib.emu_frame_decode_batch_scratch_bytes.restype = C.c_uint64
        _lib.emu_frame_decode_batch_scratch_bytes.argtypes = [C.c_uint32, C.c_uint64, C.c_uint32]
        _lib.emu_frame_decode_batch.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                                C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64]
    return _lib


def _text(n, seed=0):
    base = corpus("alice29.txt") + corpus("lcet10.txt") + corpus("html_x_4")
    k = seed * 7919 % len(base)
    return ((base[k:] + base) * (n // len(base) + 2))[:n]


def _random(n, seed):
    return np.random.default_rng(seed).integers(0, 256, n, dtype=np.uint8).tobytes()


def chain(stream, fragment=False):
    """The header chain of a stream from its first chunk: every header offset, then where the chain ends."""
    pos, offs = (0 if fragment else 10), []
    while pos + 4 <= len(stream):
        offs.append(pos)
        pos += 4 + int.from_bytes(stream[pos + 1:pos + 4], "little")
    return offs + [pos]


def data_chunks(stream, fragment=False):
    """Data chunks (type 0/1) in a clean chain."""
    return sum(1 for o in chain(stream, fragment)[:-1] if stream[o] in (0, 1))


def single(stream, cap, fragment=False):
    """The emulator's single-stream decode (K5) with a chunk table large enough: (status, bytes)."""
    st, out, _ = emu.frame_decode(stream, cap, fragment=fragment, max_chunks=len(stream) // 8 + 16)
    return st, out


def run_batch(streams, caps, flags=0, index=None, index_base=0, max_chunks=None, in_bytes=None, addressing="ptrs",
              uniform=False, scratch_short=0, seg=SEG):
    """sb_frame_decode_batch_device_ws under the emulator. index: per-unit lists for d_chunk_offs (laid out from entry
    index_base on), or None. Returns rc, [(status, bytes)] and d_unit_chunks; checks the guard bytes after every cap and
    after the scratch."""
    n = len(streams)
    if in_bytes is None:
        in_bytes = sum(len(s) for s in streams)
    if max_chunks is None:
        max_chunks = sum(len(s) // 8 + 2 for s in streams)
    if addressing == "ptrs":
        ioffs, at = [], 1
        for s in streams:
            ioffs.append(at)
            at += len(s) + 3 + (at + len(s)) % 2
        ooffs, oat = [], 3
        for c in caps:
            ooffs.append(oat)
            oat += c + 16 + 1 - (c % 2)
        inbuf = np.zeros(at + 16, dtype=np.uint8)
    else:
        in_stride = max([len(s) for s in streams] + [1]) | 1
        out_stride = (max(list(caps) + [1]) + 16) | 1
        ioffs = [1 + i * in_stride for i in range(n)]
        ooffs = [3 + i * out_stride for i in range(n)]
        inbuf = np.zeros(1 + n * in_stride + 16, dtype=np.uint8)
        oat = 3 + n * out_stride
    for o, s in zip(ioffs, streams):
        inbuf[o:o + len(s)] = np.frombuffer(s, dtype=np.uint8)
    out = np.full(oat + 16, 0xEE, dtype=np.uint8)
    lens = np.array([len(s) for s in streams] + [0], dtype=np.uint32)
    capa = np.array(list(caps) + [0], dtype=np.uint32)
    in_ptrs = np.array([inbuf.ctypes.data + o for o in ioffs] + [0], dtype=np.uint64)
    out_ptrs = np.array([out.ctypes.data + o for o in ooffs] + [0], dtype=np.uint64)
    out_lens = np.full(n + 1, 0xDEADBEEF, dtype=np.uint32)
    unit_chunks = np.full(n + 1, 0xDEADBEEF, dtype=np.uint32)
    st = (emu.SbError * max(n, 1))()
    b = emu.SbBatch()
    if addressing == "ptrs":
        b.in_ptrs, b.out_ptrs = in_ptrs.ctypes.data, out_ptrs.ctypes.data
    else:
        b.in_base, b.in_stride = inbuf.ctypes.data + 1, in_stride
        b.out_base, b.out_stride = out.ctypes.data + 3, out_stride
    if uniform:
        assert len({len(s) for s in streams}) == 1 and len(set(caps)) == 1
        b.in_len_uniform, b.out_cap_uniform = len(streams[0]), caps[0]
    else:
        b.in_lens, b.out_caps = lens.ctypes.data, capa.ctypes.data
    b.out_lens, b.statuses, b.count = out_lens.ctypes.data, C.addressof(st), n
    cidx = cat = None
    if index is not None:
        at_list, flat = [], [0xABAB] * index_base
        for ix in index:
            at_list.append(len(flat))
            flat += list(ix)
        at_list.append(len(flat))
        cidx = np.array(flat + [0xCDCD] * 4, dtype=np.uint64)
        cat = np.array(at_list, dtype=np.uint64)
    L = kdlib()
    size = L.emu_frame_decode_batch_scratch_bytes(n, in_bytes, max_chunks)
    scratch = np.full(size + GUARD, 0xCD, dtype=np.uint8)
    rc = L.emu_frame_decode_batch(C.byref(b), in_bytes, flags, cidx.ctypes.data if cidx is not None else None,
                                  cat.ctypes.data if cat is not None else None, max_chunks, unit_chunks.ctypes.data,
                                  scratch.ctypes.data, size - scratch_short, SEG if seg is None else seg)
    if rc:
        assert (out_lens == 0xDEADBEEF).all() and (out == 0xEE).all() and (unit_chunks == 0xDEADBEEF).all()
        return rc, None, None
    assert bytes(scratch[size:]) == b"\xcd" * GUARD                    # nothing written past the scratch
    assert int(out_lens[n]) == 0xDEADBEEF and int(unit_chunks[n]) == 0xDEADBEEF
    res = []
    for i in range(n):
        e, o, k = st[i], ooffs[i], int(out_lens[i])
        assert bytes(out[o + caps[i]:o + caps[i] + 16]) == b"\xee" * 16, i   # nothing written past the cap
        assert k <= caps[i], i
        res.append(((emu.ERR.get(e.code, NAMES.get(e.code, str(e.code))), e.a, e.b, e.c), bytes(out[o:o + k])))
    return 0, res, [int(x) for x in unit_chunks[:n]]


def oracle_decode(oracle, s):
    from oracle.oracle import OracleError
    try:
        return ("Ok", 0, 0, 0), oracle.frame_decode(s)
    except OracleError as e:
        err = e.err
        if err[0] == "StreamHeaderMismatch" and isinstance(err[1], (bytes, bytearray)):
            return (err[0], int.from_bytes(err[1], "little"), 0, 0), None
        return tuple(err), None


def check(oracle, streams, caps=None, flags=0, **kw):
    """Every unit against the single-stream decode, and (whole streams that fit) against the oracle."""
    if caps is None:
        caps = [max(len(single(s, 1 << 22, flags & 1)[1]), 1) + 7 for s in streams]
    rc, res, uc = run_batch(streams, caps, flags=flags, **kw)
    assert rc == 0
    for i, s in enumerate(streams):
        want = single(s, caps[i], flags & 1)
        assert res[i] == want, (i, len(s), res[i][0], want[0])
        if not flags & 1 and want[0][0] != "BufferTooSmall":
            ost, odata = oracle_decode(oracle, s)
            assert res[i][0] == ost, (i, res[i][0], ost)
            if odata is not None:
                assert res[i][1] == odata, i
    return res, uc


def _flip(s, at):
    b = bytearray(s)
    b[at] ^= 0x5A
    return bytes(b)


def mixed_streams(oracle):
    """(stream, clean) pairs: clean streams are a run of data chunks that K7 or a caller index describes."""
    rng = random.Random(11)
    enc = oracle.frame_encode
    big = enc(_text(700_000, 1))                                       # 11 chunks over 6 segments of 128 KiB
    three = enc(_text(3 * 65536 - 100, 2))
    c3 = chain(three)
    units = [
        (b"", False), (IDENT, True), (enc(_text(1000, 3)), True), (big, True), (enc(_random(70000, 4)), True),
        (enc(bytes(5)), True),
        (ls.gen_frame(rng, oracle.crc32c_masked, 12).stream, False),   # padding and skippable chunks: walked
        (ls.gen_frame(rng, oracle.crc32c_masked, 6, kinds=("pad", "skip", "raw")).stream, False),
        (enc(_text(5000, 5)) + enc(_text(300, 6)), False),             # a repeated identifier
        (_flip(three, c3[1] + 5), True),                               # a bad CRC in the middle chunk
        (three[:-5], False),                                           # truncated
        (three + bytes([0x05, 4, 0, 0]) + bytes(4), False),            # a reserved chunk type
        (IDENT[:4] + b"sNaPpZ" + three[10:], False),                   # a wrong identifier
        (_flip(three, c3[2] + 20), True),                              # corrupt compressed data in the last chunk
    ]
    # a compressed chunk whose body ends inside its varint: the parse rejects it, the reader's walk reads the rest of
    # the varint from its persistent buffer (src/read.rs:216)
    for body in (b"\x85", b"\xff\xff", b"\x80\x80\x80", b"\x8a\x01\x00" + bytes(9)):
        s = IDENT + enc(_text(900, 7))[10:] + bytes([0, len(body) + 4, 0, 0]) + (0x1234).to_bytes(4, "little") + body
        units.append((s, True))
    return units


@pytest.mark.parametrize("addressing", ["ptrs", "base"])
def test_mixed_batch_matches_single_stream_and_oracle(oracle, addressing):
    units = mixed_streams(oracle)
    streams = [s for s, _ in units]
    res, uc = check(oracle, streams, addressing=addressing)
    for i, (s, clean) in enumerate(units):
        # K7 indexes every clean stream; the short-varint units are indexed but their parse fails: walked
        parsed = clean and res[i][0][0] not in ("Header",) and i < len(units) - 4
        if parsed:
            assert uc[i] == data_chunks(s), i
        if not clean:
            assert uc[i] == 0, i
    assert sum(1 for x in uc[-4:] if x) == 1                            # only the complete varint parses
    assert res[3][1] == _text(700_000, 1) and res[3][0][0] == "Ok"


def _index_of(s):
    return chain(s) if s else [0]


@pytest.mark.parametrize("base", [0, 5])
def test_caller_index(oracle, base):
    units = mixed_streams(oracle)
    streams = [s for s, _ in units]
    index = [_index_of(s) for s in streams]
    res0, uc0 = check(oracle, streams)
    res, uc = check(oracle, streams, index=index, index_base=base)
    assert res == res0
    for i, (s, clean) in enumerate(units):
        if clean and res[i][0][0] == "Ok":
            assert uc[i] == data_chunks(s), i
    # a padding or skippable chunk inside a linked chain: the parse rejects it and the walk decodes the unit
    assert uc[6] == 0 and uc[7] == 0


def test_wrong_caller_index(oracle):
    enc = oracle.frame_encode
    good = [enc(_text(n, 20 + n % 7)) for n in (70000, 200000, 140000, 30000, 65536 * 3, 9000)]
    ix = [chain(s) for s in good]
    wrong = [list(x) for x in ix]
    wrong[0][1] += 1                                                   # a shifted entry
    wrong[1][-1] -= 1                                                  # a wrong last entry
    del wrong[2][1]                                                    # too few chunks
    wrong[3] = [123456789, 5, 77]                                      # garbage
    wrong[4] = []                                                      # no entries at all
    res0, uc0 = check(oracle, good, index=ix)
    assert uc0 == [data_chunks(s) for s in good]
    res, uc = check(oracle, good, index=wrong)
    assert res == res0
    assert uc == [0, 0, 0, 0, 0, data_chunks(good[5])]


def test_rejected_encoder_unit_index(oracle):
    """A unit the batch encoder rejected leaves its index entries unwritten: garbage, so the unit is walked."""
    s = oracle.frame_encode(_text(150000, 3))
    res, uc = check(oracle, [s, s], index=[[0xA5A5A5A5A5A5A5A5] * 4, chain(s)])
    assert uc == [0, 3] and res[0] == res[1]


def test_fragments(oracle):
    rng = random.Random(5)
    frags = [oracle.frame_encode(_text(n, n))[10:] for n in (1, 65536, 300000)]
    g = ls.gen_frame(rng, oracle.crc32c_masked, 9)
    frags += [b"", g.stream[10:], IDENT + frags[0]]
    res, uc = check(oracle, frags, flags=1)
    assert [r[0][0] for r in res] == ["Ok"] * 6
    assert res[4][1] == g.data
    assert uc[:4] == [1, 1, 5, 0] and uc[4] == 0 and uc[5] == 0
    res2, uc2 = check(oracle, frags, flags=1, index=[chain(f, True) if f else [0] for f in frags])
    assert res2 == res and uc2[:3] == [1, 1, 5]


@pytest.mark.parametrize("indexed", [False, True])
def test_chunk_table_one_short(oracle, indexed):
    enc = oracle.frame_encode
    streams = [enc(_text(n, n)) for n in (100000, 5000, 200000, 70000, 0)] + [enc(_text(10, 1))]
    need = [data_chunks(s) for s in streams]
    assert need == [2, 1, 4, 2, 0, 1]
    index = [_index_of(s) for s in streams] if indexed else None
    caps = [300000] * len(streams)
    for k in (2, 3, 5):
        mc = sum(need[:k + 1]) - 1                                     # unit k is one chunk short
        rc, res, uc = run_batch(streams, caps, index=index, max_chunks=mc)
        assert rc == 0
        for i, s in enumerate(streams):
            if i < k:
                assert res[i] == single(s, caps[i]), (k, i)
            else:
                assert res[i] == (("Invalid", mc, 1, 0), b""), (k, i)
                assert uc[i] == 0
    rc, res, _ = run_batch(streams, caps, index=index, max_chunks=sum(need))
    assert [r[0][0] for r in res] == ["Ok"] * len(streams)


def test_walked_units_take_their_walk_count(oracle):
    """Units K7 declines get the range of their own walk; the first that does not fit and every unit after it fail."""
    rng = random.Random(8)
    gs = [ls.gen_frame(rng, oracle.crc32c_masked, 10) for _ in range(4)]
    streams = [g.stream for g in gs]
    need = [len(chain(s)) - 1 - sum(1 for o in chain(s)[:-1] if s[o] not in (0, 1)) for s in streams]
    caps = [len(g.data) + 3 for g in gs]
    mc = need[0] + need[1] - 1
    rc, res, _ = run_batch(streams, caps, max_chunks=mc)
    assert res[0] == single(streams[0], caps[0])
    assert all(r == (("Invalid", mc, 1, 0), b"") for r in res[1:])
    check(oracle, streams, caps=caps, max_chunks=sum(need))


def test_caps_one_byte_short(oracle):
    enc = oracle.frame_encode
    datas = [_text(n, n) for n in (1, 65536, 65537, 250000)] + [_random(3000, 2)]
    streams = [enc(d) for d in datas]
    caps = [len(d) - 1 for d in datas]
    res, _ = check(oracle, streams, caps=caps)
    for r, d in zip(res, datas):
        assert r == (("BufferTooSmall", len(d) - 1, len(d), 0), b"")
    res, _ = check(oracle, streams, caps=[len(d) for d in datas], index=[chain(s) for s in streams])
    assert [r[1] for r in res] == datas


def test_in_bytes_underestimated(oracle):
    units = mixed_streams(oracle)
    streams = [s for s, _ in units]
    res0, _ = check(oracle, streams)
    res, uc = check(oracle, streams, in_bytes=sum(len(s) for s in streams) - 1)
    assert res == res0 and uc == [0] * len(streams)                   # nothing indexed: every unit walked
    res, _ = check(oracle, streams, in_bytes=0)
    assert res == res0


def test_results_do_not_depend_on_unit_order(oracle):
    streams = [s for s, _ in mixed_streams(oracle)]
    perm = list(range(len(streams)))
    random.Random(4).shuffle(perm)
    res, uc = check(oracle, streams)
    res2, uc2 = check(oracle, [streams[i] for i in perm], addressing="base")
    for k, i in enumerate(perm):
        assert res2[k] == res[i] and uc2[k] == uc[i], (k, i)


@pytest.mark.parametrize("addressing", ["ptrs", "base"])
def test_uniform_lengths_and_caps(oracle, addressing):
    d = [_text(200000, s) for s in range(3)]
    streams = [oracle.frame_encode(x) for x in d]
    n = min(len(s) for s in streams)
    streams = [s[:n] for s in streams]                                 # same length: some are truncated
    res, _ = check(oracle, streams, caps=[200000] * 3, addressing=addressing, uniform=True)
    res2, _ = check(oracle, streams, caps=[200000] * 3, addressing=addressing, uniform=True, seg=0)
    assert res == res2


def test_call_checks_and_scratch():
    L = kdlib()
    f = L.emu_frame_decode_batch_scratch_bytes
    assert f(5, 0, 10) < f(5, 1 << 20, 10) < f(5, 1 << 20, 1000) < f(9, 1 << 20, 1000)
    assert f(5, 1 << 40, 10) == f(5, 1 << 36, 10)                      # bounds above 2^36 count as 2^36
    b = emu.SbBatch()
    lens = np.zeros(4, dtype=np.uint32)
    st = (emu.SbError * 4)()
    scratch = np.zeros(1 << 16, dtype=np.uint8)
    ix = np.zeros(4, dtype=np.uint64)
    sp = scratch.ctypes.data
    b.out_lens, b.statuses, b.count = lens.ctypes.data, C.addressof(st), 0
    call = lambda bb, mc=8, a=None, c=None, s=sp, sz=1 << 16: L.emu_frame_decode_batch(bb, 0, 0, a, c, mc, None, s, sz, 0)
    assert call(C.byref(b)) == 0
    assert call(None) == INVALID
    assert call(C.byref(b), mc=0) == INVALID
    assert call(C.byref(b), mc=(1 << 22) - 1) == INVALID
    assert call(C.byref(b), a=ix.ctypes.data) == INVALID
    assert call(C.byref(b), c=ix.ctypes.data) == INVALID
    assert call(C.byref(b), s=None) == INVALID
    b.count = 1 << 31
    assert call(C.byref(b)) == INVALID
    b.count = 1
    b.statuses = None
    assert call(C.byref(b)) == INVALID
    b.statuses, b.out_lens = C.addressof(st), None
    assert call(C.byref(b)) == INVALID


def test_scratch_one_byte_short(oracle):
    streams = [oracle.frame_encode(_text(n, 3)) for n in (70000, 10)]
    rc, _, _ = run_batch(streams, [80000, 80000], scratch_short=1)
    assert rc == INVALID
    check(oracle, streams)
