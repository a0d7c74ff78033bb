"""K8 raw-stream split LOGIC on CPU: the kernel bodies of rust-snappy_b200/csrc/k8_raw_split.cuh (header, canonical
chains, merge, stitch, counts, scan, cuts, block decode, one-warp fallback) compiled by g++ against the fiber warp
emulator (tests/emu) and compared with the oracle: the cut table against the compressed lengths of each 64 KB slice,
the decoded bytes and errors against the oracle's. Test tooling only, like tests/test_frame_index_emu.py."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import emu_helpers as emu
from conftest import corpus

SEG_MIN = 128 << 10
BLOCK = 65536

_HERE = os.path.dirname(os.path.abspath(__file__))
_EMU = os.path.join(_HERE, "emu")
_SO = os.path.join(_EMU, "_build", "libemu_raw_split.so")
_k8 = None


def k8lib():
    """The emulator build of K8 (tests/emu/emu_raw_split.cpp), rebuilt when a source is newer; its own library next to
    libemu_kernels.so, -Bsymbolic keeps each bound to its own emulator copy."""
    global _k8
    if _k8 is None:
        csrc = os.path.join(os.path.dirname(_HERE), "rust-snappy_b200", "csrc")
        srcs = [os.path.join(_EMU, f) for f in ("emu_raw_split.cpp", "simt_emu.cpp", "simt_emu.h")]
        srcs += [os.path.join(csrc, f) for f in os.listdir(csrc)]
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            tmp = "%s.%d.tmp" % (_SO, os.getpid())
            subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unused-function",
                                   "-Wno-unknown-pragmas", "-Wl,-Bsymbolic", "-o", tmp,
                                   os.path.join(_EMU, "emu_raw_split.cpp"), os.path.join(_EMU, "simt_emu.cpp")])
            os.replace(tmp, _SO)
        _k8 = C.CDLL(_SO)
    return _k8


def raw_decode(stream, cap, seg=SEG_MIN):
    """sb_decompress_device_ws under the emulator: (status tuple, bytes, nchunks, cut table, split declined)."""
    n = len(stream)
    src = np.frombuffer(bytes(stream) + b"\0" * 16, dtype=np.uint8).copy()
    out = np.full(cap + 16, 0xEE, dtype=np.uint8)
    res = emu.SbFrameResult()
    cuts = np.zeros(BLOCK + 1, dtype=np.uint32)
    declined = C.c_uint32(7)
    seg_out = C.c_uint64(0)
    k8lib().emu_raw_decode(C.c_void_p(src.ctypes.data), C.c_uint64(n), C.c_void_p(out.ctypes.data), C.c_uint64(cap),
                           C.byref(res), C.c_uint64(seg), C.c_void_p(cuts.ctypes.data), C.byref(declined), C.byref(seg_out))
    assert seg_out.value == max(seg, SEG_MIN)
    assert bytes(out[cap:cap + 16]) == b"\xee" * 16
    e = res.status
    status = (emu.ERR.get(e.code, str(e.code)), e.a, e.b, e.c)
    assert res.bytes == (0 if e.code else res.bytes)
    return status, bytes(out[:res.bytes]), res.nchunks, [int(x) for x in cuts], declined.value


def varint(v):
    out = b""
    while v >= 0x80:
        out += bytes([v & 0x7F | 0x80])
        v >>= 7
    return out + bytes([v])


def oracle_result(oracle, stream, cap):
    from oracle.oracle import OracleError
    try:
        return ("Ok", 0, 0, 0), oracle.decompress(stream, cap)
    except OracleError as e:
        return tuple(e.err), None


def expected_cuts(oracle, data, stream):
    """Cut table of a stream of independent 64 KB blocks: the bodies of each slice compressed alone, concatenated,
    must be the stream's body; the cuts are their cumulative lengths after the header."""
    hl = len(varint(len(data)))
    bodies = []
    for i in range(0, len(data), BLOCK):
        piece = data[i:i + BLOCK]
        c = oracle.compress(piece)
        bodies.append(c[len(varint(len(piece))):])
    assert stream[hl:] == b"".join(bodies)
    cuts = [hl]
    for b in bodies:
        cuts.append(cuts[-1] + len(b))
    return cuts


def check_parallel(stream, data, cuts, seg=SEG_MIN):
    st, out, nchunks, got, declined = raw_decode(stream, len(data), seg)
    B = (len(data) + BLOCK - 1) // BLOCK
    assert st == ("Ok", 0, 0, 0) and declined == 0 and nchunks == B
    assert out == data
    if cuts is not None:
        assert got[:B + 1] == cuts
    return got[:B + 1]


def check_declined(oracle, stream, cap, at_split=True):
    """The verdict is decline (at the split, or at a block's decode) and the result is the oracle's, exactly."""
    want_st, want = oracle_result(oracle, stream, cap)
    st, out, nchunks, _, declined = raw_decode(stream, cap)
    assert nchunks == 0
    if at_split is not None:
        assert declined == (1 if at_split else 0)
    assert st == want_st
    if want is not None:
        assert out == want
    return st


def _tile(b, n):
    return (b * (n // len(b) + 1))[:n]


def _data(kind, n):
    rng = random.Random(n)
    if kind == "text":
        return _tile(corpus("alice29.txt") + corpus("lcet10.txt"), n)
    if kind == "random":
        return bytes(rng.getrandbits(8) for _ in range(n))
    if kind == "zeros":
        return b"\0" * n
    return _tile(corpus(kind), n)


@pytest.mark.parametrize("rem", [1, 65535, 65536])
@pytest.mark.parametrize("kind", ["text", "urls.10K", "geo.protodata", "kppkn.gtb", "fireworks.jpeg", "random", "zeros"])
def test_cut_table_is_exact(oracle, kind, rem):
    blocks = 6 if kind in ("fireworks.jpeg", "random") else 9 if kind != "zeros" else 40
    data = _data(kind, blocks * BLOCK + rem)
    stream = oracle.compress(data)
    check_parallel(stream, data, expected_cuts(oracle, data, stream))


def test_cut_table_of_pyarrow_streams(oracle):
    pa = pytest.importorskip("pyarrow")
    for kind, blocks in (("text", 12), ("fireworks.jpeg", 5), ("kppkn.gtb", 10)):
        data = _data(kind, blocks * BLOCK + 777)
        stream = pa.compress(data, codec="snappy", asbytes=True)
        hl = len(varint(len(data)))
        bodies = [pa.compress(data[i:i + BLOCK], codec="snappy", asbytes=True) for i in range(0, len(data), BLOCK)]
        bodies = [b[len(varint(min(BLOCK, len(data) - i * BLOCK))):] for i, b in enumerate(bodies)]
        assert stream[hl:] == b"".join(bodies)
        cuts = [hl]
        for b in bodies:
            cuts.append(cuts[-1] + len(b))
        check_parallel(stream, data, cuts)


def _lit(b):
    """One literal element of b (1..65536 bytes)."""
    n = len(b) - 1
    if n < 60:
        return bytes([n << 2]) + b
    if n < 256:
        return bytes([60 << 2, n]) + b
    return bytes([61 << 2]) + n.to_bytes(2, "little") + b


def _copy2(length, off):
    return bytes([((length - 1) << 2) | 2]) + off.to_bytes(2, "little")


def _copy4(length, off):
    return bytes([((length - 1) << 2) | 3]) + off.to_bytes(4, "little")


def _two_literal_blocks(rng, firsts):
    """Blocks of two literals each (random bytes), the first of firsts[j] bytes: controls where element starts fall."""
    data, body = b"", b""
    for a in firsts:
        blk = bytes(rng.getrandbits(8) for _ in range(BLOCK))
        body += _lit(blk[:a]) + _lit(blk[a:])
        data += blk
    return data, varint(len(data)) + body


@pytest.mark.parametrize("delta", [-1, 0, 1])
def test_element_starts_around_segment_starts(oracle, delta):
    """A true element start at b_k - 1, b_k and b_k + 1 for the segment starts b_1, b_2, b_3, with 64 KB literals
    crossing the other segment ends."""
    rng = random.Random(delta + 10)
    hl = 3
    firsts, pos, starts = [], hl, []
    for j in range(8):
        target = next((k * SEG_MIN + delta for k in (1, 2, 3) if pos + 260 <= k * SEG_MIN + delta <= pos + 3 + 65535), None)
        a = target - pos - 3 if target is not None else rng.randint(300, 65000)
        firsts.append(a)
        blen = 3 + a + len(_lit(b"x" * (BLOCK - a)))
        starts += [pos, pos + 3 + a]
        pos += blen
    data, stream = _two_literal_blocks(rng, firsts)
    assert len(varint(len(data))) == hl
    for k in (1, 2, 3):
        assert k * SEG_MIN + delta in starts
    cuts = [s for i, s in enumerate(starts) if i % 2 == 0] + [len(stream)]
    check_parallel(stream, data, cuts)


def test_many_segments_of_text(oracle):
    data = _data("text", 31 * BLOCK + 5)
    stream = oracle.compress(data)
    cuts = expected_cuts(oracle, data, stream)
    assert len(stream) > 5 * SEG_MIN
    assert check_parallel(stream, data, cuts) == check_parallel(stream, data, None, seg=3 * SEG_MIN + 32)


def test_copies_into_an_earlier_block_decline(oracle):
    rng = random.Random(3)
    head = bytes(rng.getrandbits(8) for _ in range(BLOCK))
    blk0 = _lit(head)
    # copy-4 whose offset reaches into block 0 (valid in the whole stream, not in its block)
    far = blk0 + _lit(head[:10000]) + _copy4(40, 70000)
    want = head + head[:10000] + (head + head[:10000])[10000 + BLOCK - 70000:][:40]
    s = varint(len(want)) + far
    assert oracle.decompress(s) == want
    check_declined(oracle, s, len(want), at_split=False)
    # copy-2 with an offset <= 65535 into the previous block, as an encoder without block resets writes
    near = blk0 + _lit(head[:100]) + _copy2(20, 1000)
    s = varint(BLOCK + 120) + near
    check_declined(oracle, s, BLOCK + 120, at_split=False)
    # the far-offset stream of the GPU parity suite: 60-byte literals straddle the first block boundary
    head2 = bytes(rng.getrandbits(8) for _ in range(70000))
    want2 = head2 + head2[:40] + head2[100:131] + head2[65500:65560]
    lits = b"".join(_lit(head2[i:i + 60]) for i in range(0, len(head2), 60))
    s2 = varint(len(want2)) + lits + _copy4(40, 70000) + _copy4(31, 70040 - 100) + _copy4(60, 70071 - 65500)
    assert oracle.decompress(s2) == want2
    check_declined(oracle, s2, len(want2))


def test_straddle_and_long_literal_decline(oracle):
    rng = random.Random(4)
    d = bytes(rng.getrandbits(8) for _ in range(3 * BLOCK))
    straddle = varint(len(d)) + _lit(d[:65500]) + _lit(d[65500:65600]) + _lit(d[65600:2 * BLOCK]) + _lit(d[2 * BLOCK:])
    assert oracle.decompress(straddle) == d
    check_declined(oracle, straddle, len(d))
    big = 140000                                                     # one literal longer than the segment floor
    lit = bytes([62 << 2]) + (big - 1).to_bytes(3, "little") + d[:big]
    s = varint(len(d)) + lit + _lit(d[big:])
    assert oracle.decompress(s) == d
    check_declined(oracle, s, len(d))


def test_parses_that_never_merge_decline(oracle):
    """1-byte literals (00 xx, a hop of 2) behind a 3-byte header: the true starts are odd, every segment start is
    even, and an even parse of the same bytes is also a chain of 2-byte elements, so the two never meet. The hop cap
    declines the stream. One 3-byte copy-2 early on flips the true parity to even: then every segment merges at once,
    and the stream is split."""
    n = 300000
    data = bytes(random.Random(5).choice((0, 0, 1)) for _ in range(n))
    odd = varint(n) + b"".join(b"\x00" + bytes([c]) for c in data)
    assert oracle.decompress(odd) == data
    check_declined(oracle, odd, n)
    flip = varint(n) + b"".join(b"\x00" + bytes([c]) for c in data[:1000]) + _copy2(4, 2) + \
        b"".join(b"\x00" + bytes([c]) for c in data[1004:])
    want = data[:1000] + (data[998:1000] * 2) + data[1004:]
    assert oracle.decompress(flip) == want
    check_parallel(flip, want, None)


def test_corrupt_and_truncated_streams_match_oracle(oracle):
    data = _data("text", 5 * BLOCK + 1234)
    good = oracle.compress(data)
    rng = random.Random(6)
    streams = []
    for _ in range(10):
        b = bytearray(good)
        b[rng.randrange(3, len(b))] ^= 1 << rng.randrange(8)
        streams.append(bytes(b))
    streams += [good[:-1], good[:len(good) // 2], good[:SEG_MIN + 1], good + b"\x00", varint(len(data) + 1) + good[3:],
                varint(len(data) - 1) + good[3:], b"\xff\xff\xff\xff\xff", b""]
    for s in streams:
        want_st, want = oracle_result(oracle, s, len(data) + 8)
        st, out, nchunks, _, _ = raw_decode(s, len(data) + 8)
        assert st == want_st, (st, want_st)
        if want is not None:
            assert out == want
        elif st[0] != "Ok":
            assert nchunks == 0
    # the output buffer is smaller than the header says: the serial path's BufferTooSmall
    st, _, nchunks, _, declined = raw_decode(good, len(data) - 1)
    assert st[:3] == ("BufferTooSmall", len(data) - 1, len(data)) and declined == 1 and nchunks == 0


def test_canonical_parse_restarts_after_an_impossible_element(oracle):
    """Segment 1 starts on the offset byte 0xF8 of a copy-1: read as a tag it is a literal whose 3-byte length is far
    over 64 KB. That parse is dropped and restarted at the next byte, which is the true next element, so the stream is
    still split (the rest of the segment is compressed text, too many elements for the true parse to walk alone)."""
    rng = random.Random(8)
    blk0 = bytes(rng.getrandbits(8) for _ in range(BLOCK))
    hl, A = 3, 131071 - (3 + len(_lit(blk0))) - 3
    b1 = bytes(rng.getrandbits(8) for _ in range(A))
    tail = bytes([7, 9]) + bytes(rng.getrandbits(8) for _ in range(4))
    body = _lit(blk0) + _lit(b1) + bytes([1, 0xF8]) + _lit(tail)
    ref = blk0 + b1
    block1 = b1 + (ref[-248:] * 2)[:4] + tail
    assert len(block1) == BLOCK
    rest = [_data("text", 4 * BLOCK)[i * BLOCK:(i + 1) * BLOCK] for i in range(1, 4)]
    data = blk0 + block1 + b"".join(rest)
    stream = varint(len(data)) + body + b"".join(oracle.compress(r)[3:] for r in rest)
    assert len(varint(len(data))) == hl and stream[SEG_MIN] == 0xF8 and stream[SEG_MIN + 1] == len(tail) - 1 << 2
    assert oracle.decompress(stream) == data
    check_parallel(stream, data, None)
