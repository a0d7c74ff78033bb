"""K7 chunk indexer LOGIC on CPU: the kernel bodies of rust-snappy_b200/csrc/k7_frame_index.cuh compiled by g++ against
the fiber warp emulator (tests/emu), compared with the chunk header offsets of a Python walk of the stream, and the
decoder's index-first path compared with the oracle. Test tooling only, like tests/test_emu_kernels.py."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import emu_helpers as emu
from conftest import corpus
from kats import RANDOM

NOT_INDEXABLE = 0xFFFFFFFF
IDENT = b"\xff\x06\x00\x00sNaPpY"
SPAN = 4 + 76490                 # most bytes one chunk occupies
SEG_MIN = 128 << 10

_HERE = os.path.dirname(os.path.abspath(__file__))
_EMU = os.path.join(_HERE, "emu")
_SO = os.path.join(_EMU, "_build", "libemu_frame_index.so")
_k7 = None


def k7lib():
    """The emulator build of K7 and the index-first decode (tests/emu/emu_frame_index.cpp), rebuilt when a source
    is newer. Its own library next to libemu_kernels.so; -Bsymbolic keeps each bound to its own emulator copy."""
    global _k7
    if _k7 is None:
        csrc = os.path.join(os.path.dirname(_HERE), "rust-snappy_b200", "csrc")
        srcs = [os.path.join(_EMU, f) for f in ("emu_frame_index.cpp", "simt_emu.cpp", "simt_emu.h")]
        srcs += [os.path.join(csrc, f) for f in os.listdir(csrc)]
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            tmp = "%s.%d.tmp" % (_SO, os.getpid())
            subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unused-function",
                                   "-Wno-unknown-pragmas", "-Wl,-Bsymbolic", "-o", tmp,
                                   os.path.join(_EMU, "emu_frame_index.cpp"), os.path.join(_EMU, "simt_emu.cpp")])
            os.replace(tmp, _SO)
        _k7 = C.CDLL(_SO)
    return _k7


def frame_index(stream, fragment=False, max_chunks=None, seg=0):
    """sb_frame_index_device_ws under the emulator: (count or NOT_INDEXABLE, index list or None, segment length)."""
    n = len(stream)
    src = np.frombuffer(bytes(stream) + b"\0" * 16, dtype=np.uint8).copy()
    maxc = max_chunks if max_chunks is not None else n // 8 + 16
    idx = np.full(maxc + 1, 0xAB, dtype=np.uint64)
    count = np.zeros(1, dtype=np.uint32)
    seg_out = C.c_uint64(0)
    k7lib().emu_frame_index(C.c_void_p(src.ctypes.data), C.c_uint64(n), 1 if fragment else 0, C.c_void_p(idx.ctypes.data),
                            C.c_uint32(maxc), C.c_void_p(count.ctypes.data), C.c_uint64(seg), C.byref(seg_out))
    k = int(count[0])
    return k, (None if k == NOT_INDEXABLE else [int(x) for x in idx[:k + 1]]), seg_out.value


def frame_decode_indexed(stream, cap, fragment=False, max_chunks=None, seg=0):
    """The decoder's no-index path under the emulator (K7 first): (status tuple, produced bytes, need_serial)."""
    n = len(stream)
    src = np.frombuffer(bytes(stream) + b"\0" * 16, dtype=np.uint8).copy()
    out = np.full(cap + 16, 0xEE, dtype=np.uint8)
    res = emu.SbFrameResult()
    maxc = max_chunks if max_chunks is not None else n // 8 + 16
    need = C.c_uint32(7)
    k7lib().emu_frame_decode_indexed(C.c_void_p(src.ctypes.data), C.c_uint64(n), C.c_void_p(out.ctypes.data), C.c_uint64(cap),
                                     1 if fragment else 0, C.byref(res), C.c_uint32(maxc), C.c_uint64(seg), C.byref(need))
    assert bytes(out[cap:cap + 16]) == b"\xee" * 16
    e = res.status
    names = {10: "StreamHeader", 11: "StreamHeaderMismatch", 12: "UnsupportedChunkType", 13: "UnsupportedChunkLength",
             14: "Checksum", 100: "UnexpectedEof", 202: "Invalid"}
    status = (emu.ERR.get(e.code, names.get(e.code, str(e.code))), e.a, e.b, e.c)
    return status, bytes(out[:res.bytes]), need.value


def walk(stream, fragment=False):
    """Offsets of every chunk header of a clean stream, then its length."""
    pos, offs = (0 if fragment else 10), []
    while pos < len(stream):
        offs.append(pos)
        pos += 4 + int.from_bytes(stream[pos + 1:pos + 4], "little")
    assert pos == len(stream)
    return offs + [len(stream)]


def chunk(ty, body, crc=0):
    return bytes([ty]) + (len(body) + 4).to_bytes(3, "little") + crc.to_bytes(4, "little") + body


def rechunk(oracle, pieces):
    """One stream of the chunks of independent frame_encode calls (random-sized writes), identifier once."""
    return IDENT + b"".join(oracle.frame_encode(p)[10:] for p in pieces)


def _frame_err(e):
    name = e[0]
    if name == "StreamHeaderMismatch":
        return (name, int.from_bytes(e[1], "little") if isinstance(e[1], (bytes, bytearray)) else e[1], 0, 0)
    return tuple(e)


def oracle_decode(oracle, s):
    from oracle.oracle import OracleError
    try:
        return ("Ok", 0, 0, 0), oracle.frame_decode(s)
    except OracleError as e:
        return _frame_err(e.err), None


def check_decode(oracle, s, cap=None, need_serial=None, **kw):
    want_st, want = oracle_decode(oracle, s)
    st, out, ns = frame_decode_indexed(s, cap if cap is not None else (len(want) if want is not None else 400000), **kw)
    assert st == want_st, (s[:24], st, want_st)
    if want is not None:
        assert out == want
    if need_serial is not None:
        assert ns == need_serial
    return out


@pytest.mark.parametrize("name,cut", [("alice29.txt", 150000), ("fireworks.jpeg", 70000), ("html", 65536),
                                      ("paper-100k.pdf", None), ("geo.protodata", 1), ("kppkn.gtb", None)])
def test_index_of_encoder_streams(oracle, name, cut):
    data = corpus(name)[:cut] if cut else corpus(name)
    stream, offs, _ = emu.frame_encode(data)
    assert stream == oracle.frame_encode(data)
    k, idx, seg = frame_index(stream)
    assert seg == 256 << 10
    assert idx == offs == walk(stream) and k == len(offs) - 1
    out = check_decode(oracle, stream, need_serial=0)
    assert out == data


def test_index_of_small_and_mixed_chunks(oracle):
    rng = random.Random(5)
    text = corpus("lcet10.txt") + corpus("html")
    pieces, at = [], 0
    while at < 500000:
        ln = rng.choice([rng.randint(1, 300), rng.randint(1, 4096), rng.randint(1, 70000)])
        pieces.append(text[at:at + ln])
        at += ln
    stream = rechunk(oracle, pieces)
    k, idx, _ = frame_index(stream)
    assert idx == walk(stream) and k == len(idx) - 1 >= 40
    assert check_decode(oracle, stream, need_serial=0) == b"".join(pieces)
    # uniformly small chunks: many true headers in every window
    small = rechunk(oracle, [text[i:i + 1000] for i in range(0, 400000, 1000)])
    assert frame_index(small)[1] == walk(small)
    check_decode(oracle, small, need_serial=0)


def test_index_of_incompressible_chunks(oracle):
    rng = random.Random(9)
    data = bytes(rng.getrandbits(8) for _ in range(200000)) + RANDOM[0]
    stream = oracle.frame_encode(data)
    assert stream[10] == 0x01                                        # uncompressed chunk
    assert frame_index(stream)[1] == walk(stream)
    assert check_decode(oracle, stream, need_serial=0) == data


def test_index_of_fragments_and_identifier_alone(oracle):
    data = corpus("alice29.txt")[:140000]
    frag = oracle.frame_encode(data)[10:]
    k, idx, _ = frame_index(frag, fragment=True)
    assert idx == walk(frag, fragment=True) and idx[0] == 0 and k == 3
    st, out, ns = frame_decode_indexed(frag, len(data), fragment=True)
    assert st[0] == "Ok" and out == data and ns == 0
    assert frame_index(frag)[0] == NOT_INDEXABLE                     # no identifier: only as a fragment
    assert frame_index(IDENT) == (0, [10], 256 << 10)
    st, out, ns = frame_decode_indexed(IDENT, 16)
    assert st[0] == "Ok" and out == b"" and ns == 0
    assert frame_index(b"", fragment=True)[:2] == (0, [0])


def _boundary_stream(seed, seg, nseg):
    """Structure-only stream (random bodies) with chunk headers placed at, just after and at the far end of the window
    of segment boundaries b_k = 10 + k*seg."""
    rng = random.Random(seed)
    parts, pos = [IDENT], 10

    def add(size):
        nonlocal pos
        parts.append(chunk(0, bytes(rng.getrandbits(8) for _ in range(size - 8))))
        pos += size

    def fill(target):
        while pos < target:
            gap = target - pos
            size = gap if gap <= SPAN else rng.randint(8, min(SPAN, gap - 8))
            add(size)

    for k in range(1, nseg):
        b = 10 + k * seg
        d = [0, 1, 3, 4, 7, SPAN - 1, 2, 0, 12345, SPAN - 9][k % 10]
        if d == SPAN - 1:
            fill(b - 1)
            add(SPAN)                                                # starts 1 byte before b_k, next header at b_k + 76493
        else:
            fill(b + d)
    fill(10 + nseg * seg - rng.randint(0, 5000))
    return b"".join(parts)


@pytest.mark.parametrize("seed", [1, 2])
def test_index_across_segment_boundaries_at_the_floor(seed):
    s = _boundary_stream(seed, SEG_MIN, 12)
    k, idx, seg = frame_index(s, seg=SEG_MIN)
    assert seg == SEG_MIN
    assert idx == walk(s)
    for k_ in range(1, 11):                                          # headers really sit on the boundaries
        b = 10 + k_ * SEG_MIN
        assert any(b <= o < b + SPAN for o in idx)
    b = [10 + k_ * SEG_MIN for k_ in range(12)]
    assert b[1] + 1 in idx and b[2] + 3 in idx and b[7] in idx and b[10] in idx and b[5] + SPAN - 1 in idx
    # the default segment length on the same stream, and a fragment of it
    assert frame_index(s)[1] == idx
    assert frame_index(s[10:], fragment=True, seg=SEG_MIN)[1] == [o - 10 for o in idx]


def test_segment_length_floor_and_table_fit():
    s = _boundary_stream(3, SEG_MIN, 3)
    assert frame_index(s, seg=1000)[2] == SEG_MIN                    # below the floor: the floor
    assert frame_index(s, seg=SEG_MIN)[1] == walk(s)


def _hostile(rng, nchunks, fake_len, body_len, oracle):
    """Type-0x01 chunks (valid checksums) whose bodies are packed with plausible data-chunk headers."""
    parts = [IDENT]
    for _ in range(nchunks):
        body = bytearray()
        while len(body) < body_len:
            fl = fake_len if fake_len else rng.randint(4, 300)
            body += bytes([rng.choice([0, 1])]) + fl.to_bytes(3, "little") + bytes(rng.getrandbits(8) for _ in range(min(fl, 12)))
            body += b"\0" * max(0, fl - 12)
        body = bytes(body[:body_len])
        parts.append(chunk(1, body, oracle.crc32c_masked(body)))
    return b"".join(parts)


@pytest.mark.parametrize("fake_len,body_len", [(12, 4096), (12, 4093), (60, 65536), (0, 30000), (4, 1000)])
def test_hostile_fake_headers_give_the_exact_index_or_none(oracle, fake_len, body_len):
    rng = random.Random(fake_len * 7 + body_len)
    s = _hostile(rng, max(3, 600000 // (body_len + 8)), fake_len, body_len, oracle)
    for seg in (SEG_MIN, 0):
        k, idx, _ = frame_index(s, seg=seg)
        assert k == NOT_INDEXABLE or idx == walk(s), (k, seg)
    check_decode(oracle, s, seg=SEG_MIN)                             # either path: the oracle's bytes


def test_decode_index_first_matches_oracle_on_malformed_streams(oracle):
    """The malformed streams of the K5 emulator test through the index-first decoder: same status, same bytes before
    the error."""
    data = corpus("alice29.txt")[:150000]
    good = oracle.frame_encode(data)
    flip = bytearray(good); flip[len(good) // 2] ^= 0x10
    crc = bytearray(good); crc[14] ^= 1
    streams = [bytes(flip), bytes(crc), good[:-7], good + b"\x00\x07", IDENT + b"\x02\x00\x00\x00", b"123",
               IDENT + b"\x80\x03\x00\x00xyz" + b"\xfe\x02\x00\x00\x00\x00" + IDENT + good[10:],
               IDENT + b"\x00\x05\x00\x00\x00\x00\x00\x00\x80", IDENT + b"\x01\x03\x00\x00abc", b"\xff\x05\x00\x00sNaPp",
               b"\xff\x06\x00\x00sNaPpZ", IDENT + b"\x00\xff\xff\xff", IDENT + b"\x00\x04\x00\x00\x00\x00\x00\x00", b""]
    for s in streams:
        want_st, want = oracle_decode(oracle, s)
        st, out, _ = frame_decode_indexed(s, 200000)
        assert st == want_st, (s[:20], st, want_st)
        assert out == want if want is not None else data.startswith(out)
    # payload damage keeps a clean structure: indexed, and the error still comes from the chunk decode
    assert frame_index(bytes(flip))[1] == walk(good)
    assert frame_decode_indexed(bytes(flip), 200000)[2] == 0
    st, out, _ = frame_decode_indexed(good, 1000)
    assert st[:3] == ("BufferTooSmall", 1000, len(data)) and out == b""
    st, _, _ = frame_decode_indexed(good, len(data), max_chunks=2)   # chunk table too small: declined, then the walk
    assert st[0] == "Invalid" and st[2] == 1


def test_unclean_streams_are_declined(oracle):
    data = corpus("alice29.txt")[:200000]
    good = oracle.frame_encode(data)
    c0 = walk(good)[1]                                               # second chunk header
    unclean = {
        "padding": IDENT + b"\xfe\x03\x00\x00abc" + good[10:],
        "skippable": good[:c0] + b"\x80\x02\x00\x00zz" + good[c0:],
        "repeated identifier": good + good,
        "reserved type": good[:c0] + b"\x02" + good[c0 + 1:],
        "truncated": good[:-100],
        "trailing bytes": good + b"\x00\x07",
        "bad identifier": b"\xff\x06\x00\x00sNaPpZ" + good[10:],
    }
    for name, s in unclean.items():
        assert frame_index(s)[0] == NOT_INDEXABLE, name
        check_decode(oracle, s, need_serial=1)
    nchunks = len(walk(good)) - 1
    assert frame_index(good, max_chunks=nchunks - 1)[0] == NOT_INDEXABLE
    assert frame_index(good, max_chunks=nchunks)[1] == walk(good)
    # a padding chunk forces the walk, which still decodes the same bytes
    assert check_decode(oracle, unclean["padding"], need_serial=1) == data
