"""Validation without decoded bytes on CPU: K2's output-free loop (k2_decode_stream<true, false>), K8b's validate mode
and K19's frame validation (rust-snappy_b200/csrc/k19_validate.cuh) compiled by g++ against the fiber warp emulator
(tests/emu/emu_validate.cpp). Every unit's status, out_lens and d_unit_blocks / d_unit_chunks must equal the emulator's
decode harnesses (one-warp K2, K8b, K11) given caps a decode cannot exceed, and the oracle; output pointers aimed at a
canary must leave it untouched. Also checks that every new entry point of the library refuses to run without a GPU.
Test tooling only, like tests/test_raw_batch_split_emu.py."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest

import emu_helpers as emu
import legal_streams as ls
import test_frame_batch_decode_emu as fb
import test_raw_batch_split_emu as rb
import test_raw_split_emu as single
from conftest import CORPUS, corpus

BLOCK = 65536
INVALID = 202
GUARD = 512
U32 = 0xFFFFFFFF

_HERE = os.path.dirname(os.path.abspath(__file__))
_EMU = os.path.join(_HERE, "emu")
_SO = os.path.join(_EMU, "_build", "libemu_validate.so")
_lib = None


def vlib():
    """The emulator build of the validation bodies (tests/emu/emu_validate.cpp), rebuilt when a source is newer."""
    global _lib
    if _lib is None:
        csrc = os.path.join(os.path.dirname(_HERE), "rust-snappy_b200", "csrc")
        srcs = [os.path.join(_EMU, f) for f in ("emu_validate.cpp", "simt_emu.cpp", "simt_emu.h")]
        srcs += [os.path.join(csrc, f) for f in os.listdir(csrc)]
        if not os.path.exists(_SO) or os.path.getmtime(_SO) < max(os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(_SO), exist_ok=True)
            tmp = "%s.%d.tmp" % (_SO, os.getpid())
            subprocess.check_call(["g++", "-O2", "-g", "-std=c++17", "-fPIC", "-shared", "-Wall", "-Wno-unused-function",
                                   "-Wno-unknown-pragmas", "-Wl,-Bsymbolic", "-o", tmp,
                                   os.path.join(_EMU, "emu_validate.cpp"), os.path.join(_EMU, "simt_emu.cpp")])
            os.replace(tmp, _SO)
        _lib = C.CDLL(_SO)
        _lib.emu_raw_validate_scratch_bytes.restype = C.c_uint64
        _lib.emu_raw_validate_scratch_bytes.argtypes = [C.c_uint32, C.c_uint64]
        _lib.emu_raw_validate_batch.argtypes = [C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64]
        _lib.emu_frame_validate_scratch_bytes.restype = C.c_uint64
        _lib.emu_frame_validate_scratch_bytes.argtypes = [C.c_uint32, C.c_uint64, C.c_uint32]
        _lib.emu_frame_validate_batch.argtypes = [C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_void_p, C.c_uint32,
                                                  C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64]
        _lib.emu_k2_validate.argtypes = [C.c_void_p, C.c_uint32]
    return _lib


def _status(e):
    return (emu.ERR.get(e.code, fb.NAMES.get(e.code, str(e.code))), e.a, e.b, e.c)


class _Units:
    """Inputs at odd addresses (pointers, or a base with an odd stride), results with a guard entry, and a canary
    output region the validation calls may be pointed at but must not write."""

    def __init__(self, streams, addressing="ptrs", canary=True):
        n = self.n = len(streams)
        if addressing == "ptrs":
            offs, at = [], 1
            for s in streams:
                offs.append(at)
                at += len(s) + 3 + (at + len(s)) % 2
            self.inbuf = np.zeros(at + 16, dtype=np.uint8)
        else:
            stride = max([len(s) for s in streams] + [1]) | 1
            offs = [1 + i * stride for i in range(n)]
            self.inbuf = np.zeros(1 + n * stride + 16, dtype=np.uint8)
        for o, s in zip(offs, streams):
            self.inbuf[o:o + len(s)] = np.frombuffer(s, dtype=np.uint8)
        self.lens = np.array([len(s) for s in streams] + [0], dtype=np.uint32)
        self.in_ptrs = np.array([self.inbuf.ctypes.data + o for o in offs] + [0], dtype=np.uint64)
        self.canary = np.full(4096, 0xEE, dtype=np.uint8)
        self.out_ptrs = np.array([self.canary.ctypes.data + 3] * (n + 1), dtype=np.uint64)
        self.caps = np.full(n + 1, 7, dtype=np.uint32)
        self.out_lens = np.full(n + 1, 0xDEADBEEF, dtype=np.uint32)
        self.st = (emu.SbError * max(n, 1))()
        self.extra = np.full(n + 1, 0xDEADBEEF, dtype=np.uint32)   # d_unit_blocks / d_unit_chunks
        b = self.b = emu.SbBatch()
        if addressing == "ptrs":
            b.in_ptrs = self.in_ptrs.ctypes.data
            if canary:
                b.out_ptrs, b.out_caps = self.out_ptrs.ctypes.data, self.caps.ctypes.data
        else:
            b.in_base, b.in_stride = self.inbuf.ctypes.data + 1, stride
            if canary:
                b.out_base, b.out_stride, b.out_cap_uniform = self.canary.ctypes.data + 5, 1, 3
        b.in_lens = self.lens.ctypes.data
        b.out_lens, b.statuses, b.count = self.out_lens.ctypes.data, C.addressof(self.st), n

    def results(self):
        assert (self.canary == 0xEE).all()                                  # no decoded byte written
        assert int(self.out_lens[self.n]) == 0xDEADBEEF and int(self.extra[self.n]) == 0xDEADBEEF
        return [(_status(self.st[i]), int(self.out_lens[i])) for i in range(self.n)], [int(x) for x in self.extra[:self.n]]


def _scratch(size):
    return np.full(size + GUARD, 0xCD, dtype=np.uint8)


def raw_validate(streams, addressing="ptrs", canary=True, in_bytes=None, seg=rb.SEG_MIN):
    """sb_validate_batch_device_ws under the emulator: [(status, out_len)], d_unit_blocks."""
    u = _Units(streams, addressing, canary)
    if in_bytes is None:
        in_bytes = sum(len(s) for s in streams)
    L = vlib()
    size = L.emu_raw_validate_scratch_bytes(u.n, in_bytes)
    scratch = _scratch(size)
    assert L.emu_raw_validate_batch(C.byref(u.b), in_bytes, u.extra.ctypes.data, scratch.ctypes.data, size, seg) == 0
    assert bytes(scratch[size:]) == b"\xcd" * GUARD
    return u.results()


def frame_validate(streams, flags=0, index=None, max_chunks=None, in_bytes=None, addressing="ptrs", canary=True):
    """sb_frame_validate_batch_device_ws under the emulator: [(status, out_len)], d_unit_chunks."""
    u = _Units(streams, addressing, canary)
    if in_bytes is None:
        in_bytes = sum(len(s) for s in streams)
    if max_chunks is None:
        max_chunks = sum(len(s) // 8 + 2 for s in streams)
    cidx = cat = None
    if index is not None:
        flat, at_list = [], []
        for ix in index:
            at_list.append(len(flat))
            flat += list(ix)
        at_list.append(len(flat))
        cidx = np.array(flat + [0xCDCD] * 4, dtype=np.uint64)
        cat = np.array(at_list, dtype=np.uint64)
    L = vlib()
    size = L.emu_frame_validate_scratch_bytes(u.n, in_bytes, max_chunks)
    scratch = _scratch(size)
    rc = L.emu_frame_validate_batch(C.byref(u.b), in_bytes, flags, cidx.ctypes.data if cidx is not None else None,
                                    cat.ctypes.data if cat is not None else None, max_chunks, u.extra.ctypes.data,
                                    scratch.ctypes.data, size, fb.SEG)
    assert rc == 0
    assert bytes(scratch[size:]) == b"\xcd" * GUARD
    return u.results()


# ------------------------------------------------------------------------------------------------------------- raw

def _header(s):
    """The header's value, or None when it is malformed."""
    v, shift = 0, 0
    for i, c in enumerate(s[:10]):
        v |= (c & 0x7F) << shift
        shift += 7
        if c < 0x80:
            return v
    return None


def _decode_cap(s):
    """A cap under which a decode decides as it would with 2^32 - 1: the header's value (any cap for a bad or too big
    header). Streams announcing more than 4 MiB that a decode accepts are not used here."""
    v = _header(s)
    if v is None or v > U32:
        return 16
    assert v <= 1 << 22
    return v


def raw_reference(oracle, streams, in_bytes=None):
    """The K8b decode harness with caps no decision depends on, checked against the oracle: [(status, len)], blocks."""
    caps = [_decode_cap(s) for s in streams]
    res, blocks, _ = rb.run_batch(streams, caps, in_bytes=in_bytes)
    out = []
    for s, cap, (st, data) in zip(streams, caps, res):
        want_st, want = single.oracle_result(oracle, s, cap)
        assert st == want_st
        if want is not None:
            assert data == want
        out.append((st, len(data) if data is not None else 0))
    return out, blocks


def check_raw(oracle, streams, addressing="ptrs", canary=True, **kw):
    want, want_blocks = raw_reference(oracle, streams, kw.get("in_bytes"))
    got, blocks = raw_validate(streams, addressing, canary, **kw)
    assert got == want
    assert blocks == want_blocks
    # K2 alone, one warp per unit, with the same caps: the decode harness's status and length
    caps = [_decode_cap(s) for s in streams]
    u = _Units(streams, canary=False)
    u.b.out_caps = u.caps.ctypes.data
    u.caps[:len(caps)] = caps
    vlib().emu_k2_validate(C.byref(u.b), 2)
    k2 = u.results()[0]
    one = emu.decompress_units(streams, caps, grid=2, block=64)
    assert k2 == [(st, len(data)) for st, data, _ in one]
    return got, blocks


def _golden(oracle):
    streams = [oracle.compress(corpus(name)) for name in CORPUS]
    streams += [corpus("Mark.Twain-Tom.Sawyer.txt.rawsnappy")] + [corpus("baddata%d.snappy" % i) for i in (1, 2, 3)]
    return streams


@pytest.mark.parametrize("addressing", ["ptrs", "base"])
def test_golden_files(oracle, addressing):
    streams = _golden(oracle)
    got, blocks = check_raw(oracle, streams, addressing, canary=addressing == "ptrs")
    assert sum(1 for b in blocks if b) >= 6                             # the split path ran
    assert [r[0][0] for r in got[:len(CORPUS)]] == ["Ok"] * len(CORPUS)
    assert any(r[0][0] != "Ok" for r in got[-3:])


@pytest.mark.parametrize("mode", ["blocked", "unblocked"])
def test_generated_streams_and_corruptions(oracle, mode):
    rng = random.Random(41 if mode == "blocked" else 42)
    streams = []
    for size in (1, 100, 5000, 65536, 65537, 3 * BLOCK + 17):
        s = ls.gen_stream(rng, size, mode=mode, pad=rng.choice((None, 3, 5)))
        streams.append(s.stream)
        streams += ls.corrupt(rng, s)
    for _ in range(6):
        s = ls.gen_single(rng)
        streams.append(s.stream)
        streams += ls.corrupt(rng, s)
    _, blocks = check_raw(oracle, streams)
    if mode == "blocked":
        assert any(blocks)


def test_giant_literal_and_edges(oracle):
    rng = random.Random(7)
    streams = [ls.giant_literal(rng, n, form)[0] for n, form in ((70000, "lit62"), (140000, "lit63"))]
    small = oracle.compress(b"abcd" * 50 + bytes(range(200)) + b"abcd" * 40)
    streams += [small[:k] for k in range(len(small) + 1)]                # every truncation, the empty one included
    streams += [b"\x00", b"\x05", ls.varint(1 << 32) + b"\x00\x00", ls.varint(1 << 22) + b"\x00",
                small[:1] + small[1:] + b"\x00\x41",                         # one element more than the header says
                bytes([small[0] + 1]) + small[1:]]                          # one byte more announced
    got, blocks = check_raw(oracle, streams)
    assert blocks[:2] == [0, 0]                                          # the split declines literals over 64 KB
    names = {r[0][0] for r in got}
    assert {"Empty", "TooBig", "HeaderMismatch", "Ok"} <= names


def test_declined_and_corrupt_split_units(oracle):
    streams = rb._declined_units() + rb._corrupt_units(oracle) + rb._clean_units(oracle)[:6]
    check_raw(oracle, streams, addressing="base", canary=False)
    _, blocks = check_raw(oracle, streams, in_bytes=sum(len(s) for s in streams) - 1)
    assert blocks == [0] * len(streams)                                  # nothing split


def test_raw_call_checks():
    L = vlib()
    b = emu.SbBatch()
    lens = np.zeros(4, dtype=np.uint32)
    st = (emu.SbError * 4)()
    scratch = np.zeros(1 << 16, dtype=np.uint8)
    b.out_lens, b.statuses, b.count = lens.ctypes.data, C.addressof(st), 0
    call = lambda bb, s=scratch.ctypes.data, sz=1 << 16: L.emu_raw_validate_batch(bb, 1 << 10, None, s, sz, 0)
    assert call(C.byref(b)) == 0
    assert call(None) == INVALID
    assert call(C.byref(b), s=None) == INVALID
    b.count = 3
    assert call(C.byref(b), sz=L.emu_raw_validate_scratch_bytes(3, 1 << 10) - 1) == INVALID
    b.statuses = None
    assert call(C.byref(b)) == INVALID
    b.statuses, b.out_lens = C.addressof(st), None
    assert call(C.byref(b)) == INVALID


# ----------------------------------------------------------------------------------------------------------- frame

def frame_reference(streams, **kw):
    """The K11 decode harness with every cap at the unit's need (what a cap of 2^32 - 1 gives): [(status, len)], chunks.
    A first pass with caps of 0 reports each need as BufferTooSmall{0, need}."""
    rc, res, _ = fb.run_batch(streams, [0] * len(streams), **kw)
    assert rc == 0
    caps = [st[2] if st[0] == "BufferTooSmall" else 0 for st, _ in res]
    rc, res, uc = fb.run_batch(streams, caps, **kw)
    assert rc == 0
    return [(st, len(data)) for st, data in res], uc


def check_frame(oracle, streams, flags=0, **kw):
    want, want_uc = frame_reference(streams, flags=flags, **kw)
    for mode in ("ptrs", "base"):
        got, uc = frame_validate(streams, flags=flags, addressing=mode, canary=mode == "ptrs", **kw)
        assert got == want
        assert uc == want_uc
    if not flags & 1:
        for (st, k), s in zip(got, streams):
            if st[0] == "Invalid":
                continue
            ost, odata = fb.oracle_decode(oracle, s)
            assert st == ost
            if odata is not None:
                assert k == len(odata)
    return got, uc


def _frames(oracle):
    rng = random.Random(23)
    enc = oracle.frame_encode
    three = enc(fb._text(3 * 65536 - 100, 2))
    c3 = fb.chain(three)
    gens = [ls.gen_frame(rng, oracle.crc32c_masked, k) for k in (4, 9)]
    mid = c3[1] + 20
    stored = enc(fb._random(3 * 65536 - 7, 8))                         # three stored chunks (random bytes)
    cs = fb.chain(stored)
    assert [stored[o] for o in cs[:-1]] == [1, 1, 1]
    return [
        b"", fb.IDENT, enc(fb._text(1000, 3)), enc(fb._text(700_000, 1)), enc(fb._random(70000, 4)),
        gens[0].stream, gens[1].stream,
        ls.gen_frame(rng, oracle.crc32c_masked, 6, kinds=("pad", "skip", "raw")).stream,
        fb._flip(three, c3[0] + 5), fb._flip(three, c3[1] + 5), fb._flip(three, c3[2] + 5),   # CRC flips
        fb._flip(three, c3[2] + 30),                                                          # corrupt body
        three[:mid], three[:-5],                                                              # truncations
        three + bytes([0x05, 4, 0, 0]) + bytes(4), fb.IDENT[:4] + b"sNaPpZ" + three[10:],
        fb._flip(stored, cs[0] + 6), fb._flip(stored, cs[2] + 4),      # CRC flips in stored chunks
        fb._flip(stored, cs[1] + 100),                                 # a stored body that no longer matches its CRC
    ]


def test_frames(oracle):
    streams = _frames(oracle)
    got, uc = check_frame(oracle, streams)
    assert got[3][0][0] == "Ok" and uc[3] == fb.data_chunks(streams[3])
    assert [g[0][0] for g in got[8:11]] == ["Checksum"] * 3
    assert [g[0][0] for g in got[-3:]] == ["Checksum"] * 3
    assert [g[1] for g in got[-3:]] == [0, 2 * 65536, 65536]            # bytes before the bad stored chunk
    assert got[9][1] == 65536 and got[10][1] == 2 * 65536                # bytes produced before the bad chunk


def test_frame_caller_index(oracle):
    streams = _frames(oracle)
    good = [fb._index_of(s) for s in streams]
    got, uc = check_frame(oracle, streams, index=good)
    wrong = [list(x) for x in good]
    wrong[2] = [123456789, 5, 77]
    wrong[3][1] += 1
    got2, uc2 = check_frame(oracle, streams, index=wrong)
    assert [g for g in got2] == got and uc2[3] == 0 and uc[3] > 0


def test_frame_fragments(oracle):
    rng = random.Random(5)
    frags = [oracle.frame_encode(fb._text(n, n))[10:] for n in (1, 65536, 300000)]
    frags += [b"", ls.gen_frame(rng, oracle.crc32c_masked, 7).stream[10:], fb.IDENT + frags[0]]
    check_frame(oracle, frags, flags=1)


@pytest.mark.parametrize("indexed", [False, True])
def test_frame_chunk_table_too_small(oracle, indexed):
    enc = oracle.frame_encode
    streams = [enc(fb._text(n, n)) for n in (100000, 5000, 200000, 70000)]
    need = [fb.data_chunks(s) for s in streams]
    index = [fb.chain(s) for s in streams] if indexed else None
    for k in (1, 3):
        got, uc = check_frame(oracle, streams, index=index, max_chunks=sum(need[:k + 1]) - 1)
        assert got[k] == (("Invalid", sum(need[:k + 1]) - 1, 1, 0), 0)
    check_frame(oracle, streams, index=index, max_chunks=sum(need))


def _many_chunks(oracle, n, bad):
    """A frame stream of n small chunks, compressed and stored in turn; chunk `bad` (if any) with a wrong CRC."""
    parts = [fb.IDENT]
    for i in range(n):
        data = bytes([i & 0xFF, (i >> 8) & 0xFF]) * (1 + i % 5)
        crc = oracle.crc32c_masked(data) ^ (1 if i == bad else 0)
        parts.append(ls.chunk(0, oracle.compress(data), crc) if i % 2 == 0 else ls.chunk(1, data, crc))
    return b"".join(parts)


def test_frame_more_live_chunks_than_slots(oracle):
    """4,300 live chunks against a pool of 4,096 slots (max_chunks above 4,096): warps take chunks from the counter
    until the table is done, and the first bad chunk of a unit is still the one reported."""
    streams = [_many_chunks(oracle, 2000, 1999), _many_chunks(oracle, 2200, 777), _many_chunks(oracle, 100, None)]
    L = vlib()
    mc = sum(len(s) // 8 + 2 for s in streams)
    assert mc > 4096
    assert L.emu_frame_validate_scratch_bytes(3, 0, mc) - fb.kdlib().emu_frame_decode_batch_scratch_bytes(3, 0, mc) == \
        4096 * 65536 + 256                                             # the pool holds 4,096 slots, fewer than the chunks
    got, uc = check_frame(oracle, streams)
    assert [g[0][0] for g in got] == ["Checksum", "Checksum", "Ok"] and uc == [2000, 2200, 100]


def test_frame_call_checks_and_scratch():
    L = vlib()
    f, g = L.emu_frame_validate_scratch_bytes, fb.kdlib().emu_frame_decode_batch_scratch_bytes
    for count, in_bytes, mc in ((5, 0, 10), (5, 1 << 20, 1000), (9, 1 << 30, 1 << 20), (1, 1 << 36, 4194302)):
        extra = f(count, in_bytes, mc) - g(count, in_bytes, mc)
        assert extra == min(mc, 4096) * 65536 + 256 and extra <= (256 << 20) + 256
    b = emu.SbBatch()
    lens = np.zeros(4, dtype=np.uint32)
    st = (emu.SbError * 4)()
    scratch = np.zeros(1 << 16, dtype=np.uint8)
    ix = np.zeros(4, dtype=np.uint64)
    b.out_lens, b.statuses, b.count = lens.ctypes.data, C.addressof(st), 0
    call = lambda bb, mc=8, a=None, c=None, s=scratch.ctypes.data, sz=1 << 16: \
        L.emu_frame_validate_batch(bb, 0, 0, a, c, mc, None, s, sz, 0)
    assert call(C.byref(b)) == 0
    assert call(None) == INVALID
    assert call(C.byref(b), mc=0) == INVALID
    assert call(C.byref(b), mc=(1 << 22) - 1) == INVALID
    assert call(C.byref(b), a=ix.ctypes.data) == INVALID
    assert call(C.byref(b), s=None) == INVALID
    b.count = 1
    assert call(C.byref(b), sz=f(1, 0, 8) - 1) == INVALID
    b.statuses = None
    assert call(C.byref(b)) == INVALID


# -------------------------------------------------------------------------------------------------------- no device

def test_entry_points_refuse_without_a_device():
    import torch
    if torch.cuda.is_available():
        pytest.skip("a GPU is visible; the refusal path is for GPU-less hosts")
    import __graft_entry__ as g
    g.build_cuda()
    snap = g.load_package()
    L = snap._lib.lib()
    e = snap._lib.SbError()
    n = C.c_size_t(0)
    data = b"\x05\x10hello"
    assert L.sb_validate(data, len(data), C.byref(n), C.byref(e)) == 200 and e.code == 200
    assert L.snappy_validate_compressed_buffer(data, len(data)) == 1
    b = snap._lib.SbBatch()
    res = (C.c_uint8 * 64)()
    b.out_lens, b.statuses, b.count = C.addressof(res), C.addressof(res) + 8, 1
    scr = (C.c_uint8 * L.sb_frame_validate_batch_scratch_bytes(1, 64, 8))()
    e.code = 0
    assert L.sb_validate_batch_device_ws(C.byref(b), 64, None, scr, L.sb_decompress_batch_scratch_bytes(1, 64), None,
                                         C.byref(e)) == 200 and e.code == 200
    e.code = 0
    assert L.sb_frame_validate_batch_device_ws(C.byref(b), 64, 0, None, None, 8, None, scr,
                                               L.sb_frame_validate_batch_scratch_bytes(1, 64, 8), None, C.byref(e)) == 200
    assert e.code == 200
    with pytest.raises(snap.NoDevice):
        snap.raw.validate(data)
