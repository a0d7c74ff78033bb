"""Validation without decoded bytes on the GPU, through the C ABI: sb_validate_batch_device_ws and
sb_frame_validate_batch_device_ws must give every unit the status, out_lens and d_unit_blocks / d_unit_chunks of
sb_decompress_batch_device_ws and sb_frame_decode_batch_device_ws with caps a decode cannot exceed, with output pointers
null or aimed at a canary that stays untouched; sb_validate and snappy_validate_compressed_buffer must agree with
sb_decompress and snappy_uncompress; the Python wrappers with Decoder().decompress_vec and frame.decode_batch."""
import ctypes as C
import random

import numpy as np
import pytest

import legal_streams as ls
from conftest import CORPUS, corpus

pytestmark = pytest.mark.gpu

BLOCK = 65536
U32 = 0xFFFFFFFF


@pytest.fixture(scope="module")
def snap():
    import torch
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)
    import gpu_helpers
    return gpu_helpers.snap()


def _header(s):
    v, shift = 0, 0
    for c in s[:10]:
        v |= (c & 0x7F) << shift
        shift += 7
        if c < 0x80:
            return v
    return None


def _decode_cap(s):
    """A cap under which a decode decides as with 2^32 - 1: the header's value (any cap for a bad or too big one)."""
    v = _header(s)
    return 16 if v is None or v > U32 else v


class Batch:
    """Units at odd device addresses (pointers, or a base with an odd stride), results, a canary output region."""

    def __init__(self, snap, streams, addressing="ptrs"):
        import torch
        self.snap, self.n, self.dev = snap, len(streams), torch.device("cuda", 0)
        n = self.n
        if addressing == "ptrs":
            offs, at = [], 1
            for s in streams:
                offs.append(at)
                at += len(s) + 3 + (at + len(s)) % 2
            size = at + 16
        else:
            self.stride = max([len(s) for s in streams] + [1]) | 1
            offs = [1 + i * self.stride for i in range(n)]
            size = 1 + n * self.stride + 16
        host = np.zeros(size, dtype=np.uint8)
        for o, s in zip(offs, streams):
            host[o:o + len(s)] = np.frombuffer(s, dtype=np.uint8)
        self.t_in = torch.from_numpy(host).to(self.dev)
        self.offs, self.addressing = offs, addressing
        self.t_lens = torch.tensor([len(s) for s in streams] + [0], dtype=torch.int32, device=self.dev)
        self.t_ptrs = torch.tensor([self.t_in.data_ptr() + o for o in offs] + [0], dtype=torch.int64, device=self.dev)
        self.t_res = torch.empty(8 * (n + 1) + 32 * (n + 1), dtype=torch.uint8, device=self.dev)
        self.t_canary = torch.full((1 << 16,), 0xEE, dtype=torch.uint8, device=self.dev)

    def batch(self, out_ptrs=None, caps=None, out_base=None, out_stride=0, cap_uniform=0):
        b = self.snap._lib.SbBatch()
        if self.addressing == "ptrs":
            b.in_ptrs = self.t_ptrs.data_ptr()
        else:
            b.in_base, b.in_stride = self.t_in.data_ptr() + 1, self.stride
        b.in_lens = self.t_lens.data_ptr()
        b.out_ptrs, b.out_caps, b.out_base, b.out_stride, b.out_cap_uniform = out_ptrs, caps, out_base, out_stride, cap_uniform
        self.t_res.fill_(0xAB)
        b.out_lens, b.statuses, b.count = self.t_res.data_ptr(), self.t_res.data_ptr() + 8 * (self.n + 1), self.n
        return b

    def canary_batch(self):
        """Output pointers into the canary, caps of 3 (ignored by validation)."""
        import torch
        self._cptrs = torch.tensor([self.t_canary.data_ptr() + 7] * (self.n + 1), dtype=torch.int64, device=self.dev)
        self._ccaps = torch.full((self.n + 1,), 3, dtype=torch.int32, device=self.dev)
        if self.addressing == "ptrs":
            return self.batch(self._cptrs.data_ptr(), self._ccaps.data_ptr())
        return self.batch(out_base=self.t_canary.data_ptr() + 5, out_stride=1, cap_uniform=3)

    def results(self, extra=None):
        back = self.t_res.cpu().numpy()
        lens = back[:4 * self.n].view(np.uint32)
        st = back[8 * (self.n + 1):8 * (self.n + 1) + 32 * self.n].view(np.uint64).reshape(self.n, 4)
        out = [((int(s[0] & 0xFFFFFFFF), int(s[1]), int(s[2]), int(s[3])), int(k)) for s, k in zip(st, lens)]
        return out, (extra.cpu().numpy().view(np.uint32)[:self.n].tolist() if extra is not None else None)

    def canary_ok(self):
        return bool((self.t_canary == 0xEE).all())


def _raw_decode(snap, B, caps):
    """sb_decompress_batch_device_ws with per-unit caps: [(status, len)], unit_blocks."""
    import torch
    L = snap._lib.lib()
    outs = torch.empty(sum(caps) + 16, dtype=torch.uint8, device=B.dev)
    offs = np.concatenate([[0], np.cumsum(caps[:-1])]).astype(np.int64) if caps else np.zeros(0, np.int64)
    t_ptrs = torch.tensor(list(offs + outs.data_ptr()) + [0], dtype=torch.int64, device=B.dev)
    t_caps = torch.tensor(list(caps) + [0], dtype=torch.int32, device=B.dev)
    b = B.batch(t_ptrs.data_ptr(), t_caps.data_ptr())
    ib = sum(int(x) for x in B.t_lens.cpu())
    need = L.sb_decompress_batch_scratch_bytes(B.n, ib)
    scr = torch.empty(need, dtype=torch.uint8, device=B.dev)
    blocks = torch.full((B.n + 1,), -1, dtype=torch.int32, device=B.dev)
    e = snap._lib.SbError()
    assert L.sb_decompress_batch_device_ws(C.byref(b), ib, blocks.data_ptr(), scr.data_ptr(), need, None, C.byref(e)) == 0
    return B.results(blocks)


def _raw_validate(snap, B, b, scr=None):
    import torch
    L = snap._lib.lib()
    ib = sum(int(x) for x in B.t_lens.cpu())
    need = L.sb_decompress_batch_scratch_bytes(B.n, ib)
    if scr is None:
        scr = torch.empty(need, dtype=torch.uint8, device=B.dev)
    blocks = torch.full((B.n + 1,), -1, dtype=torch.int32, device=B.dev)
    e = snap._lib.SbError()
    assert L.sb_validate_batch_device_ws(C.byref(b), ib, blocks.data_ptr(), scr.data_ptr(), need, None, C.byref(e)) == 0
    res = B.results(blocks)
    assert int(blocks[B.n]) == -1
    return res


def _raw_streams(oracle):
    rng = random.Random(17)
    streams = [oracle.compress(corpus(name)) for name in CORPUS]              # several take the split path
    streams += [corpus("Mark.Twain-Tom.Sawyer.txt.rawsnappy")] + [corpus("baddata%d.snappy" % i) for i in (1, 2, 3)]
    for size in (10, 3000, 3 * BLOCK + 5):
        for mode in ("blocked", "unblocked"):
            s = ls.gen_stream(rng, size, mode=mode)
            streams += [s.stream] + ls.corrupt(rng, s)
    streams.append(ls.giant_literal(rng, 70000, "lit62")[0])                 # declined by the split
    big = oracle.compress(corpus("lcet10.txt"))
    b = bytearray(big)
    b[len(b) // 2] ^= 0x10
    streams += [bytes(b), big[:-3], b"", b"\x00", ls.varint(1 << 32) + b"\x00", bytes([big[0] + 1]) + big[1:]]
    return streams


@pytest.mark.parametrize("addressing", ["ptrs", "base"])
def test_raw_batch_matches_decode(snap, oracle, addressing):
    streams = _raw_streams(oracle)
    B = Batch(snap, streams, addressing)
    want, want_blocks = _raw_decode(snap, B, [_decode_cap(s) for s in streams])
    assert sum(1 for x in want_blocks if x) >= 6
    got, blocks = _raw_validate(snap, B, B.batch())                          # null output pointers
    assert got == want and blocks == want_blocks
    got, blocks = _raw_validate(snap, B, B.canary_batch())
    assert got == want and blocks == want_blocks
    assert B.canary_ok()


def test_raw_batch_allocates_nothing(snap, oracle):
    import torch
    streams = _raw_streams(oracle)[:20]
    B = Batch(snap, streams)
    L = snap._lib.lib()
    scr = torch.empty(L.sb_decompress_batch_scratch_bytes(B.n, sum(len(s) for s in streams)), dtype=torch.uint8,
                      device=B.dev)
    first = _raw_validate(snap, B, B.batch(), scr)
    before = L.sb_alloc_count()
    for _ in range(3):
        assert _raw_validate(snap, B, B.batch(), scr) == first
    assert L.sb_alloc_count() == before


def test_sb_validate_and_snappy_shim(snap, oracle):
    L = snap._lib.lib()
    for s in _raw_streams(oracle):
        try:
            want = len(snap.raw.Decoder().decompress_vec(s))
        except snap.Error as e:
            want = e
        try:
            got = snap.raw.validate(s)
        except snap.Error as e:
            got = e
        assert got == want
        cap = _decode_cap(s)
        buf = (C.c_char * max(cap, 1))()
        n = C.c_size_t(cap)
        ok = L.snappy_uncompress(s, len(s), buf, C.byref(n)) == 0
        assert (L.snappy_validate_compressed_buffer(s, len(s)) == 0) == ok
        assert ok == isinstance(want, int)


def test_raw_validate_batch_python(snap, oracle):
    streams = _raw_streams(oracle)
    res = snap.raw.validate_batch(streams[:12] + [bytearray(streams[3]), memoryview(streams[4]),
                                                  np.frombuffer(streams[5], dtype=np.uint8)] + streams[12:])
    res = res[:12] + res[15:]
    assert len(res) == len(streams)
    for s, (k, err) in zip(streams, res):
        try:
            assert (k, err) == (len(snap.raw.Decoder().decompress_vec(s)), None)
        except snap.Error as e:
            assert (k, err) == (0, e)


# ----------------------------------------------------------------------------------------------------------- frame

def _frames(oracle):
    rng = random.Random(29)
    enc = oracle.frame_encode
    text = (corpus("alice29.txt") + corpus("lcet10.txt")) * 2
    three = enc(text[:3 * BLOCK - 100])
    offs = [10, 10 + 4 + int.from_bytes(three[11:14], "little")]
    offs.append(offs[1] + 4 + int.from_bytes(three[offs[1] + 1:offs[1] + 4], "little"))

    def flip(s, at):
        b = bytearray(s)
        b[at] ^= 0x5A
        return bytes(b)

    stored = enc(bytes(rng.getrandbits(8) for _ in range(3 * BLOCK - 7)))
    assert [stored[10 + k * (8 + BLOCK)] for k in range(3)] == [1, 1, 1]
    return [b"", ls.IDENT, enc(text[:1000]), enc(text[:700_000]), enc(bytes(rng.getrandbits(8) for _ in range(70000))),
            ls.gen_frame(rng, oracle.crc32c_masked, 9).stream,
            ls.gen_frame(rng, oracle.crc32c_masked, 6, kinds=("pad", "skip", "raw")).stream,
            flip(three, offs[0] + 5), flip(three, offs[1] + 5), flip(three, offs[2] + 5), flip(three, offs[2] + 30),
            three[:offs[1] + 20], three[:-5], three + bytes([0x05, 4, 0, 0]) + bytes(4),
            # stored chunks (random bytes): CRC flips in the first and the last, a body byte flipped in the middle one
            flip(stored, 10 + 6), flip(stored, 10 + 2 * (8 + BLOCK) + 4), flip(stored, 10 + 8 + BLOCK + 100)]


def _frame_call(snap, B, b, validate, max_chunks):
    import torch
    L = snap._lib.lib()
    ib = sum(int(x) for x in B.t_lens.cpu())
    f = L.sb_frame_validate_batch_scratch_bytes if validate else L.sb_frame_decode_batch_scratch_bytes
    need = f(B.n, ib, max_chunks)
    scr = torch.empty(need, dtype=torch.uint8, device=B.dev)
    chunks = torch.full((B.n + 1,), -1, dtype=torch.int32, device=B.dev)
    e = snap._lib.SbError()
    call = L.sb_frame_validate_batch_device_ws if validate else L.sb_frame_decode_batch_device_ws
    assert call(C.byref(b), ib, 0, None, None, max_chunks, chunks.data_ptr(), scr.data_ptr(), need, None, C.byref(e)) == 0
    res = B.results(chunks)
    assert int(chunks[B.n]) == -1
    return res


def _frame_decode(snap, B, max_chunks):
    """sb_frame_decode_batch_device_ws with every cap at the unit's need (found by a pass with caps of 0)."""
    import torch
    zeros = torch.zeros(B.n + 1, dtype=torch.int32, device=B.dev)
    nulls = torch.zeros(B.n + 1, dtype=torch.int64, device=B.dev)
    st, _ = _frame_call(snap, B, B.batch(nulls.data_ptr(), zeros.data_ptr()), False, max_chunks)
    caps = [s[2] if s[0] == 2 else 0 for s, _ in st]
    outs = torch.empty(sum(caps) + 16, dtype=torch.uint8, device=B.dev)
    offs = np.concatenate([[0], np.cumsum(caps[:-1])]).astype(np.int64)
    t_ptrs = torch.tensor(list(offs + outs.data_ptr()) + [0], dtype=torch.int64, device=B.dev)
    t_caps = torch.tensor(caps + [0], dtype=torch.int32, device=B.dev)
    return _frame_call(snap, B, B.batch(t_ptrs.data_ptr(), t_caps.data_ptr()), False, max_chunks)


@pytest.mark.parametrize("addressing", ["ptrs", "base"])
def test_frame_batch_matches_decode(snap, oracle, addressing):
    streams = _frames(oracle)
    B = Batch(snap, streams, addressing)
    for mc in (sum(len(s) // 8 + 2 for s in streams), 14):                 # ample, and too small for the later units
        want = _frame_decode(snap, B, mc)
        got = _frame_call(snap, B, B.batch(), True, mc)
        assert got == want
        got = _frame_call(snap, B, B.canary_batch(), True, mc)
        assert got == want
        assert B.canary_ok()


def test_frame_scratch_bound(snap):
    L = snap._lib.lib()
    for count, ib, mc in ((1, 100, 1), (5, 1 << 20, 1000), (4096, 1 << 32, 1 << 20)):
        extra = L.sb_frame_validate_batch_scratch_bytes(count, ib, mc) - L.sb_frame_decode_batch_scratch_bytes(count, ib, mc)
        assert 0 < extra <= (256 << 20) + 256
        assert extra == min(mc, 4096) * BLOCK + 256                        # nothing depends on decoded sizes


def test_frame_validate_batch_python(snap, oracle):
    streams = _frames(oracle)
    res = snap.frame.validate_batch(streams)
    for s, (k, err) in zip(streams, res):
        try:
            out = snap.frame.decode_batch([s])[0]
            assert (k, err) == (len(out), None)
        except (snap.Error, snap.UnexpectedEof) as e:
            assert err is not None and type(err) is type(e) and str(err) == str(e)
    assert [r[1] is None for r in res] == [True] * 7 + [False] * 10
    assert res[8][0] == BLOCK and res[9][0] == 2 * BLOCK                   # bytes before the bad chunk
    assert [r[0] for r in res[-3:]] == [0, 2 * BLOCK, BLOCK]               # ... and before the bad stored chunk


def test_frame_batch_allocates_nothing(snap, oracle):
    import torch
    streams = _frames(oracle)
    B = Batch(snap, streams)
    L = snap._lib.lib()
    mc = sum(len(s) // 8 + 2 for s in streams)
    ib = sum(len(s) for s in streams)
    need = L.sb_frame_validate_batch_scratch_bytes(B.n, ib, mc)
    scr = torch.empty(need, dtype=torch.uint8, device=B.dev)
    chunks = torch.full((B.n + 1,), -1, dtype=torch.int32, device=B.dev)
    e = snap._lib.SbError()

    def run():
        b = B.batch()
        assert L.sb_frame_validate_batch_device_ws(C.byref(b), ib, 0, None, None, mc, chunks.data_ptr(), scr.data_ptr(), need,
                                                   None, C.byref(e)) == 0
        return B.results(chunks)

    first = run()
    before = L.sb_alloc_count()
    for _ in range(3):
        assert run() == first
    assert L.sb_alloc_count() == before


def test_frame_more_live_chunks_than_slots(snap, oracle):
    """5,100 small live chunks against the pool of 4,096 slots: warps take chunks from the counter until the table is
    done; the first bad chunk of each unit is the one reported."""
    def many(n, bad):
        parts = [ls.IDENT]
        for i in range(n):
            data = bytes([i & 0xFF, (i >> 8) & 0xFF]) * (1 + i % 5)
            crc = oracle.crc32c_masked(data) ^ (1 if i in bad else 0)
            parts.append(ls.chunk(0, oracle.compress(data), crc) if i % 2 == 0 else ls.chunk(1, data, crc))
        return b"".join(parts)

    streams = [many(2000, {1999}), many(3000, {2500, 777}), many(100, ())]
    B = Batch(snap, streams)
    mc = sum(len(s) // 8 + 2 for s in streams)
    want = _frame_decode(snap, B, mc)
    got = _frame_call(snap, B, B.batch(), True, mc)
    assert got == want
    assert [s[0] for s, _ in got[0]] == [14, 14, 0] and got[1] == [2000, 3000, 100]
