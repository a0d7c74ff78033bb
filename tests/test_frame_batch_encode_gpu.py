"""Frame encode of a batch of units of any length on the GPU (sb_frame_encode_batch_device_ws): every unit's chunks go
through one K1 launch and each unit is assembled in its output as a complete framed stream. Every unit must equal the
oracle's frame_encode, host sb_frame_encode and sb_frame_encode_device_ws of the same unit (bytes and chunk index), or
carry the reference's exact error, and must decode back to its input through sb_frame_decode_device_ws."""
import ctypes as C

import numpy as np
import pytest

from conftest import corpus

pytestmark = pytest.mark.gpu

BLOCK = 65536
MIB = 1 << 20
INVALID = 202
MAX_OK = 3_679_453_184                 # 56,144 chunks: the largest n whose sb_frame_max_len fits a u32 cap
CODES = {0: "Ok", 2: "BufferTooSmall", INVALID: "Invalid"}
IDX_FILL = -0x5A5A5A5A5A5A5A5B         # 0xA5A5A5A5A5A5A5A5 as an int64


@pytest.fixture(scope="module")
def snap():
    import torch
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)
    import gpu_helpers
    return gpu_helpers.snap()


def chunks(n):
    return (n + BLOCK - 1) // BLOCK


def frame_max_len(n):
    return 10 + chunks(n) * (8 + 76490)


def _base():
    return corpus("alice29.txt") + corpus("lcet10.txt") + corpus("html_x_4") + corpus("kppkn.gtb")


def _text(n, seed):
    base = _base()
    k = seed * 7919 % len(base)
    return ((base[k:] + base) * (n // len(base) + 2))[:n]


def _u32(values):
    """A device int32 tensor holding u32 values (lengths and caps may exceed 2^31)."""
    import torch
    return torch.from_numpy(np.array(values, dtype=np.uint32).view(np.int32)).cuda()


def index_bases(lens):
    """Where every unit's index starts: i + Σ_{j<i} ceil(n_j / 65536); and the entry count."""
    bases, at = [], 0
    for n in lens:
        bases.append(at)
        at += chunks(n) + 1
    return bases, at


def encode_ws(L, snap, in_ptrs, lens, out_ptrs, caps, in_bytes=None, scratch_bytes=None, stream=None, base=None,
              uniform=None, index=True):
    """One sb_frame_encode_batch_device_ws call. base = (in_base, in_stride, out_base, out_stride) replaces the pointer
    arrays; uniform = (len, cap) replaces the length and cap arrays. Returns rc, [(status, out_len)], the index tensor."""
    import torch
    n = len(lens)
    if in_bytes is None:
        in_bytes = sum(k for k, c in zip(lens, caps) if k > BLOCK and c >= frame_max_len(k))
    t_ol = torch.full((n + 1,), -1, dtype=torch.int32, device="cuda")
    t_st = torch.full((max(n, 1) * 32,), 0x77, dtype=torch.uint8, device="cuda")
    _, nidx = index_bases(lens)
    t_idx = torch.full((nidx + 4,), IDX_FILL, dtype=torch.int64, device="cuda")
    b = snap._lib.SbBatch()
    if base is None:
        t_ip = torch.tensor(list(in_ptrs) + [0], dtype=torch.int64, device="cuda")
        t_op = torch.tensor(list(out_ptrs) + [0], dtype=torch.int64, device="cuda")
        b.in_ptrs, b.out_ptrs = t_ip.data_ptr(), t_op.data_ptr()
    else:
        b.in_base, b.in_stride, b.out_base, b.out_stride = base
    if uniform is None:
        t_lens, t_caps = _u32(list(lens) + [0]), _u32(list(caps) + [0])
        b.in_lens, b.out_caps = t_lens.data_ptr(), t_caps.data_ptr()
    else:
        b.in_len_uniform, b.out_cap_uniform = uniform
    b.out_lens, b.statuses, b.count = t_ol.data_ptr(), t_st.data_ptr(), n
    need = L.sb_frame_encode_batch_scratch_bytes(n, in_bytes)
    sb = need if scratch_bytes is None else scratch_bytes
    t_scr = torch.full((sb + 4096,), 0x5A, dtype=torch.uint8, device="cuda")
    e = snap._lib.SbError()
    st = (stream or torch.cuda.current_stream()).cuda_stream
    rc = L.sb_frame_encode_batch_device_ws(C.byref(b), in_bytes, t_idx.data_ptr() if index else None, t_scr.data_ptr(), sb,
                                           st, C.byref(e))
    torch.cuda.synchronize()
    if rc:
        assert bool((t_ol == -1).all()) and bool((t_st == 0x77).all()) and bool((t_idx == IDX_FILL).all())
        return rc, None, None
    assert bool((t_scr[sb:] == 0x5A).all()), "scratch overrun"
    assert bool((t_idx[nidx:] == IDX_FILL).all()), "index overrun"
    ol = t_ol.cpu().numpy().view(np.uint32)
    assert ol[n] == 0xFFFFFFFF
    sts = np.frombuffer(t_st.cpu().numpy().tobytes(), dtype=np.uint64).reshape(-1, 4)
    res = []
    for i in range(n):
        code = int(sts[i][0] & 0xFFFFFFFF)
        res.append(((CODES.get(code, str(code)), int(sts[i][1]), int(sts[i][2])), int(ol[i])))
    return rc, res, t_idx


class Batch:
    """Units packed into one device input buffer (odd gaps, start offset `off`) and outputs of cap + 16 guard bytes."""

    def __init__(self, datas, caps=None, off=0, out_off=0, even=False):
        import torch
        self.datas = datas
        self.lens = [len(d) for d in datas]
        self.caps = list(caps) if caps is not None else [frame_max_len(k) for k in self.lens]
        iw, ow = (max(self.lens) + 7) | 1, (max(self.caps) + 21) | 1
        self.offs, at = [], off
        for d in datas:
            self.offs.append(at)
            at += iw if even else len(d) + 7
        host = np.zeros(at + 16, dtype=np.uint8)
        for o, d in zip(self.offs, datas):
            host[o:o + len(d)] = np.frombuffer(d, dtype=np.uint8)
        self.t_in = torch.from_numpy(host).cuda()
        self.ooffs, at = [], out_off
        for c in self.caps:
            self.ooffs.append(at)
            at += ow if even else c + 16 + 5
        self.out_total = at + 16
        self.bases, _ = index_bases(self.lens)

    def run(self, L, snap, addressing="ptrs", **kw):
        import torch
        t_out = torch.full((self.out_total,), 0xEE, dtype=torch.uint8, device="cuda")
        if addressing == "ptrs":
            rc, res, t_idx = encode_ws(L, snap, [self.t_in.data_ptr() + o for o in self.offs], self.lens,
                                       [t_out.data_ptr() + o for o in self.ooffs], self.caps, **kw)
        else:
            n = len(self.lens)
            stride = self.offs[1] - self.offs[0] if n > 1 else 0
            ostride = self.ooffs[1] - self.ooffs[0] if n > 1 else 0
            rc, res, t_idx = encode_ws(L, snap, None, self.lens, None, self.caps,
                                       base=(self.t_in.data_ptr() + self.offs[0], stride, t_out.data_ptr() + self.ooffs[0],
                                             ostride), **kw)
        if res is not None:
            for i, c in enumerate(self.caps):                          # nothing written past a cap
                o = self.ooffs[i]
                assert bool((t_out[o + c:o + c + 16] == 0xEE).all()), i
        return rc, res, t_out, t_idx

    def out_bytes(self, t_out, i, k):
        return bytes(t_out[self.ooffs[i]:self.ooffs[i] + k].cpu().numpy())

    def index(self, t_idx, i):
        b = self.bases[i]
        return [int(x) for x in t_idx[b:b + chunks(self.lens[i]) + 1].cpu()]


def check_oracle(oracle, b, res, t_out, t_idx=None):
    for i, d in enumerate(b.datas):
        n = len(d)
        if n and b.caps[i] < frame_max_len(n):
            assert res[i] == (("BufferTooSmall", b.caps[i], frame_max_len(n)), 0), i
            assert bool((t_out[b.ooffs[i]:b.ooffs[i] + b.caps[i]] == 0xEE).all()), i
            if t_idx is not None:
                assert all(x == IDX_FILL for x in b.index(t_idx, i)), i
            continue
        want = oracle.frame_encode(d) if n else b""
        assert res[i] == (("Ok", 0, 0), len(want)), (i, n)
        assert b.out_bytes(t_out, i, len(want)) == want, (i, n)
        if t_idx is not None:
            ix = b.index(t_idx, i)
            assert ix[-1] == len(want) and ix[0] == (10 if n else 0), i
            for k in ix[:-1]:
                assert want[k] in (0, 1), (i, k)


def host_frame_encode(L, snap, d):
    """Host sb_frame_encode."""
    out = (C.c_uint8 * max(frame_max_len(len(d)), 1))()
    m, e = C.c_size_t(0), snap._lib.SbError()
    assert L.sb_frame_encode(d if d else None, len(d), out, len(out), C.byref(m), C.byref(e)) == 0
    return bytes(out[:m.value])


EDGE_LENGTHS = (0, 1, 16, 17, BLOCK - 1, BLOCK, BLOCK + 1, 2 * BLOCK, 3 * BLOCK + 1)
CORPUS = ("alice29.txt", "lcet10.txt", "urls.10K", "kppkn.gtb", "fireworks.jpeg", "geo.protodata", "html_x_4")


def _mixed():
    datas = [_text(n, i) for i, n in enumerate(EDGE_LENGTHS)] + [corpus(c) for c in CORPUS]
    rng = np.random.default_rng(3)
    datas += [rng.integers(0, 256, 2 * BLOCK + 999, dtype=np.uint8).tobytes(), rng.integers(0, 256, 900, dtype=np.uint8).tobytes(),
              bytes(3 * BLOCK + 5), bytes(BLOCK)]
    caps = [frame_max_len(len(d)) for d in datas]
    for n in (5 * BLOCK + 3, BLOCK + 1, BLOCK, 100):
        datas.append(_text(n, 9))
        caps.append(frame_max_len(n) - 1)
    return datas, caps


def test_mixed_batch_matches_oracle_host_and_single_stream_encoder(snap, oracle):
    import gpu_helpers
    L = snap._lib.lib()
    datas, caps = _mixed()
    b = Batch(datas, caps)
    rc, res, t_out, t_idx = b.run(L, snap)
    assert rc == 0
    check_oracle(oracle, b, res, t_out, t_idx)
    for i, d in enumerate(datas):
        if res[i][0][0] != "Ok":
            continue
        got = b.out_bytes(t_out, i, res[i][1])
        assert got == host_frame_encode(L, snap, d), i
        stream, offs, r = gpu_helpers.frame_encode_device_ws(d)
        assert got == stream and b.index(t_idx, i) == offs, i


def test_round_trip_through_the_decoder(snap, oracle):
    """Every unit decodes to its input with sb_frame_decode_device_ws, given the batch's index and without one."""
    import gpu_helpers
    L = snap._lib.lib()
    datas, caps = _mixed()
    b = Batch(datas, caps)
    rc, res, t_out, t_idx = b.run(L, snap)
    assert rc == 0
    for i, d in enumerate(datas):
        if res[i][0][0] != "Ok" or not d:
            continue
        stream = b.out_bytes(t_out, i, res[i][1])
        for index in (b.index(t_idx, i), None):
            status, got = gpu_helpers.frame_decode_device(stream, len(d), index=index, ws=True)
            assert status == ("Ok", 0, 0, 0) and got == d, (i, index is None)


def _device_text(total):
    """A device text of `total` bytes (the corpus repeated)."""
    import torch
    base = torch.frombuffer(bytearray(_base()), dtype=torch.uint8).cuda()
    return base.repeat(total // base.numel() + 1)[:total].contiguous()


def _single_stream(L, snap, t_in, n, scratch):
    """sb_frame_encode_device_ws of one device unit: (stream tensor, index tensor)."""
    import torch
    t_o = torch.empty(frame_max_len(n), dtype=torch.uint8, device="cuda")
    t_x = torch.empty(chunks(n) + 1, dtype=torch.int64, device="cuda")
    t_r = torch.zeros(64, dtype=torch.uint8, device="cuda")
    e = snap._lib.SbError()
    assert L.sb_frame_encode_device_ws(t_in.data_ptr(), n, t_o.data_ptr(), t_o.numel(), 1, t_x.data_ptr(), t_r.data_ptr(),
                                       scratch.data_ptr(), scratch.numel(), torch.cuda.current_stream().cuda_stream,
                                       C.byref(e)) == 0
    return t_o[:int(t_x[-1])], t_x


def _scale(snap, count, n):
    """count units of n text bytes (distinct offsets into a device text) through the batch, each compared on the device
    with sb_frame_encode_device_ws of the same unit (stream and index)."""
    import torch
    L = snap._lib.lib()
    text = _device_text(n + 8 * MIB)
    t_in = torch.empty(count * n, dtype=torch.uint8, device="cuda")
    e = snap._lib.SbError()
    st = torch.cuda.current_stream().cuda_stream
    assert L.sb_generate_blocks_device(text.data_ptr(), text.numel(), t_in.data_ptr(), n, n, 0, count, 1_000_003, st,
                                       C.byref(e)) == 0
    cap = frame_max_len(n)
    t_c = torch.full((count * cap,), 0xEE, dtype=torch.uint8, device="cuda")
    rc, res, t_idx = encode_ws(L, snap, None, [n] * count, None, [cap] * count, base=(t_in.data_ptr(), n, t_c.data_ptr(), cap),
                               uniform=(n, cap))
    assert rc == 0 and all(r[0] == ("Ok", 0, 0) for r in res)
    scratch = torch.empty(L.sb_frame_encode_scratch_bytes(n), dtype=torch.uint8, device="cuda")
    k = chunks(n) + 1
    for i in range(count):
        s, x = _single_stream(L, snap, t_in[i * n:(i + 1) * n], n, scratch)
        assert res[i][1] == s.numel(), i
        assert torch.equal(t_c[i * cap:i * cap + s.numel()], s), i
        assert torch.equal(t_idx[i * k:(i + 1) * k], x), i


def test_512_units_of_1mib(snap):
    _scale(snap, 512, MIB)


def test_64_units_of_16mib(snap):
    _scale(snap, 64, 16 * MIB)


def test_largest_unit_and_the_first_too_small(snap, oracle):
    """n = 3,679,453,184 (56,144 chunks, sb_frame_max_len 4,294,903,722) is encoded; one byte more needs a cap over
    u32 and is BufferTooSmall, untouched. Both inputs are the same real tensor of n + 1 bytes; the rejected unit's output
    is a real 4 KB buffer."""
    import torch
    L = snap._lib.lib()
    blocks = [_text(BLOCK, 100 + j) for j in range(7)]
    period = torch.frombuffer(bytearray(b"".join(blocks)), dtype=torch.uint8).cuda()
    t_in = period.repeat((MAX_OK + 1) // period.numel() + 1)[:MAX_OK + 1]
    cap = frame_max_len(MAX_OK)
    assert cap == 4_294_903_722 and frame_max_len(MAX_OK + 1) > 0xFFFFFFFF
    t_out = torch.full((cap + 16,), 0xEE, dtype=torch.uint8, device="cuda")
    t_small = torch.full((4096,), 0xEE, dtype=torch.uint8, device="cuda")
    rc, res, t_idx = encode_ws(L, snap, [t_in.data_ptr()] * 2, [MAX_OK, MAX_OK + 1], [t_out.data_ptr(), t_small.data_ptr()],
                               [cap, 4080])
    assert rc == 0
    assert res[1] == (("BufferTooSmall", 4080, frame_max_len(MAX_OK + 1)), 0)
    assert bool((t_small == 0xEE).all())
    nk = chunks(MAX_OK) + 1
    assert bool((t_idx[nk:] == IDX_FILL).all())
    assert bool((t_out[cap:] == 0xEE).all())
    got = res[0][1]
    # the oracle on the first and the last 16 chunks
    head = oracle.frame_encode(bytes(t_in[:16 * BLOCK].cpu().numpy()))
    ix = t_idx[:nk].cpu().numpy()
    assert bytes(t_out[:ix[16]].cpu().numpy()) == head
    tail = oracle.frame_encode(bytes(t_in[MAX_OK - 16 * BLOCK:MAX_OK].cpu().numpy()))
    assert ix[-1] == got and bytes(t_out[ix[nk - 17]:got].cpu().numpy()) == tail[10:]
    # sb_frame_encode_device_ws of the same unit, on the device
    del t_small
    scratch = torch.empty(L.sb_frame_encode_scratch_bytes(MAX_OK), dtype=torch.uint8, device="cuda")
    s, x = _single_stream(L, snap, t_in[:MAX_OK], MAX_OK, scratch)
    del scratch
    assert s.numel() == got
    assert torch.equal(t_out[:got], s) and torch.equal(t_idx[:nk], x)


@pytest.mark.parametrize("addressing", ["ptrs", "base"])
def test_unaligned_buffers(snap, oracle, addressing):
    L = snap._lib.lib()
    datas = [_text(13 * BLOCK + 7, 1), _text(3 * BLOCK, 2), _text(500, 3), _text(2 * BLOCK + 1, 4)]
    for off in range(1, 16):
        b = Batch(datas, off=off, out_off=16 - off, even=addressing == "base")
        rc, res, t_out, t_idx = b.run(L, snap, addressing=addressing)
        assert rc == 0, off
        check_oracle(oracle, b, res, t_out, t_idx)


def test_count_zero_and_one(snap, oracle):
    import torch
    L = snap._lib.lib()
    b = snap._lib.SbBatch()
    t_ol = torch.zeros(4, dtype=torch.int32, device="cuda")
    b.out_lens, b.count = t_ol.data_ptr(), 0
    e = snap._lib.SbError()
    t_scr = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    before = L.sb_launch_count()
    assert L.sb_frame_encode_batch_device_ws(C.byref(b), 0, None, t_scr.data_ptr(), 4096, None, C.byref(e)) == 0
    assert L.sb_launch_count() == before
    for d in (_text(7 * BLOCK + 3, 9), _text(BLOCK, 8), b"", _text(33, 7)):
        bt = Batch([d])
        rc, res, t_out, t_idx = bt.run(L, snap)
        assert rc == 0
        check_oracle(oracle, bt, res, t_out, t_idx)


def test_short_scratch_underestimated_in_bytes_and_null_pointers(snap, oracle):
    import torch
    L = snap._lib.lib()
    datas = [_text(4 * BLOCK + i, i) for i in range(3)] + [_text(BLOCK, 5), b"abc", b""]
    b = Batch(datas)
    total = sum(len(d) for d in datas[:3])
    need = L.sb_frame_encode_batch_scratch_bytes(len(datas), total)
    before = L.sb_launch_count()
    rc, _, _, _ = b.run(L, snap, scratch_bytes=need - 1)
    assert rc == INVALID and L.sb_launch_count() == before
    rc, res, t_out, t_idx = b.run(L, snap, in_bytes=total - 1)
    assert rc == 0
    for i in range(3):
        assert res[i] == (("Invalid", total, total - 1), 0), i
        assert bool((t_out[b.ooffs[i]:b.ooffs[i] + b.caps[i]] == 0xEE).all()), i
        assert all(x == IDX_FILL for x in b.index(t_idx, i)), i
    for i in (3, 4, 5):
        want = oracle.frame_encode(datas[i]) if datas[i] else b""
        assert res[i] == (("Ok", 0, 0), len(want)) and b.out_bytes(t_out, i, len(want)) == want
    rc, res, t_out, t_idx = b.run(L, snap)
    check_oracle(oracle, b, res, t_out, t_idx)
    # null batch, out_lens or scratch; count >= 2^31; a bound no launch takes
    e = snap._lib.SbError()
    t_ol = torch.zeros(4, dtype=torch.int32, device="cuda")
    t_scr = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    bb = snap._lib.SbBatch()
    bb.out_lens, bb.count, bb.in_len_uniform, bb.out_cap_uniform = t_ol.data_ptr(), 1, 3, 100
    before = L.sb_launch_count()
    assert L.sb_frame_encode_batch_device_ws(None, 0, None, t_scr.data_ptr(), 4096, None, C.byref(e)) == INVALID
    assert L.sb_frame_encode_batch_device_ws(C.byref(bb), 0, None, None, 4096, None, C.byref(e)) == INVALID
    bb.count = 1 << 31
    assert L.sb_frame_encode_batch_device_ws(C.byref(bb), 0, None, t_scr.data_ptr(), 4096, None, C.byref(e)) == INVALID
    assert L.sb_frame_encode_batch_scratch_bytes(0xFFFFFFFF >> 1, 1 << 48) == 2 ** 64 - 1
    bb.count, bb.out_lens = 1, None
    assert L.sb_frame_encode_batch_device_ws(C.byref(bb), 0, None, t_scr.data_ptr(), 4096, None, C.byref(e)) == INVALID
    assert L.sb_launch_count() == before and bool((t_ol == 0).all())


def test_enqueued_behind_pending_work_on_a_side_stream(snap, oracle):
    import torch
    L = snap._lib.lib()
    datas = [_text(9 * BLOCK + i, i) for i in range(8)] + [_text(1000, 8)]
    b = Batch(datas)
    src = b.t_in.clone()
    b.t_in.zero_()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)
        b.t_in.copy_(src)                                              # the input is written by work still pending
        rc, res, t_out, t_idx = b.run(L, snap, stream=side)
    assert rc == 0
    check_oracle(oracle, b, res, t_out, t_idx)


def test_no_allocation_in_the_steady_state(snap, oracle):
    L = snap._lib.lib()
    datas = [_text(3 * BLOCK + 17 * i, i) for i in range(4)] + [_text(900, 5)]
    b = Batch(datas)
    rc, res0, t0, _ = b.run(L, snap)
    assert rc == 0
    before = L.sb_alloc_count()
    for _ in range(3):
        rc, res, t1, _ = b.run(L, snap)
        assert rc == 0 and res == res0
        assert bool((t1 == t0).all())
    assert L.sb_alloc_count() == before


def test_python_encode_batch(snap, oracle):
    units = [b"", b"x", bytearray(_text(BLOCK, 1)), memoryview(_text(3 * BLOCK + 11, 2)),
             np.frombuffer(_text(2 * BLOCK, 3), dtype=np.uint8), np.frombuffer(_text(4000, 4), dtype=np.uint32),
             bytes(BLOCK + 1), b""]
    got = snap.frame.encode_batch(units)
    assert len(got) == len(units)
    for u, g in zip(units, got):
        d = bytes(memoryview(u).cast("B"))
        assert g == (oracle.frame_encode(d) if d else b"")
    assert snap.frame.encode_batch([]) == []
