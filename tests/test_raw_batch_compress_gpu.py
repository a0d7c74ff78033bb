"""Raw compress of a batch of units of any length on the GPU (sb_compress_batch_device_ws): every unit's 64 KB blocks
go through one K1 launch and each unit is assembled in its output. Every unit must equal the oracle's
Encoder::compress and host sb_compress byte for byte, or carry the reference's exact error; units of at most 64 KB must
also equal sb_compress_batch_device's bytes, and large units must decode block-parallel through
sb_decompress_batch_device_ws."""
import ctypes as C

import numpy as np
import pytest

from conftest import corpus

pytestmark = pytest.mark.gpu

BLOCK = 65536
MIB = 1 << 20
INVALID = 202
MAX_OK = 3_681_400_511                 # the largest n with max_compress_len(n) != 0
CODES = {0: "Ok", 1: "TooBig", 2: "BufferTooSmall", INVALID: "Invalid"}


@pytest.fixture(scope="module")
def snap():
    import torch
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)
    import gpu_helpers
    return gpu_helpers.snap()


def max_compress_len(n):
    m = 32 + n + n // 6
    return 0 if m > 0xFFFFFFFF else m


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


def compress_ws(L, snap, in_ptrs, lens, out_ptrs, caps, in_bytes=None, scratch_bytes=None, stream=None, base=None,
                uniform=None):
    """One sb_compress_batch_device_ws call. base = (in_base, in_stride, out_base, out_stride) replaces the pointer arrays;
    uniform = (len, cap) replaces the length and cap arrays. Returns rc, [(status, out_len)], the scratch tensor."""
    import torch
    n = len(lens)
    if in_bytes is None:
        in_bytes = sum(k for k, c in zip(lens, caps) if k > BLOCK and 0 < max_compress_len(k) <= c)
    t_ol = torch.full((n + 1,), -1, dtype=torch.int32, device="cuda")
    t_st = torch.full((max(n, 1) * 32,), 0x77, dtype=torch.uint8, device="cuda")
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
    need = L.sb_compress_batch_scratch_bytes(n, in_bytes)
    sb = need if scratch_bytes is None else scratch_bytes
    t_scr = torch.full((sb + 4096,), 0x5A, dtype=torch.uint8, device="cuda")
    e = snap._lib.SbError()
    st = (stream or torch.cuda.current_stream()).cuda_stream
    rc = L.sb_compress_batch_device_ws(C.byref(b), in_bytes, t_scr.data_ptr(), sb, st, C.byref(e))
    torch.cuda.synchronize()
    if rc:
        assert bool((t_ol == -1).all()) and bool((t_st == 0x77).all())
        return rc, None, t_scr
    assert bool((t_scr[sb:] == 0x5A).all()), "scratch overrun"
    ol = t_ol.cpu().numpy().view(np.uint32)
    assert ol[n] == 0xFFFFFFFF
    sts = np.frombuffer(t_st.cpu().numpy().tobytes(), dtype=np.uint64).reshape(-1, 4)
    res = []
    for i in range(n):
        code = int(sts[i][0] & 0xFFFFFFFF)
        res.append(((CODES.get(code, str(code)), int(sts[i][1]), int(sts[i][2])), int(ol[i])))
    return rc, res, t_scr


class Batch:
    """Units packed into one device input buffer (odd gaps, start offset `off`) and outputs of cap + 16 guard bytes."""

    def __init__(self, datas, caps=None, off=0, out_off=0, even=False):
        import torch
        self.datas = datas
        self.lens = [len(d) for d in datas]
        self.caps = list(caps) if caps is not None else [max_compress_len(k) for k in self.lens]
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

    def run(self, L, snap, addressing="ptrs", **kw):
        import torch
        t_out = torch.full((self.out_total,), 0xEE, dtype=torch.uint8, device="cuda")
        if addressing == "ptrs":
            rc, res, _ = compress_ws(L, snap, [self.t_in.data_ptr() + o for o in self.offs], self.lens,
                                     [t_out.data_ptr() + o for o in self.ooffs], self.caps, **kw)
        else:
            n = len(self.lens)
            stride = self.offs[1] - self.offs[0] if n > 1 else 0
            ostride = self.ooffs[1] - self.ooffs[0] if n > 1 else 0
            rc, res, _ = compress_ws(L, snap, None, self.lens, None, self.caps,
                                     base=(self.t_in.data_ptr() + self.offs[0], stride, t_out.data_ptr() + self.ooffs[0],
                                           ostride), **kw)
        if res is not None:
            for i, c in enumerate(self.caps):                          # nothing written past a cap
                o = self.ooffs[i]
                assert bool((t_out[o + c:o + c + 16] == 0xEE).all()), i
        return rc, res, t_out

    def out_bytes(self, t_out, i, k):
        return bytes(t_out[self.ooffs[i]:self.ooffs[i] + k].cpu().numpy())


def check_oracle(oracle, b, res, t_out):
    for i, d in enumerate(b.datas):
        need = max_compress_len(len(d))
        if b.caps[i] < need:
            assert res[i] == (("BufferTooSmall", b.caps[i], need), 0), i
            assert bool((t_out[b.ooffs[i]:b.ooffs[i] + b.caps[i]] == 0xEE).all()), i
            continue
        want = oracle.compress(d)
        assert res[i] == (("Ok", 0, 0), len(want)), (i, len(d))
        assert b.out_bytes(t_out, i, len(want)) == want, (i, len(d))


EDGE_LENGTHS = (0, 1, 16, 17, BLOCK - 1, BLOCK, BLOCK + 1, BLOCK + 16, BLOCK + 17, 2 * BLOCK, 3 * BLOCK + 1)
CORPUS = ("alice29.txt", "lcet10.txt", "urls.10K", "kppkn.gtb", "fireworks.jpeg", "geo.protodata", "html_x_4")


def _mixed():
    datas = [_text(n, i) for i, n in enumerate(EDGE_LENGTHS)] + [corpus(c) for c in CORPUS]
    rng = np.random.default_rng(3)
    datas += [rng.integers(0, 256, 2 * BLOCK + 999, dtype=np.uint8).tobytes(), bytes(3 * BLOCK + 5), bytes(BLOCK)]
    caps = [max_compress_len(len(d)) for d in datas]
    for n in (5 * BLOCK + 3, BLOCK + 1, BLOCK, 100, 0):
        datas.append(_text(n, 9))
        caps.append(max_compress_len(n) - 1)
    return datas, caps


def test_mixed_batch_matches_oracle_sb_compress_and_batch_device(snap, oracle):
    import torch
    L = snap._lib.lib()
    datas, caps = _mixed()
    b = Batch(datas, caps)
    rc, res, t_out = b.run(L, snap)
    assert rc == 0
    check_oracle(oracle, b, res, t_out)
    enc = snap.raw.Encoder()
    for i, d in enumerate(datas):
        if res[i][0][0] == "Ok":
            assert b.out_bytes(t_out, i, res[i][1]) == enc.compress_vec(d), i
    # the units of at most 64 KB through sb_compress_batch_device (K1 with its own header) give the same bytes
    small = [i for i, d in enumerate(datas) if len(d) <= BLOCK and res[i][0][0] == "Ok"]
    stride = 76544
    t_in = torch.zeros(len(small) * BLOCK + 16, dtype=torch.uint8, device="cuda")
    for k, i in enumerate(small):
        if datas[i]:
            t_in[k * BLOCK:k * BLOCK + len(datas[i])] = torch.frombuffer(bytearray(datas[i]), dtype=torch.uint8).cuda()
    t_o = torch.zeros(len(small) * stride, dtype=torch.uint8, device="cuda")
    t_ol = torch.zeros(len(small), dtype=torch.int32, device="cuda")
    t_l = torch.tensor([len(datas[i]) for i in small], dtype=torch.int32, device="cuda")
    import gpu_helpers
    bb = gpu_helpers.batch_from_tensors(t_in, BLOCK, 0, t_o, stride, stride, t_ol, None, len(small), in_lens_t=t_l)
    e = snap._lib.SbError()
    assert L.sb_compress_batch_device(C.byref(bb), torch.cuda.current_stream().cuda_stream, C.byref(e)) == 0
    torch.cuda.synchronize()
    for k, i in enumerate(small):
        got = bytes(t_o[k * stride:k * stride + int(t_ol[k])].cpu().numpy())
        assert got == b.out_bytes(t_out, i, res[i][1]), i


def _device_text(total):
    """A device text of `total` bytes (the corpus repeated)."""
    import torch
    base = torch.frombuffer(bytearray(_base()), dtype=torch.uint8).cuda()
    return base.repeat(total // base.numel() + 1)[:total].contiguous()


def _round_trip(snap, count, n):
    """count units of n text bytes (distinct offsets into a device text) compressed by sb_compress_batch_device_ws and
    decoded by sb_decompress_batch_device_ws: every unit decodes block-parallel to its input; two equal host sb_compress."""
    import torch
    L = snap._lib.lib()
    text = _device_text(n + 8 * MIB)
    t_in = torch.empty(count * n, dtype=torch.uint8, device="cuda")
    e = snap._lib.SbError()
    st = torch.cuda.current_stream().cuda_stream
    assert L.sb_generate_blocks_device(text.data_ptr(), text.numel(), t_in.data_ptr(), n, n, 0, count, 1_000_003, st,
                                       C.byref(e)) == 0
    cap = max_compress_len(n)
    t_c = torch.full((count * cap,), 0xEE, dtype=torch.uint8, device="cuda")
    rc, res, _ = compress_ws(L, snap, None, [n] * count, None, [cap] * count,
                             base=(t_in.data_ptr(), n, t_c.data_ptr(), cap), uniform=(n, cap))
    assert rc == 0 and all(r[0] == ("Ok", 0, 0) for r in res)
    clens = [r[1] for r in res]
    # decode: unit i reads its stream in place
    t_ip = torch.tensor([t_c.data_ptr() + i * cap for i in range(count)], dtype=torch.int64, device="cuda")
    t_il = torch.tensor(clens, dtype=torch.int32, device="cuda")
    t_d = torch.zeros(count * n, dtype=torch.uint8, device="cuda")
    t_dl = torch.zeros(count, dtype=torch.int32, device="cuda")
    t_blk = torch.zeros(count, dtype=torch.int32, device="cuda")
    t_st = torch.zeros(count * 32, dtype=torch.uint8, device="cuda")
    b = snap._lib.SbBatch()
    b.in_ptrs, b.in_lens = t_ip.data_ptr(), t_il.data_ptr()
    b.out_base, b.out_stride, b.out_cap_uniform = t_d.data_ptr(), n, n
    b.out_lens, b.statuses, b.count = t_dl.data_ptr(), t_st.data_ptr(), count
    need = L.sb_decompress_batch_scratch_bytes(count, sum(clens))
    t_scr = torch.empty(need, dtype=torch.uint8, device="cuda")
    assert L.sb_decompress_batch_device_ws(C.byref(b), sum(clens), t_blk.data_ptr(), t_scr.data_ptr(), need, st,
                                           C.byref(e)) == 0
    torch.cuda.synchronize()
    assert bool((t_blk == (n + BLOCK - 1) // BLOCK).all()) and bool((t_dl == n).all())
    assert bool((t_st == 0).all())
    assert torch.equal(t_d, t_in)
    enc = snap.raw.Encoder()
    for i in (0, count - 1):
        data = bytes(t_in[i * n:(i + 1) * n].cpu().numpy())
        assert bytes(t_c[i * cap:i * cap + clens[i]].cpu().numpy()) == enc.compress_vec(data), i


def test_512_units_of_1mib_round_trip(snap):
    _round_trip(snap, 512, MIB)


def test_64_units_of_16mib_round_trip(snap):
    _round_trip(snap, 64, 16 * MIB)


def test_largest_unit_and_the_first_too_big(snap, oracle):
    """n = 3,681,400,511 (max_compress_len 4,294,967,294) compresses; one byte more is TooBig and untouched. Both units
    are cut from one real 3.68 GB tensor, a period of 7 distinct 64 KB text blocks, so the expected stream is
    varint(n) + body[j % 7] for every full block + the body of the remainder."""
    import torch
    L = snap._lib.lib()
    blocks = [_text(BLOCK, 100 + j) for j in range(7)]
    period = torch.frombuffer(bytearray(b"".join(blocks)), dtype=torch.uint8).cuda()
    t_in = period.repeat((MAX_OK + 1) // period.numel() + 1)[:MAX_OK + 1]
    cap = max_compress_len(MAX_OK)
    assert cap == 4_294_967_294 and max_compress_len(MAX_OK + 1) == 0
    t_out = torch.full((cap + 16,), 0xEE, dtype=torch.uint8, device="cuda")
    t_small = torch.full((4096,), 0xEE, dtype=torch.uint8, device="cuda")
    rc, res, t_scr = compress_ws(L, snap, [t_in.data_ptr()] * 2, [MAX_OK, MAX_OK + 1], [t_out.data_ptr(), t_small.data_ptr()],
                                 [cap, 4080])
    del t_scr
    assert rc == 0
    assert res[1] == (("TooBig", MAX_OK + 1, 0xFFFFFFFF), 0)
    assert bool((t_small == 0xEE).all())
    nfull, rem = divmod(MAX_OK, BLOCK)
    bodies = [oracle.compress(blk)[3:] for blk in blocks]                # varint(65536) is 3 bytes
    tail = oracle.compress(blocks[nfull % 7][:rem])[3:]                  # varint(46,783) is 3 bytes
    hdr = bytes([(MAX_OK >> (7 * k)) & 0x7F | (0x80 if k < 4 else 0) for k in range(5)])
    want_len = len(hdr) + (nfull // 7) * sum(len(x) for x in bodies) + sum(len(x) for x in bodies[:nfull % 7]) + len(tail)
    assert res[0] == (("Ok", 0, 0), want_len)
    assert bool((t_out[want_len:] == 0xEE).all())
    dev = lambda x: torch.frombuffer(bytearray(x), dtype=torch.uint8).cuda()
    at = len(hdr)
    assert bytes(t_out[:at].cpu().numpy()) == hdr
    rep = dev(b"".join(bodies))
    span = (nfull // 7) * rep.numel()
    assert torch.equal(t_out[at:at + span].view(nfull // 7, rep.numel()), rep.expand(nfull // 7, rep.numel()))
    at += span
    rest = dev(b"".join(bodies[:nfull % 7]) + tail)
    assert torch.equal(t_out[at:want_len], rest)


@pytest.mark.parametrize("addressing", ["ptrs", "base"])
def test_unaligned_buffers(snap, oracle, addressing):
    L = snap._lib.lib()
    datas = [_text(13 * BLOCK + 7, 1), _text(3 * BLOCK, 2), _text(500, 3), _text(2 * BLOCK + 1, 4)]
    for off in range(1, 16):
        b = Batch(datas, off=off, out_off=16 - off, even=addressing == "base")
        rc, res, t_out = b.run(L, snap, addressing=addressing)
        assert rc == 0, off
        check_oracle(oracle, b, res, t_out)


def test_uniform_length_over_64k(snap, oracle):
    L = snap._lib.lib()
    n = 5 * BLOCK + 333
    datas = [_text(n, 20 + i) for i in range(6)]
    b = Batch(datas, even=True)
    rc, res, t_out = b.run(L, snap, addressing="base", uniform=(n, max_compress_len(n)))
    assert rc == 0
    check_oracle(oracle, b, res, t_out)


def test_count_zero_and_one(snap, oracle):
    import torch
    L = snap._lib.lib()
    b = snap._lib.SbBatch()
    t_ol = torch.zeros(4, dtype=torch.int32, device="cuda")
    b.out_lens, b.count = t_ol.data_ptr(), 0
    e = snap._lib.SbError()
    t_scr = torch.zeros(4096, dtype=torch.uint8, device="cuda")
    before = L.sb_launch_count()
    assert L.sb_compress_batch_device_ws(C.byref(b), 0, t_scr.data_ptr(), 4096, None, C.byref(e)) == 0
    assert L.sb_launch_count() == before
    enc = snap.raw.Encoder()
    for d in (_text(7 * BLOCK + 3, 9), _text(BLOCK, 8), b"", _text(33, 7)):
        bt = Batch([d])
        rc, res, t_out = bt.run(L, snap)
        assert rc == 0
        want = enc.compress_vec(d)
        assert res[0] == (("Ok", 0, 0), len(want)) and bt.out_bytes(t_out, 0, len(want)) == want


def test_short_scratch_and_underestimated_in_bytes(snap, oracle):
    L = snap._lib.lib()
    datas = [_text(4 * BLOCK + i, i) for i in range(3)] + [_text(BLOCK, 5), b"abc"]
    b = Batch(datas)
    total = sum(len(d) for d in datas[:3])
    need = L.sb_compress_batch_scratch_bytes(len(datas), total)
    before = L.sb_launch_count()
    rc, _, _ = b.run(L, snap, scratch_bytes=need - 1)
    assert rc == INVALID and L.sb_launch_count() == before
    rc, res, t_out = b.run(L, snap, in_bytes=total - 1)
    assert rc == 0
    for i in range(3):
        assert res[i] == (("Invalid", total, total - 1), 0), i
        assert bool((t_out[b.ooffs[i]:b.ooffs[i] + b.caps[i]] == 0xEE).all()), i
    for i in (3, 4):
        want = oracle.compress(datas[i])
        assert res[i] == (("Ok", 0, 0), len(want)) and b.out_bytes(t_out, i, len(want)) == want
    rc, res, t_out = b.run(L, snap)
    check_oracle(oracle, b, res, t_out)


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
        rc, res, t_out = b.run(L, snap, stream=side)
    assert rc == 0
    check_oracle(oracle, b, res, t_out)


def test_no_allocation_in_the_steady_state(snap, oracle):
    L = snap._lib.lib()
    datas = [_text(3 * BLOCK + 17 * i, i) for i in range(4)] + [_text(900, 5)]
    b = Batch(datas)
    rc, res0, t0 = b.run(L, snap)
    assert rc == 0
    before = L.sb_alloc_count()
    for _ in range(3):
        rc, res, t1 = b.run(L, snap)
        assert rc == 0 and res == res0
        assert bool((t1 == t0).all())
    assert L.sb_alloc_count() == before
