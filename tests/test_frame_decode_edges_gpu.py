"""Frame decode, K3's CRC-32C and the warp copy on the GPU at the alignment, length and chunk-count edges where the kernels
branch: the K3 batch API at every base offset and near 4 GiB, frame encode from unaligned device input, the decoder at
every (input, output) alignment pair, chunk counts around the scan tiles (up to the branch where one thread sums several
tiles), and a chunk table too small for the stream. Everything goes through the C ABI and is compared with the C oracle
(plus a bitwise CRC on a subset) or a Python walk of the stream."""
import ctypes as C
import random

import numpy as np
import pytest

from conftest import corpus
from test_crc_copy_emu import EDGE_LENS, aligned, crc_units, fill, masked, tiny_stream
from test_frame_index_emu import IDENT, chunk, oracle_decode, walk

pytestmark = pytest.mark.gpu

NAMES = {0: "Ok", 2: "BufferTooSmall", 14: "Checksum", 100: "UnexpectedEof", 202: "Invalid"}


@pytest.fixture(scope="module")
def snap():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA GPU")
    import gpu_helpers
    return gpu_helpers.snap()


def _stream():
    import torch
    return torch.cuda.current_stream().cuda_stream


def _check(rc, e):
    import gpu_helpers
    if rc:
        raise gpu_helpers.snap().error.from_c(e)


def _u32(values, dev="cuda:0"):
    import torch
    return torch.from_numpy(np.asarray(values, dtype=np.uint32).view(np.int32)).to(dev)


def _orc(fn, host, off, n):
    """An oracle CRC over host[off:off + n] through a pointer (no bytes copy)."""
    return fn(C.cast(C.c_void_p(host.ctypes.data + off), C.c_char_p), n)


def k3_batch(dev_ptr, offs=None, lens=None, stride=0, count=None):
    """sb_crc32c_masked_batch_device: in_ptrs = dev_ptr + offs[i] (offs given), else in_base = dev_ptr with in_stride."""
    import torch
    import gpu_helpers
    s, L = gpu_helpers.snap(), gpu_helpers.lib()
    count = len(lens) if count is None else count
    b = s._lib.SbBatch()
    if offs is not None:
        t_ptrs = torch.tensor([dev_ptr + o for o in offs], dtype=torch.int64, device="cuda:0")
        b.in_ptrs = t_ptrs.data_ptr()
    else:
        b.in_base = dev_ptr
        b.in_stride = stride
    t_lens = _u32(lens)
    t_out = torch.full((count,), -1, dtype=torch.int32, device="cuda:0")
    b.in_lens = t_lens.data_ptr()
    b.out_lens = t_out.data_ptr()
    b.count = count
    e = s._lib.SbError()
    _check(L.sb_crc32c_masked_batch_device(C.byref(b), _stream(), C.byref(e)), e)
    torch.cuda.synchronize()
    return [int(x) & 0xFFFFFFFF for x in t_out.cpu()]


def _bad(got, want, units):
    return [(u, hex(g), hex(w)) for g, w, u in zip(got, want, units) if g != w][:8]


@pytest.mark.parametrize("kind", ["random", "zeros", "ones"])
def test_k3_batch_every_length_and_offset(snap, oracle, kind):
    """Every n in 0..700, the edge lengths, 1 MiB and 16 MiB + 3, each at base offsets 0..15: once through in_ptrs and
    once through in_base with an odd in_stride (16 consecutive units then sit at 16 different offsets)."""
    import torch
    big = [1 << 20, (16 << 20) + 3]
    lens = list(range(701)) + EDGE_LENS + big
    units, size = crc_units(lens)
    groups = [(list(range(701)), 701), (EDGE_LENS, 65537), ([1 << 20], (1 << 20) + 1), ([(16 << 20) + 3], (16 << 20) + 3)]
    size = max(size, max(16 * len(g) * s for g, s in groups))
    host = aligned(size)
    host[:] = fill(kind, size, seed=13)
    dev = torch.empty(size + 256, dtype=torch.uint8, device="cuda:0")
    dev[:size].copy_(torch.from_numpy(host))
    ptr = dev.data_ptr()
    assert ptr % 16 == 0
    L = oracle.lib()
    want = [_orc(L.orc_crc32c_masked, host, o, n) for o, n in units]
    got = k3_batch(ptr, offs=[o for o, _ in units], lens=[n for _, n in units])
    assert got == want, _bad(got, want, units)
    if kind == "random":                             # a bit-at-a-time CRC that shares no table code with either side
        sub = [(i, u) for i, u in enumerate(units) if u[1] <= 300 or (u[1] in EDGE_LENS + big and u[0] % 16 in (0, 7))]
        assert [got[i] for i, _ in sub] == [masked(_orc(L.orc_crc32c_bitwise, host, o, n)) for _, (o, n) in sub]
    for glens, stride in groups:
        assert stride % 2 == 1 and stride >= max(glens)
        ulens = [n for n in glens for _ in range(16)]
        got = k3_batch(ptr, lens=ulens, stride=stride)
        want = [_orc(L.orc_crc32c_masked, host, i * stride, n) for i, n in enumerate(ulens)]
        assert got == want, (stride, _bad(got, want, list(enumerate(ulens))))


def test_k3_batch_near_4_gib(snap, oracle):
    """One device buffer of 2^32 - 1 bytes of a repeating pattern: the CRC of its first 2^32 - 32 bytes and of all of it.
    From 2^32 - 31 bytes on, n + 31 no longer fits in 32 bits -- the slice length must not wrap."""
    import torch
    n = (1 << 32) - 1
    period = 4093
    rows = (n + period) // period
    pat = np.random.default_rng(17).integers(0, 256, period, dtype=np.uint8)
    dev = torch.empty(rows * period, dtype=torch.uint8, device="cuda:0")
    dev.view(rows, period).copy_(torch.from_numpy(pat).to("cuda:0").expand(rows, period))
    got = k3_batch(dev.data_ptr(), offs=[0, 0], lens=[n - 31, n])
    del dev
    torch.cuda.empty_cache()
    host = np.tile(pat, rows)
    L = oracle.lib()
    want = [_orc(L.orc_crc32c_masked, host, 0, n - 31), _orc(L.orc_crc32c_masked, host, 0, n)]
    del host
    assert got[0] == want[0], "2^32 - 32 bytes"
    assert got[1] == want[1], "2^32 - 1 bytes"


def _encode_ws(ptr, n):
    """sb_frame_encode_device_ws of n device bytes at ptr: (stream, chunk index)."""
    import torch
    import gpu_helpers
    s, L = gpu_helpers.snap(), gpu_helpers.lib()
    cap = L.sb_frame_max_len(n)
    t_out = torch.zeros(cap + 16, dtype=torch.uint8, device="cuda:0")
    nchunks = (n + 65535) // 65536
    t_offs = torch.zeros(nchunks + 1, dtype=torch.int64, device="cuda:0")
    t_res = torch.zeros(64, dtype=torch.uint8, device="cuda:0")
    sb = L.sb_frame_encode_scratch_bytes(n)
    t_scr = torch.empty(sb, dtype=torch.uint8, device="cuda:0")
    e = s._lib.SbError()
    _check(L.sb_frame_encode_device_ws(ptr, n, t_out.data_ptr(), cap, 1, t_offs.data_ptr(), t_res.data_ptr(), t_scr.data_ptr(), sb,
                                       _stream(), C.byref(e)), e)
    torch.cuda.synchronize()
    res = s._lib.SbFrameResult.from_buffer_copy(bytes(t_res.cpu().numpy()[:C.sizeof(s._lib.SbFrameResult)]))
    assert res.status.code == 0 and res.nchunks == nchunks
    return bytes(t_out[:res.bytes].cpu().numpy()), [int(x) for x in t_offs.cpu()]


def test_frame_encode_from_unaligned_device_input(snap, oracle):
    """d_in + k for k in 1..15: K1 with its fused single-table chunk CRC on an unaligned head, and K4's gather copying the
    raw (incompressible) chunks from d_in + i * 65536."""
    import torch
    rnd = np.random.default_rng(21).integers(0, 256, 3 * 65536, dtype=np.uint8).tobytes()
    text = corpus("lcet10.txt")
    data = text[:65536] + rnd[:65536] + text[70000:135536] + rnd[65536:131072] + rnd[131072:131072 + 777]
    want = oracle.frame_encode(data)
    kinds = [want[o] for o in walk(want)[:-1]]
    assert kinds == [0, 1, 0, 1, 1]
    n = len(data)
    t = torch.zeros(n + 64, dtype=torch.uint8, device="cuda:0")
    src = torch.frombuffer(bytearray(data), dtype=torch.uint8).to("cuda:0")
    for k in range(1, 16):
        t.zero_()
        t[k:k + n].copy_(src)
        stream, offs = _encode_ws(t.data_ptr() + k, n)
        assert stream == want, k
        assert offs == walk(stream), k


def decode_ws(t_in, a, n, t_out, b, cap, index=None, max_chunks=None, fragment=False):
    """sb_frame_decode_device_ws of the n bytes at t_in + a into t_out + b: (status tuple, bytes, nchunks)."""
    import torch
    import gpu_helpers
    s, L = gpu_helpers.snap(), gpu_helpers.lib()
    t_idx = torch.from_numpy(np.asarray(index, dtype=np.int64)).to("cuda:0") if index is not None else None
    nidx = len(index) - 1 if index is not None else 0
    maxc = max_chunks if max_chunks is not None else max(nidx + 1, n // 8 + 16)
    sb = L.sb_frame_decode_scratch_bytes(maxc)
    t_scr = torch.empty(sb, dtype=torch.uint8, device="cuda:0")
    t_res = torch.zeros(64, dtype=torch.uint8, device="cuda:0")
    e = s._lib.SbError()
    _check(L.sb_frame_decode_device_ws(t_in.data_ptr() + a, n, t_out.data_ptr() + b, cap, t_idx.data_ptr() if t_idx is not None else None,
                                       nidx, 1 if fragment else 0, t_res.data_ptr(), t_scr.data_ptr(), sb, maxc, _stream(), C.byref(e)), e)
    torch.cuda.synchronize()
    res = s._lib.SbFrameResult.from_buffer_copy(bytes(t_res.cpu().numpy()[:C.sizeof(s._lib.SbFrameResult)]))
    st = res.status
    return (NAMES.get(st.code, str(st.code)), st.a, st.b, st.c), res.bytes, res.nchunks


def _sweep_stream(oracle):
    """Uncompressed chunks with a body length on every warp-copy path, interleaved with compressed chunks whose compressed
    and decoded lengths differ, so that input and output alignments drift apart from chunk to chunk."""
    rng = random.Random(8)
    text = corpus("alice29.txt")
    raw_lens = [0, 1, 15, 16, 17, 31, 32, 33, 47, 48, 49, 63, 64, 65, 79, 80, 81, 95, 96, 97, 127, 128, 129,
                4095, 4096, 4097, 65535, 65536]
    parts, data = [], []
    for i, ln in enumerate(raw_lens):
        body = bytes(rng.getrandbits(8) for _ in range(ln))
        parts.append(chunk(1, body, oracle.crc32c_masked(body)))
        data.append(body)
        at = rng.randrange(0, len(text) - 5000)
        piece = text[at:at + rng.choice([5, 300, 1000, 2345, 4321, 9000])]
        parts.append(oracle.compress_frame(piece))
        data.append(piece)
    assert sum(p[0] == 0 and int.from_bytes(p[1:4], "little") - 4 != len(d) for p, d in zip(parts, data)) >= 15
    return IDENT + b"".join(parts), b"".join(data)


def test_decode_every_input_and_output_alignment(snap, oracle):
    """All 256 (d_in + a, d_out + b) pairs for a, b in 0..15, each with the stream's index, without one (K7) and with a
    padding chunk that forces the walk; 16 guard bytes on both sides of the output stay untouched."""
    import torch
    stream, data = _sweep_stream(oracle)
    padded = IDENT + b"\xfe\x03\x00\x00pad" + stream[10:]
    assert oracle.frame_decode(stream) == data and oracle.frame_decode(padded) == data
    nch = len(walk(stream)) - 1
    ways = [(stream, walk(stream)), (stream, None), (padded, None)]
    cap = len(data)
    want = torch.frombuffer(bytearray(data), dtype=torch.uint8).to("cuda:0")
    t_out = torch.empty(cap + 64, dtype=torch.uint8, device="cuda:0")
    for s, index in ways:
        src = torch.frombuffer(bytearray(s), dtype=torch.uint8).to("cuda:0")
        t_in = torch.zeros(len(s) + 64, dtype=torch.uint8, device="cuda:0")
        for a in range(16):
            t_in.zero_()
            t_in[a:a + len(s)].copy_(src)
            for b in range(16):
                t_out.fill_(0xEE)
                st, got, k = decode_ws(t_in, a, len(s), t_out, 16 + b, cap, index=index)
                where = (a, b, index is not None, s is padded)
                assert (st, got, k) == (("Ok", 0, 0, 0), cap, nch), where
                assert torch.equal(t_out[16 + b:16 + b + cap], want), where
                assert bool((t_out[:16 + b] == 0xEE).all()) and bool((t_out[16 + b + cap:] == 0xEE).all()), where
    assert snap.frame.decode_all(stream) == data
    assert snap.frame.decode_all(padded) == data


@pytest.mark.parametrize("count", [1, 1023, 1024, 1025, 2049, 1049601])
def test_chunk_counts_at_scan_tile_edges(snap, oracle, count):
    """Chunk counts around the 1024-chunk scan tiles. 1,049,601 chunks make 1,026 tiles, more than the 1,024 threads of
    the tile scan, so one thread sums two tiles. Index given, index built by K7, and the walk (padding chunk)."""
    import torch
    stream, offs, data = tiny_stream(oracle, count, seed=count)
    padded, _, _ = tiny_stream(oracle, count, seed=count, pad=True)
    assert oracle.frame_decode(stream) == data
    want = torch.frombuffer(bytearray(data) + bytearray(1), dtype=torch.uint8).to("cuda:0")[:len(data)]
    t_out = torch.empty(len(data) + 32, dtype=torch.uint8, device="cuda:0")
    for s, index in ((stream, offs), (stream, None), (padded, None)):
        t_in = torch.frombuffer(bytearray(s) + bytearray(16), dtype=torch.uint8).to("cuda:0")
        t_out.fill_(0xEE)
        st, got, k = decode_ws(t_in, 0, len(s), t_out, 0, len(data), index=index)
        assert (st, got, k) == (("Ok", 0, 0, 0), len(data), count), (index is not None, s is padded)
        assert torch.equal(t_out[:len(data)], want) and bool((t_out[len(data):] == 0xEE).all())


def _uncompressed_chunks(oracle, count, size, seed):
    body = np.random.default_rng(seed).integers(0, 256, count * size, dtype=np.uint8).tobytes()
    parts = [IDENT]
    for i in range(count):
        piece = body[i * size:(i + 1) * size]
        parts.append(chunk(1, piece, oracle.crc32c_masked(piece)))
    return b"".join(parts), body


def test_chunk_table_overflow_without_an_index(snap, oracle):
    """20,000 chunks of 100 bytes: more than sb_frame_decode_device's first table (n / 1024 + 4096 = 6,205), so K7 declines,
    the walk overflows the table and the call retries with a larger one. A too-small output must report the full size,
    not the size of the chunks that fit the first table."""
    import gpu_helpers
    import torch
    count, size = 20000, 100
    stream, data = _uncompressed_chunks(oracle, count, size, seed=2)
    assert len(stream) // 1024 + 4096 < count
    assert gpu_helpers.frame_decode_device(stream, len(data)) == (("Ok", 0, 0, 0), data)
    assert gpu_helpers.frame_decode_device(stream, 1000) == (("BufferTooSmall", 1000, len(data), 0), b"")
    t_in = torch.frombuffer(bytearray(stream) + bytearray(16), dtype=torch.uint8).to("cuda:0")
    t_out = torch.empty(len(data) + 16, dtype=torch.uint8, device="cuda:0")
    for cap in (1000, len(data)):
        st, got, _ = decode_ws(t_in, 0, len(stream), t_out, 0, cap, max_chunks=5000)
        assert (st, got) == (("Invalid", 5000, 1, 0), 0), cap
    offs = walk(stream)
    for bad_chunk in (100, 15000):                   # before and past the end of the first table
        bad = bytearray(stream)
        bad[offs[bad_chunk] + 8 + 37] ^= 0x01
        want_st, _ = oracle_decode(oracle, bytes(bad))
        assert want_st[0] == "Checksum"
        assert gpu_helpers.frame_decode_device(bytes(bad), len(data)) == (want_st, data[:bad_chunk * size]), bad_chunk
