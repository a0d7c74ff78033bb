"""CUDA path vs the oracle, through the C ABI (python -m pytest -m gpu).

Mirrors the reference's test/tests.rs: round trips on the corpus (raw + frame),
the golden encoder vector, decoder KATs with exact error payloads, the small
input sweeps, property round trips, and the frame encoder equivalences.
"""
import io
import random

import pytest

from conftest import CORPUS, corpus
from kats import (COPY_CLOSE_TO_END, DECODE_ERRORS, RANDOM, adversarial_blocks, small_copy_inputs,
                  small_regular_inputs)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def snap():
    import torch
    assert torch.cuda.is_available()
    torch.cuda.set_device(0)
    import gpu_helpers
    return gpu_helpers.snap()


def press(snap, d):
    return snap.raw.Encoder().compress_vec(d)


def depress(snap, d):
    return snap.raw.Decoder().decompress_vec(d)


def test_golden_rev(snap, oracle):
    # test/tests.rs:199-205
    gold = corpus("Mark.Twain-Tom.Sawyer.txt.rawsnappy")
    assert press(snap, depress(snap, gold)) == gold


@pytest.mark.parametrize("name", CORPUS)
def test_corpus_raw_bit_exact_and_roundtrip(snap, oracle, name):
    # testtrip!(data_*): roundtrip_raw + compressed bytes equal to the reference encoder (oracle)
    data = corpus(name)
    c = press(snap, data)
    assert c == oracle.compress(data)
    assert depress(snap, c) == data


@pytest.mark.parametrize("name", CORPUS)
def test_corpus_frame(snap, oracle, name):
    # roundtrip_frame + read_and_write_frame_encoder_match (test/tests.rs:75-88)
    data = corpus(name)
    w = snap.write.FrameEncoder(io.BytesIO())
    w.write_all(data)
    written = w.into_inner().getvalue()
    assert written == oracle.frame_encode(data)
    assert snap.read.FrameEncoder(io.BytesIO(data)).read_to_end() == written
    assert snap.frame.decode_all(written) == data
    if len(data) <= 200000:
        assert snap.read.FrameDecoder(io.BytesIO(written)).read_to_end() == data


def test_config1_html_single_block(snap, oracle):
    # BASELINE.json configs[0]: data/html, one 64KB block and the whole (2-block) file
    html = corpus("html")
    for d in (html[:65536], html):
        c = press(snap, d)
        assert c == oracle.compress(d)
        assert depress(snap, c) == d
    assert len(press(snap, html)) == 22843 and len(press(snap, html[:65536])) == 16533


@pytest.mark.parametrize("name,data,want,bad_header", DECODE_ERRORS, ids=[k[0] for k in DECODE_ERRORS])
def test_decode_error_kats(snap, name, data, want, bad_header):
    import gpu_helpers
    if bad_header:
        with pytest.raises(snap.Error) as ei:
            snap.raw.decompress_len(data)
        assert ei.value.as_tuple() == want
        cap = 1024
    else:
        cap = snap.raw.decompress_len(data)
    with pytest.raises(snap.Error) as ei:
        snap.raw.Decoder().decompress(data, bytearray(cap))
    assert ei.value.as_tuple() == want
    # the batched kernel path reports the same status
    if data:
        (st, _), = gpu_helpers.decompress_batch_host([data], [cap])
        assert st == want


@pytest.mark.parametrize("stream,want", COPY_CLOSE_TO_END)
def test_copy_close_to_end(snap, stream, want):
    assert depress(snap, stream) == want


def test_empty_and_tiny(snap, oracle):
    assert press(snap, b"") == b"\x00"
    assert depress(snap, b"\x00") == b""
    assert press(snap, b"\x00") == oracle.compress(b"\x00")
    w = snap.write.FrameEncoder(io.BytesIO())
    w.write_all(b"")
    assert w.into_inner().getvalue() == b""                      # src/write.rs:155-157
    assert snap.frame.decode_all(b"") == b""
    with pytest.raises(snap.Error) as ei:
        snap.raw.Encoder().compress(b"abc", bytearray(10))
    assert ei.value.as_tuple() == ("BufferTooSmall", 10, 35, 0)   # src/compress.rs:111-116


def test_small_sweeps_batched(snap, oracle):
    import gpu_helpers
    units = RANDOM + small_copy_inputs() + small_regular_inputs()
    got = gpu_helpers.compress_batch_host(units)
    for u, g in zip(units, got):
        assert g == oracle.compress(u)
    back = gpu_helpers.decompress_batch_host(got, [len(u) for u in units])
    for u, (st, b) in zip(units, back):
        assert st[0] == "Ok" and b == u


def test_property_roundtrip(snap, oracle):
    import gpu_helpers
    import pyarrow as pa
    rng = random.Random(99)
    units = []
    for _ in range(400):
        n = rng.randrange(0, 10000)
        alpha = rng.choice([2, 3, 16, 256])
        units.append(bytes(rng.randrange(alpha) for _ in range(n)))
    got = gpu_helpers.compress_batch_host(units)
    assert all(g == oracle.compress(u) for u, g in zip(units, got))
    back = gpu_helpers.decompress_batch_host(got, [len(u) for u in units])
    assert all(st[0] == "Ok" and b == u for u, (st, b) in zip(units, back))
    # streams from another encoder (Google C++ snappy via pyarrow) decode to the same bytes
    codec = pa.Codec("snappy")
    foreign = [codec.compress(u).to_pybytes() for u in units if u]
    back = gpu_helpers.decompress_batch_host(foreign, [len(u) for u in units if u])
    assert all(st[0] == "Ok" and b == u for u, (st, b) in zip([u for u in units if u], back))


def test_corrupt_streams_match_oracle(snap, oracle):
    """Bit-flipped / truncated streams: identical status (variant + payload) or identical output."""
    import gpu_helpers
    from oracle.oracle import OracleError
    rng = random.Random(5)
    base = oracle.compress(corpus("alice29.txt")[:20000])
    streams = []
    for _ in range(300):
        s = bytearray(base)
        for _ in range(rng.randrange(1, 4)):
            s[rng.randrange(len(s))] ^= 1 << rng.randrange(8)
        if rng.random() < 0.3:
            s = s[:rng.randrange(1, len(s))]
        streams.append(bytes(s))
    for i in (1, 2, 3):
        streams.append(corpus("baddata%d.snappy" % i))
    caps = []
    for s in streams:
        try:
            caps.append(min(oracle.decompress_len(s), 1 << 20))
        except OracleError:
            caps.append(1024)
    got = gpu_helpers.decompress_batch_host(streams, caps)
    for s, cap, (st, out) in zip(streams, caps, got):
        try:
            want = (("Ok", 0, 0, 0), oracle.decompress(s, cap=cap))
        except OracleError as e:
            want = (e.err, b"")
        assert (st, out) == want


def test_foreign_tag_forms(snap, oracle):
    """copy-4 tags and 3/4-byte literal lengths (never emitted by the encoder; build.rs:61-64)."""
    lit = bytes(range(256)) * 2
    streams = [
        bytes([0x80, 0x04]) + bytes([62 << 2, 0xFF, 0x01, 0x00]) + lit,                      # 3-byte literal length
        bytes([0x80, 0x04]) + bytes([63 << 2, 0xFF, 0x01, 0x00, 0x00]) + lit,                # 4-byte literal length
        bytes([0x88, 0x04]) + bytes([61 << 2, 0xFF, 0x01]) + lit + bytes([(7 << 2) | 3, 0x00, 0x02, 0x00, 0x00]),  # copy4
    ]
    for s in streams:
        assert depress(snap, s) == oracle.decompress(s)


def test_crc32c(snap, oracle):
    rng = random.Random(3)
    for n in [0, 1, 3, 4, 5, 63, 64, 65, 127, 1000, 4097, 65535, 65536, 100000]:
        d = bytes(rng.randrange(256) for _ in range(n))
        assert snap.raw.crc32c_masked(d) == oracle.crc32c_masked(d)


def test_frame_decoder_errors(snap, oracle):
    import gpu_helpers
    from oracle.oracle import OracleError
    ident = b"\xff\x06\x00\x00sNaPpY"
    good = oracle.frame_encode(b"hello world, hello world, hello world")
    bad = bytearray(good); bad[14] ^= 1
    pdf = oracle.frame_encode(corpus("paper-100k.pdf"))
    late = bytearray(pdf); late[-5] ^= 0x40
    streams = [
        b"123", b"\x00\x04\x00\x00abcd", ident + b"\x02\x00\x00\x00", b"\xff\x05\x00\x00sNaPp",
        b"\xff\x06\x00\x00sNaPpZ", ident + b"\x00\xff\xff\xff", ident + b"\x01\x03\x00\x00abc", bytes(bad),
        ident + b"\x80\x03\x00\x00xyz" + b"\xfe\x02\x00\x00\x00\x00" + ident + good[10:],
        good + b"\x00\x07", good[:-3], bytes(late), ident + b"\x00\x04\x00\x00\x00\x00\x00\x00",
        ident + b"\x00\x05\x00\x00\x00\x00\x00\x00\x80",
    ]
    for s in streams:
        try:
            want = ("Ok", oracle.frame_decode(s))
        except OracleError as e:
            want = (e.err, None)
        for impl in (snap.frame.decode_all, lambda x: snap.read.FrameDecoder(io.BytesIO(x)).read_to_end()):
            try:
                got = ("Ok", impl(s))
            except Exception as e:  # noqa: BLE001
                got = (gpu_helpers.err_tuple(e), None)
            assert got == want, (s[:24], got, want)


def test_write_frame_encoder_buffering(snap, oracle):
    """Chunk boundaries follow the reference's staging rules (src/write.rs:123-161)."""
    data = corpus("html_x_4")[:250000]
    for pieces in ([100000, 100000, 50000], [1, 65535, 70000, 114464], [65536, 65536, 65536, 53392], [30000] * 8 + [10000]):
        w = snap.write.FrameEncoder(io.BytesIO())
        at, src, model = 0, b"", [b"\xff\x06\x00\x00sNaPpY"]

        def inner(buf):
            for i in range(0, len(buf), 65536):
                model.append(oracle.compress_frame(buf[i:i + 65536]))
        for p in pieces:
            buf = data[at:at + p]; at += p
            w.write(buf)
            while True:                       # model of src/write.rs:123-152
                free = 65536 - len(src)
                if len(buf) <= free:
                    break
                if not src:
                    inner(buf); buf = b""
                else:
                    src += buf[:free]; inner(src); src = b""; buf = buf[free:]
            src += buf
        if src:
            inner(src)
        assert w.into_inner().getvalue() == b"".join(model)
        assert snap.frame.decode_all(b"".join(model)) == data[:at]


def test_read_frame_encoder_big_and_little_buffers(snap):
    # test/tests.rs:321-340
    data = corpus("html")
    big = snap.read.FrameEncoder(io.BytesIO(data)).read_to_end()
    r = snap.read.FrameEncoder(io.BytesIO(data))
    little = bytearray()
    while True:
        p = r.read(5)
        if not p:
            break
        little += p
    assert bytes(little) == big


def test_device_batch_api_full_size_blocks(snap, oracle):
    """Device-resident batch (the measured path): 64KB text blocks generated on device,
    compressed, compared with the oracle, decompressed and compared with the input."""
    import ctypes as C
    import torch
    import gpu_helpers
    L = gpu_helpers.lib()
    text = b"".join(corpus(n) for n in ("alice29.txt", "asyoulik.txt", "lcet10.txt", "plrabn12.txt"))
    count, blk, stride, mul = 3000, 65536, 76544, 65521
    dev = torch.device("cuda:0")
    t_text = torch.frombuffer(bytearray(text), dtype=torch.uint8).to(dev)
    t_in = torch.empty(count * blk, dtype=torch.uint8, device=dev)
    t_c = torch.empty(count * stride, dtype=torch.uint8, device=dev)
    t_out = torch.zeros(count * blk, dtype=torch.uint8, device=dev)
    t_clen = torch.zeros(count, dtype=torch.int32, device=dev)
    t_dlen = torch.zeros(count, dtype=torch.int32, device=dev)
    t_st = torch.zeros(count * 4, dtype=torch.int64, device=dev)
    e = snap._lib.SbError()
    st = torch.cuda.current_stream().cuda_stream
    assert L.sb_generate_blocks_device(t_text.data_ptr(), len(text), t_in.data_ptr(), blk, blk, 0, count, mul, st, C.byref(e)) == 0
    b = gpu_helpers.batch_from_tensors(t_in, blk, blk, t_c, stride, stride, t_clen, None, count)
    assert L.sb_compress_batch_device(C.byref(b), st, C.byref(e)) == 0
    b2 = gpu_helpers.batch_from_tensors(t_c, stride, 0, t_out, blk, blk, t_dlen, t_st, count, in_lens_t=t_clen)
    assert L.sb_decompress_batch_device(C.byref(b2), st, C.byref(e)) == 0
    torch.cuda.synchronize()
    assert torch.equal(t_in, t_out)
    assert int(t_st.view(count, 4)[:, 0].abs().sum()) == 0
    assert bool((t_dlen == blk).all())
    clen = t_clen.cpu().numpy()
    c_host = t_c.cpu().numpy()
    span = len(text) - blk
    for i in list(range(0, count, 97)) + [count - 1]:
        off = (i * mul) % span
        want = oracle.compress(text[off:off + blk])
        assert bytes(c_host[i * stride:i * stride + int(clen[i])]) == want


def test_gpu_sharded_frame_encode(snap, oracle):
    """Two chunk ranges encoded on the device (rank 0 carries the stream identifier) concatenate
    to the single-stream bytes; the frame decoder accepts the result."""
    import torch
    data = corpus("lcet10.txt")
    t = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    parts = []
    for rank in range(2):
        part, _, _ = snap.shard.frame_encode_sharded(t, rank, 2)
        parts.append(bytes(part.cpu().numpy()))
    torch.cuda.synchronize()
    assert b"".join(parts) == oracle.frame_encode(data)
    assert snap.frame.decode_all(b"".join(parts)) == data


def test_libsnappy_compatible_symbols(snap, oracle):
    """snappy_compress / snappy_uncompress / ... as bound by the reference's snappy-cpp crate
    (snappy-cpp/src/lib.rs:13-88): Rust decompresses "cpp", "cpp" decompresses Rust."""
    import ctypes as C
    L = snap._lib.lib()
    data = corpus("geo.protodata")
    cap = L.snappy_max_compressed_length(len(data))
    assert cap == snap.raw.max_compress_len(len(data))
    buf, n = C.create_string_buffer(cap), C.c_size_t(cap)
    assert L.snappy_compress(data, len(data), buf, C.byref(n)) == 0
    comp = buf.raw[:n.value]
    assert comp == oracle.compress(data)
    m = C.c_size_t(0)
    assert L.snappy_uncompressed_length(comp, len(comp), C.byref(m)) == 0 and m.value == len(data)
    out, k = C.create_string_buffer(len(data)), C.c_size_t(len(data))
    assert L.snappy_uncompress(comp, len(comp), out, C.byref(k)) == 0 and out.raw[:k.value] == data
    small = C.c_size_t(10)
    assert L.snappy_compress(data, len(data), buf, C.byref(small)) == 2          # SNAPPY_BUFFER_TOO_SMALL
    bad, k2 = b"\x05\x00a", C.c_size_t(16)
    assert L.snappy_uncompress(bad, 3, out, C.byref(k2)) == 1                      # SNAPPY_INVALID_INPUT


def test_config3_urls_tiled_decompress(snap, oracle):
    """BASELINE configs[2] shape at test scale: data/urls.10K cut into 11 blocks, each compressed
    independently (oracle), tiled round-robin into 22000 streams, decoded by the batched kernel."""
    import ctypes as C
    import numpy as np
    import torch
    import gpu_helpers
    L = gpu_helpers.lib()
    data = corpus("urls.10K")
    blocks = [data[i:i + 65536] for i in range(0, len(data), 65536)]
    comp = [oracle.compress(b) for b in blocks]
    assert [len(c) for c in comp] == [31817, 30911, 30063, 30746, 30054, 31451, 32143, 32131, 32204, 31097, 22905]  # SURVEY 8d
    reps = 2000
    n = len(blocks) * reps
    dev = torch.device("cuda:0")
    src = torch.frombuffer(bytearray(b"".join(comp)), dtype=torch.uint8).to(dev)
    coff = np.concatenate([[0], np.cumsum([len(c) for c in comp])[:-1]])
    in_ptrs = torch.tensor([src.data_ptr() + int(coff[i % 11]) for i in range(n)], dtype=torch.int64, device=dev)
    in_lens = torch.tensor([len(comp[i % 11]) for i in range(n)], dtype=torch.int32, device=dev)
    out = torch.zeros(n * 65536, dtype=torch.uint8, device=dev)
    dlen = torch.zeros(n, dtype=torch.int32, device=dev)
    st = torch.zeros(n * 4, dtype=torch.int64, device=dev)
    b = snap._lib.SbBatch()
    b.in_ptrs, b.in_lens = in_ptrs.data_ptr(), in_lens.data_ptr()
    b.out_base, b.out_stride, b.out_cap_uniform = out.data_ptr(), 65536, 65536
    b.out_lens, b.statuses, b.count = dlen.data_ptr(), st.data_ptr(), n
    e = snap._lib.SbError()
    assert L.sb_decompress_batch_device(C.byref(b), torch.cuda.current_stream().cuda_stream, C.byref(e)) == 0
    torch.cuda.synchronize()
    assert int(st.view(n, 4)[:, 0].abs().sum()) == 0
    view = out.view(reps, 11, 65536)
    for k, blk in enumerate(blocks):
        want = torch.frombuffer(bytearray(blk), dtype=torch.uint8).to(dev)
        assert bool((view[:, k, :len(blk)] == want).all())
        assert bool((dlen.view(reps, 11)[:, k] == len(blk)).all())


def test_unaligned_units_device_api(snap, oracle):
    """Unit pointers at odd byte offsets (pointer-array addressing): K1 reads the window in place
    from global memory with aligned word loads around an unaligned base; K2 likewise."""
    import ctypes as C
    import numpy as np
    import torch
    import gpu_helpers
    L = gpu_helpers.lib()
    dev = torch.device("cuda:0")
    data = corpus("alice29.txt") + corpus("geo.protodata")
    rng = random.Random(17)
    units, offs, at = [], [], 1
    for _ in range(96):
        n = rng.choice([1, 15, 16, 17, 31, 100, 4097, 20000, 65535, 65536])
        o = rng.randrange(0, len(data) - n)
        units.append(data[o:o + n]); offs.append(at); at += n + rng.choice([0, 1, 2, 3, 5])
    blob = bytearray(at + 64)
    for u, o in zip(units, offs):
        blob[o:o + len(u)] = u
    t_in = torch.frombuffer(blob, dtype=torch.uint8).to(dev)
    stride = 76544 + 3                                           # odd output stride: unaligned destinations too
    t_c = torch.zeros(len(units) * stride + 64, dtype=torch.uint8, device=dev)
    in_ptrs = torch.tensor([t_in.data_ptr() + o for o in offs], dtype=torch.int64, device=dev)
    in_lens = torch.tensor([len(u) for u in units], dtype=torch.int32, device=dev)
    c_lens = torch.zeros(len(units), dtype=torch.int32, device=dev)
    b = snap._lib.SbBatch()
    b.in_ptrs, b.in_lens = in_ptrs.data_ptr(), in_lens.data_ptr()
    b.out_base, b.out_stride, b.out_cap_uniform, b.out_lens, b.count = t_c.data_ptr() + 1, stride, stride, c_lens.data_ptr(), len(units)
    e = snap._lib.SbError()
    st = torch.cuda.current_stream().cuda_stream
    assert L.sb_compress_batch_device(C.byref(b), st, C.byref(e)) == 0
    torch.cuda.synchronize()
    host_c, cl = t_c.cpu().numpy(), c_lens.cpu().numpy()
    for i, u in enumerate(units):
        assert bytes(host_c[1 + i * stride:1 + i * stride + int(cl[i])]) == oracle.compress(u), i
    # decode from the unaligned compressed streams into unaligned outputs
    ostride = 65536 + 5
    t_o = torch.zeros(len(units) * ostride + 64, dtype=torch.uint8, device=dev)
    d_lens = torch.zeros(len(units), dtype=torch.int32, device=dev)
    stt = torch.zeros(len(units) * 4, dtype=torch.int64, device=dev)
    b2 = snap._lib.SbBatch()
    b2.in_base, b2.in_stride, b2.in_lens = t_c.data_ptr() + 1, stride, c_lens.data_ptr()
    b2.out_base, b2.out_stride, b2.out_cap_uniform = t_o.data_ptr() + 3, ostride, 65536
    b2.out_lens, b2.statuses, b2.count = d_lens.data_ptr(), stt.data_ptr(), len(units)
    assert L.sb_decompress_batch_device(C.byref(b2), st, C.byref(e)) == 0
    torch.cuda.synchronize()
    assert int(stt.view(len(units), 4)[:, 0].abs().sum()) == 0
    host_o = t_o.cpu().numpy()
    for i, u in enumerate(units):
        assert bytes(host_o[3 + i * ostride:3 + i * ostride + len(u)]) == u, i


def test_large_multiblock_raw_stream(snap, oracle):
    """One raw stream of 24 MB (367 blocks behind a single varint): blocks are compressed in parallel
    and gathered on the device; the raw decode of it is one serial chain (the format has no block markers)."""
    data = (corpus("lcet10.txt") + corpus("kppkn.gtb") + corpus("html_x_4")) * 24
    c = snap.raw.Encoder().compress_vec(data)
    assert c == oracle.compress(data)
    assert snap.raw.Decoder().decompress_vec(c) == data


def test_adversarial_blocks(snap, oracle):
    """Rare parser paths (zero runs, incompressible data, dense slot clashes, offset/length limits)."""
    import gpu_helpers
    units = adversarial_blocks()
    got = gpu_helpers.compress_batch_host(units)
    assert [i for i, (g, u) in enumerate(zip(got, units)) if g != oracle.compress(u)] == []
    back = gpu_helpers.decompress_batch_host(got, [len(u) for u in units])
    assert [i for i, (u, (st, b)) in enumerate(zip(units, back)) if st[0] != "Ok" or b != u] == []


_LAYOUT_CHILD = r"""
import hashlib, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
import torch
torch.cuda.set_device(0)
import gpu_helpers
from conftest import corpus
from kats import adversarial_blocks
units = adversarial_blocks()
for name in ("alice29.txt", "html", "urls.10K", "kppkn.gtb", "fireworks.jpeg", "geo.protodata"):
    d = corpus(name)
    units += [d[i:i + 65536] for i in range(0, len(d), 65536)]
units = units * 30                     # > 132 x 14 units so every chain of every SM takes one or more
got = gpu_helpers.compress_batch_host(units)
print("DIGEST", len(units), hashlib.sha256(b"".join(len(g).to_bytes(4, "little") + g for g in got)).hexdigest())
"""


@pytest.mark.parametrize("ng", [0, 2, 4, 7])
def test_k1_chain_layouts(snap, oracle, ng):
    """K1 with 7 shared-memory-table chains per SM plus `ng` chains whose table lives in L2
    (SNAPB200_K1_NG is read once per process, hence the child process): same bytes as the oracle."""
    import hashlib
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    units = adversarial_blocks()
    for name in ("alice29.txt", "html", "urls.10K", "kppkn.gtb", "fireworks.jpeg", "geo.protodata"):
        d = corpus(name)
        units += [d[i:i + 65536] for i in range(0, len(d), 65536)]
    want_one = [oracle.compress(u) for u in units]
    want = want_one * 30
    digest = hashlib.sha256(b"".join(len(g).to_bytes(4, "little") + g for g in want)).hexdigest()
    env = dict(os.environ, SNAPB200_K1_NG=str(ng))
    res = subprocess.run([sys.executable, "-c", _LAYOUT_CHILD, root], env=env, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0, res.stderr[-2000:]
    line = [l for l in res.stdout.splitlines() if l.startswith("DIGEST")][-1].split()
    assert (int(line[1]), line[2]) == (len(want), digest)


class _Dribble(io.RawIOBase):
    """A reader that returns at most k bytes per read() call (short reads are legal for io::Read)."""

    def __init__(self, data, k):
        self._d, self._at, self._k = data, 0, k

    def readable(self):
        return True

    def read(self, n=-1):
        n = self._k if n is None or n < 0 else min(n, self._k)
        out = self._d[self._at:self._at + n]
        self._at += len(out)
        return out


def test_property_frame_roundtrip_stream(snap, oracle):
    """qc_roundtrip_stream (test/tests.rs:522-534) plus random write sizes and short reads:
    write::FrameEncoder output is modelled chunk by chunk with the oracle, read::FrameDecoder
    gives the bytes back even from a reader that dribbles 1..7 bytes per call."""
    rng = random.Random(4242)
    for case in range(40):
        n = rng.randrange(1, 10000) if case % 4 else rng.randrange(60000, 200000)
        alpha = rng.choice([2, 7, 256])
        data = bytes(rng.randrange(alpha) for _ in range(n))
        w = snap.write.FrameEncoder(io.BytesIO())
        at = 0
        while at < n:
            k = rng.choice([1, 5, 100, 4096, 65535, 65536, 65537, 100000])
            w.write(data[at:at + k]); at += k
        framed = w.into_inner().getvalue()
        assert framed[:10] == b"\xff\x06\x00\x00sNaPpY"
        assert oracle.frame_decode(framed) == data                 # any legal chunking decodes with the oracle
        assert snap.frame.decode_all(framed) == data
        if n < 20000:
            assert snap.read.FrameDecoder(_Dribble(framed, rng.randrange(1, 8))).read_to_end() == data
        # single write_all == oracle's single-stream bytes
        w2 = snap.write.FrameEncoder(io.BytesIO()); w2.write_all(data)
        assert w2.into_inner().getvalue() == oracle.frame_encode(data)


def test_packed_host_batch(snap, oracle):
    """sb_compress_batch_host_packed: the library packs densely and reports offsets (no foreknowledge of sizes)."""
    import gpu_helpers
    units = adversarial_blocks()[:20] + [b"", b"x", corpus("alice29.txt")[:65536], corpus("html")[:50000]]
    for name in ("urls.10K", "kppkn.gtb"):
        d = corpus(name)
        units += [d[i:i + 65536] for i in range(0, len(d), 65536)]
    units = units * 40                      # several waves (64 MiB first wave)
    got, dense, total = gpu_helpers.compress_batch_host_packed(units)
    want = [oracle.compress(u) for u in units[:len(units) // 40]] * 40
    assert got == want and dense and total == sum(len(w) for w in want)


def test_device_frame_encode_decode_ws(snap, oracle):
    """Stream-ordered frame encode/decode with caller scratch: bytes == write::FrameEncoder, decode with the
    encoder's chunk index (parallel parse) and without it (serial walk) give the data back."""
    import gpu_helpers
    for name, cut in (("alice29.txt", None), ("fireworks.jpeg", None), ("html", 70000), ("paper-100k.pdf", 65536), ("geo.protodata", 1)):
        data = corpus(name)[:cut] if cut else corpus(name)
        stream, offs, res = gpu_helpers.frame_encode_device_ws(data)
        assert res.status.code == 0 and res.nchunks == (len(data) + 65535) // 65536
        assert stream == oracle.frame_encode(data)
        assert offs[0] == 10 and offs[-1] == len(stream)
        for kw in (dict(index=offs), dict(index=None), dict(index=offs, ws=True), dict(index=None, ws=True)):
            st, out = gpu_helpers.frame_decode_device(stream, len(data), **kw)
            assert st[0] == "Ok" and out == data, (name, kw)
    # a rank's fragment: no stream identifier
    data = corpus("lcet10.txt")[:200000]
    stream, offs, res = gpu_helpers.frame_encode_device_ws(data, ident=False)
    assert stream == oracle.frame_encode(data)[10:] and offs[0] == 0
    for kw in (dict(index=offs), dict(index=None)):
        st, out = gpu_helpers.frame_decode_device(stream, len(data), fragment=True, **kw)
        assert st[0] == "Ok" and out == data
    st, out = gpu_helpers.frame_decode_device(stream, len(data), index=None)      # without the flag: StreamHeader
    assert st[0] == "StreamHeader"


def test_device_frame_decode_errors(snap, oracle):
    """The device decoder reports the reference's first error in stream order and the bytes before it."""
    import gpu_helpers
    from oracle.oracle import OracleError
    ident = b"\xff\x06\x00\x00sNaPpY"
    data = corpus("alice29.txt")[:150000]
    good = oracle.frame_encode(data)
    flip = bytearray(good); flip[len(good) // 2] ^= 0x10         # payload damage in the middle chunk
    crc = bytearray(good); crc[14] ^= 1                           # checksum field of chunk 0
    streams = [bytes(flip), bytes(crc), good[:-7], good + b"\x00\x07", ident + b"\x02\x00\x00\x00",
               ident + b"\x80\x03\x00\x00xyz" + b"\xfe\x02\x00\x00\x00\x00" + ident + good[10:],
               ident + b"\x00\x05\x00\x00\x00\x00\x00\x00\x80", b"123", ident + b"\x01\x03\x00\x00abc"]
    for s in streams:
        try:
            want = (("Ok", 0, 0, 0), oracle.frame_decode(s))
        except OracleError as e:
            want = (e.err, None)
        st, out = gpu_helpers.frame_decode_device(s, 200000)
        assert st == want[0], (s[:20], st, want[0])
        if want[1] is not None:
            assert out == want[1]
        else:
            assert data.startswith(out)                           # everything before the failing chunk was produced
    # a wrong index falls back to the serial walk and still decodes
    idx = [10, 50, len(good)]
    st, out = gpu_helpers.frame_decode_device(good, len(data), index=idx)
    assert st[0] == "Ok" and out == data
    # output too small
    st, out = gpu_helpers.frame_decode_device(good, 1000)
    assert st[:3] == ("BufferTooSmall", 1000, len(data))


def test_device_batch_unit_limits(snap):
    """K1 skips a unit above 64KB or with a slot below max_compress_len and says why (ADVICE r1)."""
    import ctypes as C
    import torch
    import gpu_helpers
    L = gpu_helpers.lib()
    dev = torch.device("cuda:0")
    t_in = torch.zeros(3 * 80000, dtype=torch.uint8, device=dev)
    lens = torch.tensor([100, 70000, 65536], dtype=torch.int32, device=dev)
    t_out = torch.zeros(3 * 76544, dtype=torch.uint8, device=dev)
    out_lens = torch.full((3,), 7, dtype=torch.int32, device=dev)
    st = torch.zeros(3 * 32, dtype=torch.uint8, device=dev)
    b = gpu_helpers.batch_from_tensors(t_in, 80000, 0, t_out, 76544, 76544, out_lens, st, 3, in_lens_t=lens)
    e = snap._lib.SbError()
    assert L.sb_compress_batch_device(C.byref(b), torch.cuda.current_stream().cuda_stream, C.byref(e)) == 0
    torch.cuda.synchronize()
    codes = [int.from_bytes(bytes(st[32 * i:32 * i + 4].cpu().numpy()), "little") for i in range(3)]
    assert codes == [0, 1, 0] and int(out_lens[1]) == 0 and int(out_lens[0]) > 0 and int(out_lens[2]) > 0
    # uniform length above the block limit is refused on the host
    b2 = gpu_helpers.batch_from_tensors(t_in, 80000, 70000, t_out, 76544, 76544, out_lens, None, 3)
    assert L.sb_compress_batch_device(C.byref(b2), torch.cuda.current_stream().cuda_stream, C.byref(e)) == 1


def test_steady_state_allocates_nothing(snap, oracle):
    """After sb_reserve / a first call the host entry points perform no cudaMalloc, cudaHostAlloc or event creation."""
    import ctypes as C
    import gpu_helpers
    L = gpu_helpers.lib()
    units = [corpus("alice29.txt")[:65536]] * 300
    e = snap._lib.SbError()
    assert L.sb_reserve(4096, 64 << 20, 96 << 20, C.byref(e)) == 0
    gpu_helpers.compress_batch_host_packed(units)
    comp = [oracle.compress(units[0])] * 300
    gpu_helpers.decompress_batch_host(comp, [65536] * 300)
    before = L.sb_alloc_count()
    for _ in range(3):
        got, dense, _t = gpu_helpers.compress_batch_host_packed(units)
        assert got == comp
        res = gpu_helpers.decompress_batch_host(comp, [65536] * 300)
        assert all(r[0][0] == "Ok" for r in res)
    assert L.sb_alloc_count() == before


def test_first_use_from_many_threads(snap, oracle):
    """Concurrent first calls initialise the device context once (ADVICE r1: get_ctx was not thread safe).
    Runs in a child process so that the context is really uninitialised."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    child = r"""
import sys, threading
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
import torch; torch.cuda.set_device(0)
import gpu_helpers
from oracle import oracle
snap = gpu_helpers.snap()
data = [bytes([i]) * 3000 + b"tail %d" % i for i in range(8)]
out = [None] * 8
def work(i):
    torch.cuda.set_device(0)
    out[i] = snap.raw.Encoder().compress_vec(data[i])
ts = [threading.Thread(target=work, args=(i,)) for i in range(8)]
[t.start() for t in ts]; [t.join() for t in ts]
assert out == [oracle.compress(d) for d in data]
print("THREADS OK")
"""
    res = subprocess.run([sys.executable, "-c", child, root], capture_output=True, text=True, timeout=600)
    assert res.returncode == 0 and "THREADS OK" in res.stdout, res.stderr[-2000:]


def test_foreign_far_offsets(snap, oracle):
    """Decode-side completeness (SURVEY 8f3): copy-4 elements with offsets above 65535 inside a >64KB raw stream."""
    rng = random.Random(77)
    head = bytes(rng.randrange(256) for _ in range(70000))
    want = head + head[:40] + head[100:131] + head[65500:65560]
    def lit(b):
        out = b""
        for i in range(0, len(b), 60):
            c = b[i:i + 60]
            out += bytes([(len(c) - 1) << 2]) + c
        return out
    def copy4(length, off):
        return bytes([((length - 1) << 2) | 3]) + off.to_bytes(4, "little")
    def varint(v):
        out = b""
        while v >= 0x80:
            out += bytes([v & 0x7F | 0x80]); v >>= 7
        return out + bytes([v])
    stream = varint(len(want)) + lit(head) + copy4(40, 70000) + copy4(31, 70040 - 100) + copy4(60, 70071 - 65500)
    assert oracle.decompress(stream) == want
    assert depress(snap, stream) == want
    # an offset beyond everything written so far is the reference's Offset error, also for values >= 2^31
    for off in (70001, 0x80000000, 0xFFFFFFFF):
        bad = varint(len(head) + 40) + lit(head) + copy4(40, off)
        from oracle.oracle import OracleError
        try:
            oracle.decompress(bad); w = None
        except OracleError as e:
            w = e.err
        try:
            depress(snap, bad); g = None
        except Exception as e:  # noqa: BLE001
            import gpu_helpers
            g = gpu_helpers.err_tuple(e)
        assert g == w and w[0] == "Offset"


def test_foreign_100mb_multiblock_stream(snap):
    """A 100 MB raw stream from a foreign encoder (pyarrow's bundled Google snappy: one stream, many blocks)."""
    pa = pytest.importorskip("pyarrow")
    base = corpus("alice29.txt") + corpus("html") + corpus("kppkn.gtb") + corpus("urls.10K")
    data = (base * (100 * 1000 * 1000 // len(base) + 1))[:100 * 1000 * 1000]
    comp = pa.compress(data, codec="snappy", asbytes=True)
    assert depress(snap, comp) == data


def test_streaming_wrappers_batch_mode(snap, oracle):
    """write::FrameEncoder(batch_chunks=N) queues full chunks for one device call and writes the same bytes;
    read::FrameDecoder(batch_chunks=N) reads ahead N chunks per device call and yields the same bytes and errors."""
    import gpu_helpers
    from oracle.oracle import OracleError
    rng = random.Random(99)
    data = corpus("alice29.txt") + corpus("html") + corpus("fireworks.jpeg")[:70000]
    for pattern in ([65536] * 40, [1000, 65536, 5, 200000, 65536 * 3, 70000], [7] * 3000 + [65536 * 5 + 3]):
        ref_w, bat_w = snap.write.FrameEncoder(io.BytesIO()), snap.write.FrameEncoder(io.BytesIO(), batch_chunks=16)
        at = 0
        for k in pattern:
            piece = data[at % len(data):][:k]
            ref_w.write(piece); bat_w.write(piece); at += k
            if rng.random() < 0.1:
                ref_w.flush(); bat_w.flush()
        a, b = ref_w.into_inner().getvalue(), bat_w.into_inner().getvalue()
        assert a == b
    framed = oracle.frame_encode(data)
    for k in (1, 3, 64):
        assert snap.read.FrameDecoder(io.BytesIO(framed), batch_chunks=k).read_to_end() == data
        assert snap.read.FrameDecoder(_Dribble(framed, 5000), batch_chunks=k).read_to_end() == data
    bad = bytearray(framed); bad[len(framed) // 2] ^= 4
    for s_ in (bytes(bad), framed[:-9], framed + b"\x00\x07", framed[:10] + b"\x02\x00\x00\x00" + framed[10:]):
        try:
            want = (None, oracle.frame_decode(s_))
        except OracleError as e:
            want = (e.err, None)
        for k in (1, 4, 64):
            r = snap.read.FrameDecoder(io.BytesIO(s_), batch_chunks=k)
            got, parts = None, []
            try:
                while True:
                    p = r.read(100000)
                    if not p:
                        break
                    parts.append(p)
            except Exception as e:  # noqa: BLE001
                got = gpu_helpers.err_tuple(e)
            assert got == want[0], (k, got, want[0])
            if want[1] is not None:
                assert b"".join(parts) == want[1]
            else:
                assert data.startswith(b"".join(parts))


def test_k1_reads_stay_inside_the_input(snap, oracle):
    """Blocks whose final copy runs to the very end of the block, in a tensor that ends exactly there: K1 must not read
    past the caller's allocation (round 2: k1_extend's candidate side over-read up to 6 bytes, which faulted on rank 4
    of an 8-GPU run where the next page was unmapped). Bit-exactness here; tools/sanitize.sh runs this test under
    memcheck with the caching allocator off, so that the allocation really ends at the last byte."""
    import ctypes as C
    import torch
    import gpu_helpers
    L = gpu_helpers.lib()
    dev = torch.device("cuda:0")
    base = corpus("alice29.txt")
    blocks = []
    for k, tail in enumerate((17, 64, 200, 1000, 4, 5, 6, 7, 8, 9, 31, 33)):
        b = bytearray(base[k * 1000:k * 1000 + 65536])
        b[-tail:] = b[100:100 + tail]                       # the block ends inside a match against earlier text
        blocks.append(bytes(b))
    blocks.append(bytes(65536))                             # one long run to the end
    n = len(blocks)
    t_in = torch.frombuffer(bytearray(b"".join(blocks)), dtype=torch.uint8).to(dev)      # exactly n * 65536 bytes
    t_out = torch.zeros(n * 76544, dtype=torch.uint8, device=dev)
    lens = torch.zeros(n, dtype=torch.int32, device=dev)
    b = gpu_helpers.batch_from_tensors(t_in, 65536, 65536, t_out, 76544, 76544, lens, None, n)
    e = snap._lib.SbError()
    assert L.sb_compress_batch_device(C.byref(b), torch.cuda.current_stream().cuda_stream, C.byref(e)) == 0
    torch.cuda.synchronize()
    out = t_out.cpu().numpy()
    for i, blk in enumerate(blocks):
        assert bytes(out[i * 76544:i * 76544 + int(lens[i])]) == oracle.compress(blk), i
