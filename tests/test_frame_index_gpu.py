"""K7 chunk indexer on the GPU: sb_frame_index_device_ws against a walk of the stream, the decoder's index-first path
against the oracle, and which path (parallel parse or serial walk) the decoder took."""
import ctypes as C
import random
import re

import pytest

from conftest import corpus
from test_frame_index_emu import (IDENT, NOT_INDEXABLE, SEG_MIN, _boundary_stream, _hostile, oracle_decode, rechunk,
                                  walk)

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def snap():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA GPU")
    import gpu_helpers
    return gpu_helpers.snap()


def _index_tensors(t_in, n, fragment=False, max_chunks=None):
    import torch
    import gpu_helpers
    s, L = gpu_helpers.snap(), gpu_helpers.lib()
    maxc = max_chunks if max_chunks is not None else n // 8 + 16
    t_idx = torch.full((maxc + 1,), -1, dtype=torch.int64, device=t_in.device)
    t_cnt = torch.zeros(1, dtype=torch.int32, device=t_in.device)
    sb = L.sb_frame_index_scratch_bytes(n, maxc)
    t_scr = torch.empty(sb, dtype=torch.uint8, device=t_in.device)
    e = s._lib.SbError()
    rc = L.sb_frame_index_device_ws(t_in.data_ptr(), n, 1 if fragment else 0, t_idx.data_ptr(), maxc, t_cnt.data_ptr(),
                                    t_scr.data_ptr(), sb, torch.cuda.current_stream().cuda_stream, C.byref(e))
    if rc:
        raise s.error.from_c(e)
    return t_idx, int(t_cnt.item()) & 0xFFFFFFFF


def frame_index(stream, fragment=False, max_chunks=None):
    import torch
    t_in = torch.frombuffer(bytearray(stream) + bytearray(16), dtype=torch.uint8).to("cuda:0")
    t_idx, k = _index_tensors(t_in, len(stream), fragment, max_chunks)
    return k, (None if k == NOT_INDEXABLE else [int(x) for x in t_idx[:k + 1].cpu()])


def decode_path(capfd, monkeypatch, stream, cap, **kw):
    """Decode without an index through sb_frame_decode_device_ws with SNAPB200_DEBUG_FRAME=1: (status, bytes, need_serial)."""
    import gpu_helpers
    monkeypatch.setenv("SNAPB200_DEBUG_FRAME", "1")
    capfd.readouterr()
    st, out = gpu_helpers.frame_decode_device(stream, cap, ws=True, **kw)
    monkeypatch.delenv("SNAPB200_DEBUG_FRAME")
    m = re.findall(r"need_serial=(\d+)", capfd.readouterr().err)
    assert len(m) == 1
    return st, out, int(m[0])


def test_index_matches_walk(snap, oracle):
    rng = random.Random(5)
    text = corpus("lcet10.txt") + corpus("html")
    pieces, at = [], 0
    while at < 500000:
        ln = rng.choice([rng.randint(1, 300), rng.randint(1, 4096), rng.randint(1, 70000)])
        pieces.append(text[at:at + ln])
        at += ln
    streams = [oracle.frame_encode(corpus(n)) for n in ("alice29.txt", "fireworks.jpeg", "paper-100k.pdf", "kppkn.gtb")]
    streams += [rechunk(oracle, pieces), rechunk(oracle, [text[i:i + 1000] for i in range(0, 400000, 1000)])]
    streams += [oracle.frame_encode(bytes(rng.getrandbits(8) for _ in range(200000)))]          # uncompressed chunks
    streams += [_boundary_stream(seed, SEG_MIN, 12) for seed in (1, 2)]
    for s in streams:
        k, idx = frame_index(s)
        assert idx == walk(s) and k == len(idx) - 1
    frag = streams[0][10:]
    assert frame_index(frag, fragment=True)[1] == walk(frag, fragment=True)
    assert frame_index(frag)[0] == NOT_INDEXABLE
    assert frame_index(IDENT) == (0, [10])


@pytest.mark.parametrize("fake_len,body_len", [(12, 4096), (12, 4093), (60, 65536), (0, 30000), (4, 1000)])
def test_hostile_fake_headers(snap, oracle, fake_len, body_len):
    import gpu_helpers
    rng = random.Random(fake_len * 7 + body_len)
    s = _hostile(rng, max(3, 600000 // (body_len + 8)), fake_len, body_len, oracle)
    k, idx = frame_index(s)
    assert k == NOT_INDEXABLE or idx == walk(s)
    want_st, want = oracle_decode(oracle, s)
    assert gpu_helpers.frame_decode_device(s, len(want)) == (want_st, want)


def test_unclean_streams_declined_and_walked(snap, oracle, capfd, monkeypatch):
    data = corpus("alice29.txt")
    good = oracle.frame_encode(data)
    c0 = walk(good)[1]
    unclean = [IDENT + b"\xfe\x03\x00\x00abc" + good[10:], good[:c0] + b"\x80\x02\x00\x00zz" + good[c0:], good + good,
               good[:c0] + b"\x02" + good[c0 + 1:], good[:-100], good + b"\x00\x07", b"\xff\x06\x00\x00sNaPpZ" + good[10:]]
    for s in unclean:
        assert frame_index(s)[0] == NOT_INDEXABLE
        want_st, want = oracle_decode(oracle, s)
        st, out, ns = decode_path(capfd, monkeypatch, s, 400000)
        assert st == want_st and ns == 1
        assert out == want if want is not None else data.startswith(out)
    n = len(walk(good)) - 1
    assert frame_index(good, max_chunks=n - 1)[0] == NOT_INDEXABLE
    # a clean multi-chunk stream forced onto the walk by one padding chunk still decodes
    st, out, ns = decode_path(capfd, monkeypatch, unclean[0], len(data))
    assert st[0] == "Ok" and out == data and ns == 1 and n == 3


def test_clean_streams_take_the_parallel_parse(snap, oracle, capfd, monkeypatch):
    data = corpus("lcet10.txt")
    stream = oracle.frame_encode(data)
    st, out, ns = decode_path(capfd, monkeypatch, stream, len(data))
    assert st[0] == "Ok" and out == data and ns == 0
    st, out, ns = decode_path(capfd, monkeypatch, stream[10:], len(data), fragment=True)
    assert st[0] == "Ok" and out == data and ns == 0
    flip = bytearray(stream); flip[len(stream) // 2] ^= 0x10                  # payload damage: still indexed
    want_st, _ = oracle_decode(oracle, bytes(flip))
    st, out, ns = decode_path(capfd, monkeypatch, bytes(flip), len(data))
    assert st == want_st and ns == 0 and data.startswith(out)
    assert snap.frame.decode_all(stream) == data                                # host entry point


def test_host_decode_allocates_nothing_in_steady_state(snap, oracle):
    import gpu_helpers
    L = gpu_helpers.lib()
    data = corpus("alice29.txt")
    clean = oracle.frame_encode(data)
    padded = IDENT + b"\xfe\x03\x00\x00abc" + clean[10:]
    for s in (clean, padded):
        assert snap.frame.decode_all(s) == data
    before = L.sb_alloc_count()
    for _ in range(5):
        for s in (clean, padded):
            assert snap.frame.decode_all(s) == data
    assert L.sb_alloc_count() == before


def test_one_gib_device_stream_index_equals_encoder_index(snap, capfd, monkeypatch):
    """1 GiB of text encoded on the device: K7's index equals the encoder's d_chunk_offs (compared on the device), and the
    index-less decode gives the input back through the parallel parse."""
    import torch
    import gpu_helpers
    s, L = gpu_helpers.snap(), gpu_helpers.lib()
    dev = torch.device("cuda:0")
    st = torch.cuda.current_stream().cuda_stream
    e = s._lib.SbError()
    text = b"".join(corpus(n) for n in ("alice29.txt", "asyoulik.txt", "lcet10.txt", "plrabn12.txt"))
    blocks, blk = 16384, 65536
    n = blocks * blk
    t_text = torch.frombuffer(bytearray(text), dtype=torch.uint8).to(dev)
    t_in = torch.empty(n + 16, dtype=torch.uint8, device=dev)
    assert L.sb_generate_blocks_device(t_text.data_ptr(), len(text), t_in.data_ptr(), blk, blk, 0, blocks, 65521, st, C.byref(e)) == 0
    cap = L.sb_frame_max_len(n)
    t_out = torch.empty(cap + 16, dtype=torch.uint8, device=dev)
    t_offs = torch.zeros(blocks + 1, dtype=torch.int64, device=dev)
    t_res = torch.zeros(64, dtype=torch.uint8, device=dev)
    sb = L.sb_frame_encode_scratch_bytes(n)
    t_scr = torch.empty(sb, dtype=torch.uint8, device=dev)
    assert L.sb_frame_encode_device_ws(t_in.data_ptr(), n, t_out.data_ptr(), cap, 1, t_offs.data_ptr(), t_res.data_ptr(),
                                       t_scr.data_ptr(), sb, st, C.byref(e)) == 0
    del t_scr
    torch.cuda.synchronize()
    res = s._lib.SbFrameResult.from_buffer_copy(bytes(t_res.cpu().numpy()[:C.sizeof(s._lib.SbFrameResult)]))
    assert res.status.code == 0 and res.nchunks == blocks
    m = res.bytes
    t_idx, k = _index_tensors(t_out, m, max_chunks=blocks + 100)
    assert k == blocks and torch.equal(t_idx[:blocks + 1], t_offs)
    # index-less decode of the same stream: parallel parse, same bytes
    maxc = blocks + 100
    sbd = L.sb_frame_decode_scratch_bytes(maxc)
    t_dscr = torch.empty(sbd, dtype=torch.uint8, device=dev)
    t_dec = torch.empty(n + 16, dtype=torch.uint8, device=dev)
    monkeypatch.setenv("SNAPB200_DEBUG_FRAME", "1")
    capfd.readouterr()
    assert L.sb_frame_decode_device_ws(t_out.data_ptr(), m, t_dec.data_ptr(), n, None, 0, 0, t_res.data_ptr(), t_dscr.data_ptr(),
                                       sbd, maxc, st, C.byref(e)) == 0
    monkeypatch.delenv("SNAPB200_DEBUG_FRAME")
    assert "need_serial=0" in capfd.readouterr().err
    torch.cuda.synchronize()
    res = s._lib.SbFrameResult.from_buffer_copy(bytes(t_res.cpu().numpy()[:C.sizeof(s._lib.SbFrameResult)]))
    assert res.status.code == 0 and res.bytes == n and res.nchunks == blocks
    assert torch.equal(t_dec[:n], t_in[:n])
