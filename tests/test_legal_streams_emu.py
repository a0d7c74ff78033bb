"""Every raw decode path under the CPU warp emulator, on streams that use every legal Snappy element encoding
(tests/legal_streams.py): K2 one warp per stream, K8 split into 64 KB blocks, K8 over a batch, and K5 per frame chunk
with the caller's index, K7's index and the walk. Every result is compared with the oracle's exact status and bytes; the
generator's own model decoder must agree with the oracle on the whole population. Fixed seeds only."""
import random
from collections import Counter
from functools import lru_cache

import pytest

import emu_helpers as emu
import legal_streams as G
import test_frame_index_emu as k7
import test_raw_batch_split_emu as batch
import test_raw_split_emu as single

BLOCK = G.BLOCK
N_SINGLE = 5200


@lru_cache(maxsize=None)
def singles():
    """Single-block streams and their corrupted variants: ([Stream], [corrupt bytes])."""
    rng = random.Random(20261016)
    ss = [G.gen_single(rng) for _ in range(N_SINGLE)]
    bad = []
    for s in ss:
        bad += G.corrupt(rng, s)
    return ss, bad


@lru_cache(maxsize=None)
def multis():
    """Multi-block streams: blocked (some with a padded header), unblocked, and corrupted blocked ones."""
    rng = random.Random(7)
    blocked = [G.gen_stream(rng, rng.randint(2, 4) * BLOCK + rng.choice([1, rng.randint(2, BLOCK - 1), BLOCK]),
                            "blocked", pad=rng.choice([None, None, rng.randint(4, 10)]),
                            copy_share=rng.choice([0.3, 0.6]), alphabet=rng.choice([3, 256]))
               for _ in range(40)]
    unblocked = [G.gen_stream(rng, rng.randint(1, 3) * BLOCK + rng.randint(1, BLOCK), "unblocked",
                              pad=rng.choice([None, 10]), alphabet=rng.choice([3, 256])) for _ in range(16)]
    bad = []
    for s in blocked[:20]:
        bad += G.corrupt(rng, s)
    return blocked, unblocked, bad


def _header_cap(s, limit=70000):
    """The header's length when it is a sane one, else `limit`."""
    st, _ = G.model_decode(s, 0)
    if st[0] == "BufferTooSmall":
        return min(st[2], limit)
    return limit if st[0] in ("Empty", "Header", "TooBig") else 0


def _oracle(oracle, s, cap):
    return single.oracle_result(oracle, s, cap)


# ---------------------------------------------------------------------------------------------------------------
# the generator itself


def test_model_equals_oracle_on_the_whole_population(oracle):
    ss, bad = singles()
    blocked, unblocked, mbad = multis()
    nrej = 0
    for s in ss + blocked + unblocked:
        want = _oracle(oracle, s.stream, len(s.data))
        assert G.model_decode(s.stream, len(s.data)) == want
        if want[0][0] == "Ok":
            assert want[1] == s.data
        else:
            # a long literal header needs 4 stream bytes after its tag: such a stream is kept as an error case
            assert want[0][:2] == ("Literal", 4)
            nrej += 1
    assert nrej < len(ss) // 100
    for s in blocked:
        assert not s.straddles
    assert all(s.straddles for s in unblocked)
    for b in bad + mbad:
        cap = _header_cap(b)
        assert G.model_decode(b, cap) == _oracle(oracle, b, cap)


FORM_FLOOR = 1000         # elements of each encoding form
CLASS_FLOOR = 2000        # elements (or windows) of each K2 window class
LANE_FLOOR = 50           # short literals (L <= 60) with each long header form at each lane a header can start at


def test_every_encoding_form_and_window_class_is_reached(oracle):
    ss, _ = singles()
    blocked, unblocked, _ = multis()
    forms, classes, lanes = Counter(), Counter(), Counter()
    for s in ss + blocked + unblocked:
        if G.model_decode(s.stream, len(s.data))[0][0] != "Ok":
            continue
        G.classify(s, classes, lanes)
        if s.hl > len(G.varint(len(s.data))):
            forms["padded_header"] += 1
        for at, hdr, kind, ln, off, form, d in s.elems:
            forms[form] += 1
            if kind >= 2 and ln <= 3:
                forms[form + "_len1to3"] += 1
            if kind == 3 and off < 2048:
                forms["copy4_small_off"] += 1
            if kind >= 2 and off < ln:
                forms[form + "_overlap"] += 1
            if kind == 3 and off >= 65536:
                forms["copy4_far"] += 1
    for f in G.LIT_FORMS + G.COPY_FORMS + ("copy2_len1to3", "copy4_len1to3", "copy4_small_off", "copy2_overlap",
                                           "copy4_overlap", "padded_header"):
        assert forms[f] >= FORM_FLOOR, (f, forms[f])
    assert forms["copy4_far"] >= 500
    for c in G.WINDOW_CLASSES:
        assert classes[c] >= CLASS_FLOOR, (c, classes[c])
    # lane 1 never starts an element: every element occupies at least 2 bytes
    for f in G.LIT_FORMS[1:]:
        for lane in [0] + list(range(2, 32)):
            assert lanes[(f, lane)] >= LANE_FLOOR, (f, lane, lanes[(f, lane)])


# ---------------------------------------------------------------------------------------------------------------
# K2: one warp per stream


def _check_units(oracle, streams, caps, results):
    for s, cap, (st, out, guard) in zip(streams, caps, results):
        want_st, want = _oracle(oracle, s, cap)
        assert st == want_st, (s[:16].hex(), st, want_st)
        if want is not None:
            assert out == want
        assert guard == b"\xee" * 16


def test_k2_generated_streams(oracle):
    ss, _ = singles()
    streams = [s.stream for s in ss]
    caps = [len(s.data) for s in ss]
    _check_units(oracle, streams, caps, emu.decompress_units(streams, caps, grid=2, block=128))
    # one byte short of the header's length: BufferTooSmall before any element is read
    short = [s.stream for s in ss[:200] if len(s.data) > 1]
    caps = [len(s.data) - 1 for s in ss[:200] if len(s.data) > 1]
    _check_units(oracle, short, caps, emu.decompress_units(short, caps, grid=2, block=128))


def test_k2_corrupted_generated_streams(oracle):
    _, bad = singles()
    caps = [_header_cap(b) for b in bad]
    res = emu.decompress_units(bad, caps, grid=2, block=128)
    _check_units(oracle, bad, caps, res)
    assert sum(r[0][0] == "Ok" for r in res) < len(bad) // 2


def test_k2_literal_with_a_4_byte_length_of_2_to_the_24_plus_3_bytes(oracle):
    """Tag 63 with a length that needs all four bytes, followed by copies that read across the literal."""
    s, data = G.giant_literal(random.Random(16), (1 << 24) + 3, "lit63")
    assert oracle.decompress(s) == data
    _check_units(oracle, [s], [len(data)], emu.decompress_units([s], [len(data)]))


# ---------------------------------------------------------------------------------------------------------------
# K8: one stream split into its 64 KB blocks


def test_k8_splits_every_blocked_stream(oracle):
    blocked, _, _ = multis()
    for s in blocked:
        if _oracle(oracle, s.stream, len(s.data))[0][0] != "Ok":
            continue
        single.check_parallel(s.stream, s.data, None)


def test_k8_blocked_stream_over_several_long_segments(oracle):
    """A literal-heavy blocked stream of more than one segment at a segment length above the 128 KiB floor, split into
    the same blocks as at the floor."""
    rng = random.Random(11)
    s = G.gen_stream(rng, 9 * BLOCK + 5, "blocked", pad=7, copy_share=0.15, alphabet=256)
    seg = 3 * single.SEG_MIN + 32
    assert len(s.stream) > seg + single.SEG_MIN
    assert single.check_parallel(s.stream, s.data, None, seg=seg) == single.check_parallel(s.stream, s.data, None)


@pytest.mark.parametrize("form", ["lit60", "lit61"])
def test_block_ending_in_a_short_long_header_literal(oracle, form):
    """A 1-byte literal with a 1- or 2-byte length as the last element of a block that is not the stream's last: the stream
    is legal (the next block supplies the bytes after the tag that the reference asks for), but the block decoded
    alone does not have them. The split's block decode then fails and the stream is decoded by one warp: the result
    must still be the oracle's, through K8 and K8 over a batch."""
    rng = random.Random(13)
    blk = rng.randbytes(BLOCK)
    body = G.literal_header(BLOCK - 1, "lit61") + blk[:-1] + G.literal_header(1, form) + blk[-1:]
    tail = G.gen_stream(rng, BLOCK + 7, "blocked")
    stream = G.varint(2 * BLOCK + BLOCK + 7) + body + body + tail.stream[tail.hl:]
    data = blk + blk + tail.data
    assert oracle.decompress(stream) == data == G.model_decode(stream, len(data))[1]
    st, out, _, _, _ = single.raw_decode(stream, len(data))
    assert st == ("Ok", 0, 0, 0) and out == data
    res, _, _ = batch.run_batch([stream, tail.stream], [len(data), len(tail.data)])
    assert res == [(("Ok", 0, 0, 0), data), (("Ok", 0, 0, 0), tail.data)]


def test_k8_unblocked_and_corrupted_streams(oracle):
    _, unblocked, bad = multis()
    for s in unblocked:
        want_st, want = _oracle(oracle, s.stream, len(s.data))
        st, out, nchunks, _, _ = single.raw_decode(s.stream, len(s.data))
        assert st == want_st and nchunks == 0          # an element across a block end, or a copy into an earlier block
        if want is not None:
            assert out == want
    for b in bad:
        cap = _header_cap(b, 5 * BLOCK)
        want_st, want = _oracle(oracle, b, cap)
        st, out, nchunks, _, _ = single.raw_decode(b, cap)
        assert st == want_st, (st, want_st)
        if want is not None:
            assert out == want


# ---------------------------------------------------------------------------------------------------------------
# K8 over a batch


def test_k8b_mixed_batches(oracle):
    ss, sbad = singles()
    blocked, unblocked, bad = multis()
    rng = random.Random(5)
    units = [(s.stream, len(s.data), "split") for s in blocked[:24]]
    units += [(s.stream, len(s.data), "warp") for s in unblocked[:8]]
    units += [(b, _header_cap(b, 5 * BLOCK), "either") for b in bad[:24]]
    units += [(s.stream, len(s.data), "warp") for s in ss[:60]] + [(b, _header_cap(b), "warp") for b in sbad[:60]]
    rng.shuffle(units)
    streams, caps, kinds = [u[0] for u in units], [u[1] for u in units], [u[2] for u in units]
    res, blocks, _ = batch.run_batch(streams, caps, "ptrs")
    for i, (s, cap, kind) in enumerate(units):
        want_st, want = _oracle(oracle, s, cap)
        assert res[i][0] == want_st, (i, res[i][0], want_st)
        if want is not None:
            assert res[i][1] == want, i
        if kind == "split" and want is not None:
            assert blocks[i] == (len(want) + BLOCK - 1) // BLOCK, (i, blocks[i])
        elif kind == "either" and want is not None:
            assert blocks[i] in (0, (len(want) + BLOCK - 1) // BLOCK), (i, blocks[i])
        else:
            assert blocks[i] == 0, (i, kind, blocks[i])
    perm = list(range(len(units)))
    rng.shuffle(perm)
    res2, blocks2, _ = batch.run_batch([streams[i] for i in perm], [caps[i] for i in perm], "base")
    for k, i in enumerate(perm):
        assert res2[k] == res[i] and blocks2[k] == blocks[i], (k, i)


# ---------------------------------------------------------------------------------------------------------------
# K5: frame chunks, with the caller's index, with K7's index and through the walk


def _frame_expect(oracle, s, offs):
    """(status, bytes) of the oracle: on an error, the bytes of the chunks before the first failing one."""
    st, out = k7.oracle_decode(oracle, s)
    if out is not None:
        return st, out
    good = b""
    for b in offs:
        if b > len(s):
            break
        pst, pout = k7.oracle_decode(oracle, s[:b])
        if pout is None:
            break
        good = pout
    return st, good


def _check_frame(oracle, f_stream, offs, cap):
    want_st, want = _frame_expect(oracle, f_stream, offs)
    paths = {"index": emu.frame_decode(f_stream, cap, index=offs if offs[-1] == len(f_stream) else None)[:2],
             "walk": emu.frame_decode(f_stream, cap)[:2],
             "k7": k7.frame_decode_indexed(f_stream, cap)[:2]}
    for name, (st, out) in paths.items():
        assert st == want_st, (name, st, want_st)
        assert out == want, name
    return want_st


@lru_cache(maxsize=None)
def frames():
    from oracle import oracle as o
    rng = random.Random(3)
    clean = [G.gen_frame(rng, o.crc32c_masked, rng.randint(1, 12)) for _ in range(60)]
    clean += [G.gen_frame(rng, o.crc32c_masked, rng.randint(1, 12), kinds=("comp", "comp", "raw")) for _ in range(30)]
    return clean


def test_k5_generated_frames(oracle):
    statuses = Counter()
    for f in frames():
        assert _check_frame(oracle, f.stream, f.offs, len(f.data) + 16) == ("Ok", 0, 0, 0)
        assert oracle.frame_decode(f.stream) == f.data
    rng = random.Random(4)
    for f in frames():
        cap = BLOCK * (len(f.offs) + 1)
        bodies = [(a + 4, b) for a, b in zip(f.offs, f.offs[1:]) if f.stream[a] in (0, 1) and b > a + 4]
        if bodies:
            a, b = rng.choice(bodies)
            flip = bytearray(f.stream)
            flip[rng.randrange(a, b)] ^= 1 << rng.randrange(8)
            statuses[_check_frame(oracle, bytes(flip), f.offs, cap)[0]] += 1
        cut = rng.randrange(11, len(f.stream)) if len(f.stream) > 11 else 10
        statuses[_check_frame(oracle, f.stream[:cut], f.offs, cap)[0]] += 1
    assert statuses["Checksum"] >= 5 and statuses["UnexpectedEof"] >= 5


# ---------------------------------------------------------------------------------------------------------------
# padded header varints on all four paths


def test_padded_varints_on_every_path(oracle):
    rng = random.Random(12)
    small = [G.gen_stream(rng, n, "blocked", pad=w) for n in (0, 1, 5, 127, 128, 300, 16383, 16384, BLOCK)
             for w in range(len(G.varint(n)) + 1, 11)]
    small = [s for s in small if G.model_decode(s.stream, len(s.data))[0][0] == "Ok"]
    assert len(small) >= 60
    # 11 bytes is one too many: Header
    over = [b"\x80" * 10 + b"\x00", G.varint(5, 10)[:-1] + b"\x80\x00" + b"\x10abcde"]
    streams = [s.stream for s in small] + over
    caps = [len(s.data) for s in small] + [16, 16]
    _check_units(oracle, streams, caps, emu.decompress_units(streams, caps, grid=2, block=128))
    big = [G.gen_stream(rng, 2 * BLOCK + 3, "blocked", pad=w) for w in (4, 5, 9, 10)]
    for s in big:
        single.check_parallel(s.stream, s.data, None)
    units = [s.stream for s in big + small[:20]]
    caps = [len(s.data) for s in big + small[:20]]
    batch.check_batch(oracle, units, caps, set(range(len(big))))
    # frame chunks whose bodies carry padded varints, each decoded by all three frame paths
    parts, data, offs = [G.IDENT], b"", [10]
    for s in small[:40]:
        parts.append(G.chunk(0x00, s.stream, oracle.crc32c_masked(s.data)))
        data += s.data
        offs.append(offs[-1] + len(parts[-1]))
    stream = b"".join(parts)
    assert _check_frame(oracle, stream, offs, len(data)) == ("Ok", 0, 0, 0)


@pytest.mark.parametrize("body", [b"\x80", b"\x80\x80", b"\xff\xff\xff", b"\x80" * 5, b"\xff" * 4 + b"\x0f",
                                  b"\x80" * 9 + b"\x10", b"\xff" * 9 + b"\x01", b"\x80" * 10 + b"\x00"])
@pytest.mark.parametrize("before", ["padding", "compressed"])
def test_frame_chunk_varint_longer_than_its_body(oracle, body, before):
    """A compressed chunk whose (padded) varint runs past its body: the reader reads the length from its persistent
    buffer, whose bytes past the body are the chunk header's and the previous chunk's. The walk must give the oracle's
    exact error (or result), and so must the indexed paths, which hand such a chunk to the walk."""
    if before == "padding":
        prev = G.chunk(0xFE, bytes([0x11, 0x22, 0x33, 0x44, 0x55, 0x80, 0x80, 0x81, 0x01, 0x00, 0x00]))
    else:
        s = G.gen_stream(random.Random(1), 300, "blocked", pad=10)
        prev = G.chunk(0x00, s.stream, oracle.crc32c_masked(s.data))
    bad = G.chunk(0x00, body, oracle.crc32c_masked(b""))
    stream = G.IDENT + prev + bad
    offs = [10, 10 + len(prev), len(stream)]
    st = _check_frame(oracle, stream, offs, 1 << 17)
    assert (st[0] == "Ok") == (body == b"\x80" * 9 + b"\x10")
