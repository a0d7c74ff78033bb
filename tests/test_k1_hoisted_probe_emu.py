"""K1's parser issues the next window's probe (table read + candidate loads) as soon as all of a window's
table stores are done, before the window's event-ring stores. These tests run the
K1 body under the CPU warp emulator, compare its output with the oracle byte for byte, and use the
emulator's window counters to show that both the early ("hoisted") and the loop-top probe ran, and
that no table slot changed between a probe's read and its use."""
import ctypes as C
import random

import pytest

import emu_helpers as emu
from conftest import CORPUS, corpus

BLOCK = 65536
MUL = 65521                                   # bench.py's block generator: block i starts at (i * MUL) % span
TEXT_FILES = ("alice29.txt", "asyoulik.txt", "lcet10.txt", "plrabn12.txt")


def counters():
    return (C.c_ulonglong * 3).in_dll(emu.lib(), "sb_emu_k1_windows")


def run(units, **kw):
    """Compress under the emulator; returns (streams, window counts): fast-path windows whose probe was issued
    early by the previous window (hoisted) or at the loop top, probes whose table slot changed between read and
    use (stale)."""
    cnt = counters()
    for i in range(3):
        cnt[i] = 0
    got = emu.compress_units(units, **kw)
    return got, dict(hoisted=cnt[0], loop_top=cnt[1], stale=cnt[2])


def check(oracle, units, **kw):
    got, c = run(units, **kw)
    assert [i for i, (g, u) in enumerate(zip(got, units)) if g != oracle.compress(u)] == []
    assert c["stale"] == 0
    return c


def matches(stream):
    """(start, end) of every copy the encoder took, from its raw stream (split copies merged)."""
    i, v, sh = 0, 0, 0
    while True:                                   # varint length
        b = stream[i]; i += 1
        v |= (b & 0x7F) << sh; sh += 7
        if b < 0x80:
            break
    pos, out, prev = 0, [], None
    while i < len(stream):
        t = stream[i]; k = t & 3
        if k == 0:
            ln = t >> 2
            if ln >= 60:
                nb = ln - 59
                ln = int.from_bytes(stream[i + 1:i + 1 + nb], "little"); i += nb
            i += 1; ln += 1
            pos += ln; i += ln; prev = None
            continue
        if k == 1:
            ln = 4 + ((t >> 2) & 7); off = ((t >> 5) << 8) | stream[i + 1]; i += 2
        elif k == 2:
            ln = (t >> 2) + 1; off = int.from_bytes(stream[i + 1:i + 3], "little"); i += 3
        else:
            ln = (t >> 2) + 1; off = int.from_bytes(stream[i + 1:i + 5], "little"); i += 5
        if prev is not None and prev[2] == off and out[-1][1] == pos:
            out[-1] = (out[-1][0], pos + ln)
        else:
            out.append((pos, pos + ln))
        prev = (pos, pos + ln, off)
        pos += ln
    assert pos == v
    return out


def bench_blocks(count, first=0):
    text = b"".join(corpus(f) for f in TEXT_FILES)
    span = len(text) - BLOCK
    return [text[(u * MUL) % span:(u * MUL) % span + BLOCK] for u in range(first, first + count)]


def crafted(end_in_window, seed, length=None, echo=False):
    """Text with random segments repeated so that the encoder takes copies [B, B + L) with B = 32 k + 8 and
    B + L = (B & ~31) + end_in_window, i.e. copies that end `end_in_window` bytes after the start of the window
    they begin in. echo: the 4 bytes at the copy's last byte recur 5 bytes later, so a lane of the next window
    hashes to the slot of the copy-end insert."""
    rng = random.Random(seed)
    text = corpus("lcet10.txt")
    ln = length if length is not None else end_in_window - 8
    out = bytearray(text[:1500])
    want = []
    while len(out) < 60000:
        seg = bytes(rng.randrange(256) for _ in range(ln))
        out += seg + bytes([rng.randrange(256)])
        a = rng.randrange(0, len(text) - 400)
        out += text[a:a + 200 + rng.randrange(100)]
        out += bytes(rng.randrange(256) for _ in range((8 - len(out)) % 32))    # next byte sits at 32 k + 8
        want.append(len(out))
        tail = bytes(rng.randrange(256) for _ in range(3))
        out += seg + tail
        if echo:
            out += bytes([rng.randrange(256)]) + seg[-1:] + tail
        a = rng.randrange(0, len(text) - 400)
        out += text[a:a + 300 + rng.randrange(200)]
    return bytes(out[:BLOCK]), [(b, b + ln) for b in want if b + ln < BLOCK - 64]


def test_bench_text_blocks(oracle):
    c = check(oracle, bench_blocks(3) + bench_blocks(2, first=131072))
    assert c["hoisted"] > 0 and c["loop_top"] > 0


@pytest.mark.parametrize("name", CORPUS)
def test_corpus_files(oracle, name):
    data = corpus(name)
    units = [data[o:o + BLOCK] for o in range(0, min(len(data), 3 * BLOCK), BLOCK)]
    check(oracle, units)


@pytest.mark.parametrize("hybrid", [False, True])
def test_random_and_zero_blocks(oracle, hybrid):
    rng = random.Random(7)
    units = [bytes(rng.randrange(256) for _ in range(BLOCK)), bytes(BLOCK), bytes(20000),
             bytes(rng.randrange(4) for _ in range(30000)), bytes(rng.randrange(256) for _ in range(3000))]
    check(oracle, units, hybrid=hybrid)


@pytest.mark.parametrize("end_in_window,length", [(32, None), (33, None), (64, None), (8 + 200, 200)],
                         ids=["ends_w+32", "ends_w+33", "ends_w+64", "long_copy"])
@pytest.mark.parametrize("hybrid", [False, True])
def test_copy_ends_at_window_edges(oracle, end_in_window, length, hybrid):
    block, want = crafted(end_in_window, seed=end_in_window, length=length)
    got_copies = set(matches(oracle.compress(block)))
    taken = [m for m in want if m in got_copies]
    assert len(taken) >= len(want) // 2 > 0          # the block does hold the copies it was built for
    for lo, hi in taken:
        assert hi - (lo & ~31) == end_in_window
    c = check(oracle, [block], hybrid=hybrid)
    assert c["hoisted"] > 0 and c["loop_top"] > 0


@pytest.mark.parametrize("hybrid", [False, True])
def test_copy_end_insert_slot_read_by_next_window(oracle, hybrid):
    # copies ending 40 bytes into their window (the next window starts at lane 8) whose last 4 bytes recur at
    # lane 12: the next window's probe of lane 12 must see the copy-end insert of e-1
    block, want = crafted(40, seed=40, echo=True)
    got_copies = set(matches(oracle.compress(block)))
    assert len([m for m in want if m in got_copies]) >= len(want) // 2 > 0
    c = check(oracle, [block], hybrid=hybrid)
    assert c["hoisted"] > 0 and c["loop_top"] > 0


def test_victim_cut_after_hoisted_window(oracle):
    # windows where a 4-byte group recurs 10 bytes later inside the same window: the later lane's candidate is
    # the earlier lane of the same window, so the window is cut there; placed often enough that some of them
    # follow a window that issued their probe early
    rng = random.Random(3)
    text = corpus("alice29.txt")
    out = bytearray()
    while len(out) < BLOCK - 200:
        a = rng.randrange(0, len(text) - 300)
        out += text[a:a + 60 + rng.randrange(120)]
        g = bytes(rng.randrange(256) for _ in range(4))
        out += g + bytes(rng.randrange(256) for _ in range(6)) + g + bytes(rng.randrange(256) for _ in range(3))
    units = [bytes(out[:BLOCK])]
    for hybrid in (False, True):
        c = check(oracle, units, hybrid=hybrid)
        assert c["hoisted"] > 0 and c["loop_top"] > 0


def test_serial_fallback_and_block_tail(oracle):
    # a text block with a random run in the middle (scan stride grows: serial path), and short blocks whose
    # last 47 bytes and whole body sit near the end-of-block limits
    rng = random.Random(5)
    text = corpus("plrabn12.txt")
    block = text[:20000] + bytes(rng.randrange(256) for _ in range(3000)) + text[20000:40000]
    units = [block] + [text[:n] for n in (17, 47, 48, 63, 64, 95, 96, 100, 101, 131, 132, 133, 200, 1000)]
    units += [text[:n] for n in range(BLOCK - 47, BLOCK - 40)]
    c = check(oracle, units)
    assert c["hoisted"] > 0 and c["loop_top"] > 0
