"""K2's window step at the edges of its flattened copies and of its input words, under the CPU warp emulator.

K2 (rust-snappy_b200/csrc/k2_decompress.cuh) moves the bytes of the copies whose source lies before the window's output
in one compact index, 32 or 64 at a time, and replays the other copies one by one afterwards. It keeps 128 aligned input
bytes per warp (one word per lane) across windows and loads the next span when a window no longer fits in it. The
streams here are built so that these edges are reached at each of the four input alignments: a replayed copy beside
flattened ones, flattened copies of more than 32 and more than 64 bytes in one window, the last window served from a
span (s - span start = 92) and the first that loads a new one (93), streams shorter than 128 bytes, spans that reach
past the stream's end, spills right after a new span, and corrupted variants of all of them. `window_edges` replays the
window partition to show that they are reached; every decode must be the oracle's, status, payload and bytes.
Fixed seeds only."""
import random
from collections import Counter
from functools import lru_cache

import emu_helpers as emu
import legal_streams as G
import test_legal_streams_emu as pop

SPAN, SERVE = 128, 92          # input bytes per warp; a window at most this far past the span start is served from it
# valid empty streams of 1 to 4 bytes: put in front of a batch, they shift every later unit's address by that much
SHIFTS = [b"\x00", b"\x80\x00", b"\x80\x80\x00", b"\x80\x80\x80\x00"]


def _element(rng, out, shape):
    """(encoded element, bytes it appends) for an element of the given stream shape."""
    r = rng.random()
    if not out or r < shape["lit"]:
        t = rng.random()
        n = rng.randint(1, 6) if t < 0.6 else rng.randint(20, 70) if t < 0.9 else rng.randint(100, 300)
        data = rng.randbytes(n) if shape["alphabet"] == 256 else bytes(rng.choice(b"ab ") for _ in range(n))
        return G.literal_header(n, rng.choice(G.lit_forms(n))) + data, data
    length = rng.randint(1, 32) if rng.random() < shape["short_copy"] else rng.randint(33, 64)
    if rng.random() < shape["near"]:
        off = rng.randint(1, min(len(out), 12))              # a source inside the window's output: replayed
    else:
        off = rng.randint(min(len(out), 40), len(out))
    res = bytearray(out[-off:][:length])
    while len(res) < length:
        res.append(res[len(res) - off])
    return G.copy_elem(length, off, rng.choice(G.copy_forms(length, off))), bytes(res)


def gen(rng, size, shape):
    """A legal single-block stream of about `size` output bytes, header padded at random."""
    out, body, elems = bytearray(), bytearray(), []
    while len(out) < size:
        enc, data = _element(rng, out, shape)
        kind = enc[0] & 3
        hdr = len(enc) - (len(data) if kind == 0 else 0)
        off = 0 if kind == 0 else int.from_bytes(enc[1:hdr], "little") | ((enc[0] >> 5) << 8 if kind == 1 else 0)
        elems.append([len(body), hdr, kind, len(data), off, "", len(out)])
        body += enc
        out += data
    width = rng.choice([None, None, len(G.varint(len(out))) + rng.randint(1, 3)])
    head = G.varint(len(out), width)
    for e in elems:
        e[0] += len(head)
    return G.Stream(head + bytes(body), bytes(out), len(head), [tuple(e) for e in elems])


def window_edges(s, align, seen):
    """Replay K2's window partition and its input-word refills over legal stream `s` whose body starts at an address
    that is `align` mod 4, counting the edges it reaches in `seen`."""
    sn = len(s.stream) - s.hl
    by_pos = {e[0] - s.hl: e for e in s.elems}
    if len(s.stream) < SPAN:
        seen["short_stream"] += 1
    st, wb, after_spill = 0, None, False
    while st < sn:
        refill = wb is None or st - wb > SERVE
        if refill:
            if wb is not None and st - wb == SERVE + 1:
                seen["refill_at_93"] += 1
            if after_spill:
                seen["refill_after_spill"] += 1
            wb = st - ((align + st) & 3)
            if wb + SPAN > sn and sn > SPAN:
                seen["span_past_end"] += 1
        elif st - wb == SERVE:
            seen["served_at_92"] += 1
        p, opos, ctot, flat, holes, spill = st, 0, 0, 0, 0, False     # holes: copies replayed one by one
        while p - st < 32 and p < sn:
            _, hdr, kind, ln, off, _, _ = by_pos[p]
            if kind == 0:
                if p - st + hdr + ln > 32:
                    spill = True
                    p += hdr + ln
                    break
                opos += ln
                p += hdr + ln
                continue
            if ln <= 32 and off >= opos + ln:
                ctot += ln
                flat += 1
            else:
                holes += 1
            opos += ln
            p += hdr
        if flat and holes:
            seen["replay_beside_flattened"] += 1
        if ctot > 32:
            seen["flattened_over_32"] += 1
        if ctot > 64:
            seen["flattened_over_64"] += 1
        if spill and refill:
            seen["spill_after_refill"] += 1
        after_spill = spill
        st = p


SHAPES = [
    dict(lit=0.35, short_copy=0.9, near=0.15, alphabet=4),      # text-like
    dict(lit=0.15, short_copy=1.0, near=0.05, alphabet=256),    # many short far copies: over 64 flattened bytes
    dict(lit=0.5, short_copy=0.7, near=0.4, alphabet=256),      # replays and spills
]


@lru_cache(maxsize=None)
def population():
    """Legal streams (short and long) and the corrupted variants of some of them. A stream whose long literal header
    has fewer than 4 stream bytes after its tag is an error for the reference; such streams are left out."""
    rng = random.Random(20261018)
    ss = []
    for i in range(900):
        shape = SHAPES[i % len(SHAPES)]
        size = rng.randint(1, 90) if i % 4 == 0 else rng.randint(91, 2500)
        s = gen(rng, size, shape)
        if G.model_decode(s.stream, len(s.data))[0][0] == "Ok":
            ss.append(s)
    bad = []
    for s in ss[:300]:
        bad += G.corrupt(rng, s)
    return ss, bad


EDGES = ("short_stream", "refill_at_93", "served_at_92", "refill_after_spill", "span_past_end", "replay_beside_flattened",
         "flattened_over_32", "flattened_over_64", "spill_after_refill")


def test_the_population_reaches_every_edge_at_every_alignment(oracle):
    ss, _ = population()
    for align in range(4):
        seen = Counter()
        for s in ss:
            assert oracle.decompress(s.stream) == s.data
            window_edges(s, align, seen)
        for e in EDGES:
            assert seen[e] >= 10, (align, e, seen[e])


def _check(oracle, streams, caps, results):
    for s, cap, (st, out, guard) in zip(streams, caps, results):
        want_st, want = pop._oracle(oracle, s, cap)
        assert st == want_st, (s[:16].hex(), st, want_st)
        if want is not None:
            assert out == want
        assert guard == b"\xee" * 16


def test_k2_window_edges_at_every_alignment(oracle):
    ss, _ = population()
    streams, caps = [s.stream for s in ss], [len(s.data) for s in ss]
    for pad in SHIFTS:
        res = emu.decompress_units([pad] + streams, [0] + caps, grid=2, block=128)
        assert res[0][0] == ("Ok", 0, 0, 0)
        _check(oracle, streams, caps, res[1:])


def test_k2_corrupted_window_edges(oracle):
    _, bad = population()
    caps = [pop._header_cap(b) for b in bad]
    for pad in SHIFTS[:2]:
        res = emu.decompress_units([pad] + bad, [0] + caps, grid=2, block=128)
        _check(oracle, bad, caps, res[1:])
    assert sum(r[0][0] == "Ok" for r in res[1:]) < len(bad) // 2
