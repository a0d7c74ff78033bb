"""Generator of raw and framed Snappy streams that use every legal element encoding (TEST TOOLING, pure Python).

Our encoder and pyarrow write one narrow grammar: the shortest literal header, copy-1 or copy-2 of at least 4 bytes, the
shortest varint. A decoder must accept every stream the reference accepts, so here each element of a plan is written in
any of its legal encodings:

* a literal of L bytes: the tag itself (L <= 60), tag 60 (L <= 256), tag 61 (L <= 65,536), tags 62 and 63 (any L);
* a copy (len 1..64, off): copy-1 (4 <= len <= 11, off < 2048), copy-2 (off < 65,536), copy-4 (always);
* the header varint: minimal, or padded with 0x80 continuation bytes up to 10 bytes.

Modes: "blocked" streams keep every element inside its 65,536-byte output block and every copy inside its block (the
streams a block-parallel decoder can split); "unblocked" streams let copies reach into earlier blocks and elements
straddle block boundaries. `model_decode` is a second reference beside the oracle, and `classify` replays the window
partition of K2 (rust-snappy_b200/csrc/k2_window.inc) to label every element by the kernel branch it takes; it measures
coverage only.
"""
from collections import Counter

BLOCK = 65536
MAX_INPUT = (1 << 32) - 1
IDENT = b"\xff\x06\x00\x00sNaPpY"
LIT_FORMS = ("lit1", "lit60", "lit61", "lit62", "lit63")
COPY_FORMS = ("copy1", "copy2", "copy4")


def varint(v, width=None):
    """v as a varint, minimal or padded with 0x80 continuation bytes to `width` bytes (at most 10)."""
    out = bytearray()
    while v >= 0x80:
        out.append(v & 0x7F | 0x80)
        v >>= 7
    out.append(v)
    if width is not None and width > len(out):
        assert width <= 10
        out[-1] |= 0x80
        out += b"\x80" * (width - len(out) - 1) + b"\x00"
    return bytes(out)


def lit_forms(n):
    return [f for f, ok in zip(LIT_FORMS, (n <= 60, n <= 256, n <= 65536, n <= 1 << 24, True)) if ok]


def literal_header(n, form):
    if form == "lit1":
        return bytes([(n - 1) << 2])
    nb = LIT_FORMS.index(form)
    return bytes([(59 + nb) << 2]) + (n - 1).to_bytes(nb, "little")


def copy_forms(length, off):
    return [f for f, ok in zip(COPY_FORMS, (4 <= length <= 11 and off < 2048, off < 65536, True)) if ok]


def copy_elem(length, off, form):
    if form == "copy1":
        return bytes([1 | (length - 4) << 2 | (off >> 8) << 5, off & 0xFF])
    if form == "copy2":
        return bytes([2 | (length - 1) << 2]) + off.to_bytes(2, "little")
    return bytes([3 | (length - 1) << 2]) + off.to_bytes(4, "little")


class Stream:
    """A generated raw stream: `stream` (header + body), its output `data`, header length `hl`, and per element
    (stream offset, header bytes, kind 0..3, output length, offset, form, output position)."""

    def __init__(self, stream, data, hl, elems, straddles=False):
        self.stream, self.data, self.hl, self.elems, self.straddles = stream, data, hl, elems, straddles


def _lit_len(rng, room):
    r = rng.random()
    n = rng.randint(1, 4) if r < 0.3 else rng.randint(5, 60) if r < 0.7 else \
        rng.randint(61, 300) if r < 0.9 else rng.randint(300, 5000)
    return max(1, min(n, room))


def _offset(rng, length, avail):
    cands = list(range(1, 9)) + [length - 1, length, length + 1, 31, 32, 33, 63, 64, 65, avail, avail - 1,
                                 rng.randint(1, avail)]
    if avail >= 65536:
        cands += [rng.randint(65536, avail)] * 3
    cands = [c for c in cands if 1 <= c <= avail]
    return rng.choice(cands)


def gen_stream(rng, size, mode="blocked", pad=None, copy_share=0.55, alphabet=4):
    """A stream of `size` output bytes. pad: header varint width (None = minimal). mode "blocked" or "unblocked"."""
    out = bytearray()
    body = bytearray()
    elems = []
    hdr = varint(size, pad)
    straddles = False
    while len(out) < size:
        d = len(out)
        room = size - d
        base = d - d % BLOCK if mode == "blocked" else 0
        if mode == "blocked":
            room = min(room, BLOCK - d % BLOCK)
        avail = d - base
        at = len(hdr) + len(body)
        if avail == 0 or rng.random() >= copy_share:
            n = _lit_len(rng, room)
            forms = lit_forms(n)
            if mode == "blocked" and (d + n) % BLOCK == 0 and d + n < size:
                # a block decoded alone applies the reference's checks at the block's end, where a long literal
                # header needs 4 bytes after its tag (test_block_ending_in_a_short_long_header_literal)
                forms = [f for f in forms if f == "lit1" or LIT_FORMS.index(f) + n >= 4]
            form = rng.choice(forms)
            payload = bytes(rng.randrange(alphabet) + 97 for _ in range(n)) if alphabet < 256 else rng.randbytes(n)
            h = literal_header(n, form)
            body += h + payload
            out += payload
            elems.append((at, len(h), 0, n, 0, form, d))
        else:
            length = rng.choice([rng.randint(1, 3), rng.randint(4, 11), rng.randint(1, 64), rng.randint(33, 64)])
            length = min(length, room)
            off = _offset(rng, length, avail)
            form = rng.choice(copy_forms(length, off))
            e = copy_elem(length, off, form)
            body += e
            for _ in range(length):
                out.append(out[-off])
            elems.append((at, len(e), COPY_FORMS.index(form) + 1, length, off, form, d))
            straddles = straddles or d - off < d - d % BLOCK
        straddles = straddles or (d // BLOCK != (len(out) - 1) // BLOCK)
    return Stream(hdr + bytes(body), bytes(out), len(hdr), elems, straddles)


def gen_single(rng, pad_share=0.25):
    """A single-block stream (at most 65,536 output bytes), mostly short."""
    r = rng.random()
    size = rng.randint(1, 64) if r < 0.25 else rng.randint(65, 1500) if r < 0.97 else rng.randint(1500, BLOCK)
    pad = rng.randint(len(varint(size)) + 1, 10) if rng.random() < pad_share else None
    return gen_stream(rng, size, "blocked", pad, copy_share=rng.choice([0.3, 0.55, 0.8]),
                      alphabet=rng.choice([2, 4, 256]))


def corrupt(rng, s):
    """Variants of a generated stream: a bit flip anywhere, and truncations at an element boundary, inside an element's
    trailer and inside a literal's payload."""
    b = bytearray(s.stream)
    b[rng.randrange(len(b))] ^= 1 << rng.randrange(8)
    out = [bytes(b)]
    e = rng.choice(s.elems)
    out.append(s.stream[:e[0]])
    if e[1] > 1:
        out.append(s.stream[:e[0] + rng.randint(1, e[1] - 1)])
    lits = [x for x in s.elems if x[2] == 0 and x[3] > 1]
    if lits:
        x = rng.choice(lits)
        out.append(s.stream[:x[0] + x[1] + rng.randint(1, x[3] - 1)])
    return out


def giant_literal(rng, n, form):
    """A literal of n bytes written with `form`, then copies that read across it: at its start, its middle, its end."""
    payload = rng.randbytes(n)
    body = literal_header(n, form) + payload
    copies = [(64, n), (33, n - 7), (4, 1), (64, n // 2), (17, 65536), (3, 70000), (64, 40)]
    out = bytearray(payload)
    for ln, off in copies:
        body += copy_elem(ln, off, "copy4" if off >= 65536 or ln < 4 else "copy2")
        for _ in range(ln):
            out.append(out[-off])
    return varint(len(out)) + body, bytes(out)


# ---------------------------------------------------------------------------------------------------------------
# model decoder: the reference's element loop and checks (src/decompress.rs), written plainly


def model_decode(s, cap):
    """(status tuple, bytes or None) for raw stream s decoded into a buffer of `cap` bytes."""
    n = len(s)
    if n == 0:
        return ("Empty", 0, 0, 0), None
    v, shift, hl = 0, 0, 0
    for i in range(n):
        if shift >= 64:
            break
        b = s[i]
        if b < 0x80:
            v |= b << shift
            hl = i + 1
            break
        v |= (b & 0x7F) << shift
        shift += 7
    if hl == 0:
        return ("Header", 0, 0, 0), None
    v &= (1 << 64) - 1
    if v > MAX_INPUT:
        return ("TooBig", v, MAX_INPUT, 0), None
    if v > cap:
        return ("BufferTooSmall", cap, v, 0), None
    src, dn = s[hl:], v
    sn = len(src)
    out = bytearray()
    sp = 0
    while sp < sn:
        tag = src[sp]
        sp += 1
        kind = tag & 3
        d = len(out)
        if kind == 0:
            L = tag >> 2
            if L >= 60:
                nb = L - 59
                if sp + 4 > sn:
                    return ("Literal", 4, sn - sp, dn - d), None
                ln = int.from_bytes(src[sp:sp + nb], "little") + 1
                sp += nb
            else:
                ln = L + 1
            if sn - sp < ln or dn - d < ln:
                return ("Literal", ln, sn - sp, dn - d), None
            out += src[sp:sp + ln]
            sp += ln
            continue
        nb = (1, 2, 4)[kind - 1]
        if sp + nb > sn:
            return ("CopyRead", nb, sn - sp, 0), None
        if kind == 1:
            ln, off = 4 + ((tag >> 2) & 7), (tag >> 5) << 8 | src[sp]
        else:
            ln, off = 1 + (tag >> 2), int.from_bytes(src[sp:sp + nb], "little")
        sp += nb
        if off == 0 or d < off:
            return ("Offset", off, d, 0), None
        if d + ln > dn:
            return ("CopyWrite", ln, dn - d, 0), None
        for _ in range(ln):
            out.append(out[-off])
    if len(out) != dn:
        return ("HeaderMismatch", dn, len(out), 0), None
    return ("Ok", 0, 0, 0), bytes(out)


# ---------------------------------------------------------------------------------------------------------------
# window classifier: which branch of K2 each element of a clean stream takes

WINDOW_CLASSES = ("lit_inside", "lit_spill", "hdr_crosses_end", "copy_flat", "replay_far", "replay_short_overlap",
                  "replay_long_overlap", "slow_window_mid")


def classify(s, counts=None, lane_forms=None):
    """Replay K2's window partition over the elements of clean Stream s. Adds to counts (Counter of WINDOW_CLASSES) and
    lane_forms (Counter of (form, lane) for long literal headers). A window starts at s0; an element at lane l ends its
    chain hop at l + hdr (+ len for a literal); a literal ending past lane 32 spills and closes the window; the next
    window starts where lane 0's chain leaves it."""
    counts = Counter() if counts is None else counts
    els = s.elems
    sn = len(s.stream) - s.hl
    dn = len(s.data)
    i, s0 = 0, 0
    while i < len(els) and s0 < sn:
        rem = sn - s0
        d0 = els[i][6]
        opos, chain = 0, []
        while i < len(els):
            at, hdr, kind, ln, off, form, _ = els[i]
            lane = at - s.hl - s0
            assert 0 <= lane < 32
            spill = kind == 0 and lane + hdr + ln > 32
            chain.append((lane, hdr, kind, ln, off, form, spill, opos))
            if lane_forms is not None and kind == 0 and form != "lit1":
                lane_forms[(form, lane)] += 1
            i += 1
            if spill:
                break
            opos += ln
            E = lane + hdr + (ln if kind == 0 else 0)
            if E >= 32:
                break
        win_out = sum(c[3] for c in chain if not c[6])
        spilled = chain[-1][6]
        sure = rem >= 40 and dn - d0 >= win_out and not spilled
        if not sure and rem >= 40:
            counts["slow_window_mid"] += 1
        for lane, hdr, kind, ln, off, form, spill, op in chain:
            if lane + hdr > 32:
                counts["hdr_crosses_end"] += 1
            if kind == 0:
                counts["lit_spill" if spill else "lit_inside"] += 1
            elif ln <= 32 and off >= op + ln:
                counts["copy_flat"] += 1
            elif off >= ln:
                counts["replay_far"] += 1
            elif ln <= 32:
                counts["replay_short_overlap"] += 1
            else:
                counts["replay_long_overlap"] += 1
        last = chain[-1]
        s0 = s0 + last[0] + last[1] + (last[3] if last[2] == 0 else 0)
    return counts


# ---------------------------------------------------------------------------------------------------------------
# frame streams


def chunk(ty, body, crc=None):
    head = bytes([ty]) + (len(body) + (4 if crc is not None else 0)).to_bytes(3, "little")
    return head + (crc.to_bytes(4, "little") if crc is not None else b"") + body


class Frame:
    """A generated frame stream, its decoded `data`, and the offset of every chunk header (then the length)."""

    def __init__(self, stream, data, offs):
        self.stream, self.data, self.offs = stream, data, offs


def gen_frame(rng, crc_masked, nchunks, kinds=("comp", "comp", "comp", "raw", "pad", "skip")):
    """Compressed chunks with generated bodies (some with padded varints), mixed with uncompressed, padding (0xFE) and
    skippable (0x80..0xFD) chunks, behind one stream identifier."""
    parts, data, offs, at = [IDENT], bytearray(), [], len(IDENT)
    for _ in range(nchunks):
        k = rng.choice(kinds)
        if k == "comp":
            s = gen_single(rng, pad_share=0.4)
            while model_decode(s.stream, len(s.data))[0][0] != "Ok":
                s = gen_single(rng, pad_share=0.4)
            c = chunk(0x00, s.stream, crc_masked(s.data))
            data += s.data
        elif k == "raw":
            raw = rng.randbytes(rng.randint(0, 3000))
            c = chunk(0x01, raw, crc_masked(raw))
            data += raw
        else:
            c = chunk(0xFE if k == "pad" else rng.randint(0x80, 0xFD), bytes(rng.randint(0, 40)))
        offs.append(at)
        parts.append(c)
        at += len(c)
    return Frame(b"".join(parts), bytes(data), offs + [at])
