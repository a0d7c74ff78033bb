"""K1's parser resolves 64 positions per step: lane l probes w + l and w + 32 + l, taken copies come from pointer
doubling over both halves, and the inserts of the two halves are committed in position order. These tests run the K1
body under the CPU warp emulator on blocks crafted to reach the edges of such a step, compare every output with the
oracle byte for byte, and check the emulator's step counters (no stale table slot, no fetch past the block).

A step starts at w = s & ~31, so a copy that ends at a 32-aligned position P past the end of its own step makes the
next step start exactly at P. Every crafted pattern below therefore follows an "anchor": a 200-byte segment seen
earlier in the block whose copy ends at P. The oracle's parse of the block shows that the copies the pattern was
built for are there, at the intended offsets from P."""
import ctypes as C
import random

import pytest

import emu_helpers as emu
from conftest import corpus
from test_k1_hoisted_probe_emu import bench_blocks, matches

BLOCK = 65536


def counters():
    return (C.c_ulonglong * 4).in_dll(emu.lib(), "sb_emu_k1_windows")


def check(oracle, units, hybrid=False):
    """Compress under the emulator, compare with the oracle; returns (hoisted, loop-top) fast-path step counts."""
    cnt = counters()
    for i in range(4):
        cnt[i] = 0
    got = emu.compress_units(units, hybrid=hybrid)
    assert [i for i, (g, u) in enumerate(zip(got, units)) if g != oracle.compress(u)] == []
    assert cnt[2] == 0, "a probe read a table slot that changed before its use"
    assert cnt[3] == 0, "a sequential-word fetch reached the end of its block"
    return cnt[0], cnt[1]


class Crafter:
    """Builds a block out of text filler, first occurrences of random segments and patterns placed at 32-aligned
    anchor ends P. A pattern is a list of pieces: ("rand", k) random bytes, ("copy", k) a k-byte random segment
    whose first occurrence is placed before the anchor, or ("again", name, k) the first k bytes of a segment placed
    earlier in the same pattern under `name`. It returns the copies expected at offsets from P."""

    def __init__(self, seed):
        self.rng = random.Random(seed)
        self.text = corpus("lcet10.txt")
        self.out = bytearray()
        self.anchors = []

    def rand(self, k):
        return bytes(self.rng.randrange(256) for _ in range(k))

    def filler(self, lo, hi):
        a = self.rng.randrange(0, len(self.text) - hi)
        self.out += self.text[a:a + self.rng.randrange(lo, hi)]

    def place(self, pattern):
        """Append one anchor and pattern; returns P."""
        body, seen, named = bytearray(), [], {}
        for piece in pattern:
            if piece[0] == "rand":
                body += self.rand(piece[1])
            elif piece[0] == "copy":
                seg = self.rand(piece[1])
                seen.append((seg, len(body)))
                body += seg
            else:
                _, name, k = piece
                if name in named:
                    body += named[name][:k]
                else:
                    named[name] = self.rand(k)
                    body += named[name]
        body += self.rand(8)
        anchor = self.rand(200)
        self.filler(200, 300)
        # first occurrences, each followed by a byte that differs from the one after its second occurrence
        for seg, at in [(anchor, -1)] + seen:
            nxt = body[at + len(seg)] if at >= 0 else body[0]
            self.out += seg + bytes([nxt ^ 0x5A])
            self.filler(40, 80)
        self.out += self.rand((-(len(self.out) + len(anchor))) % 32)
        self.out += anchor
        p = len(self.out)
        self.out += body
        self.filler(150, 250)
        return p

    def block(self, pattern, count=40):
        ps = []
        while len(self.out) < BLOCK - 1500 and len(ps) < count:
            ps.append(self.place(pattern))
        return bytes(self.out[:BLOCK]), ps


def craft(oracle, pattern, want, forbid=(), seed=0, count=40):
    """A block of `pattern` instances; asserts that for most of them the oracle takes the anchor copy ending at P,
    every copy in `want` (start, end offsets from P) and no copy starting in a `forbid` range."""
    block, ps = Crafter(seed).block(pattern, count)
    got = set(matches(oracle.compress(block)))
    ends = {e for _, e in got}
    starts = sorted(s for s, _ in got)
    hit = [p for p in ps if p in ends and all((p + a, p + b) in got for a, b in want)
           and not any(p + a <= s < p + b for a, b in forbid for s in starts)]
    assert len(hit) >= len(ps) // 2 > 0, (len(hit), len(ps))
    return block


@pytest.mark.parametrize("end", [31, 32, 63, 64])
def test_copy_ends_at_step_edges(oracle, end):
    # scan from P + 1, hit at P + 3: a copy [P + 3, P + end)
    block = craft(oracle, [("rand", 3), ("copy", end - 3)], [(3, end)], seed=end)
    for hybrid in (False, True):
        hoisted, loop_top = check(oracle, [block], hybrid=hybrid)
        assert hoisted > 0 and loop_top > 0


def test_sixteen_copies_in_one_step(oracle):
    # 16 back-to-back 4-byte copies from P, each found by the rematch probe at the previous one's end: the longest
    # chain 64 positions hold, which the doubling must follow to its end
    block = craft(oracle, [("copy", 4)] * 16, [(4 * k, 4 * k + 4) for k in range(16)], seed=16)
    check(oracle, [block])
    check(oracle, [block], hybrid=True)


@pytest.mark.parametrize("case", ["half0_into_half1", "half1_to_next_step", "half1_past_next_step"])
def test_long_copies_across_halves(oracle, case):
    if case == "half0_into_half1":
        # a 40-byte copy [P + 5, P + 45) whose end is only known after the extension, then a rematch hit at its end
        pattern, want = [("rand", 5), ("copy", 40), ("copy", 4)], [(5, 45), (45, 49)]
    elif case == "half1_to_next_step":
        # a 50-byte copy [P + 36, P + 86): its copy-end insert takes the hash from the next step's first half
        pattern, want = [("rand", 3), ("copy", 4), ("rand", 29), ("copy", 50)], [(3, 7), (36, 86)]
    else:
        # a 70-byte copy [P + 52, P + 122) from 48 on (no re-doubling) ending past the next step's first half
        pattern = [("rand", 3), ("copy", 4), ("rand", 23), ("copy", 4), ("rand", 18), ("copy", 70)]
        want = [(3, 7), (30, 34), (52, 122)]
    block = craft(oracle, pattern, want, seed=len(case))
    check(oracle, [block])
    check(oracle, [block], hybrid=True)


def test_same_slot_pair_across_halves(oracle):
    # a fresh 6-byte group at P + 12 recurs at P + 44: both are probed in the same step, where the probe at P + 44
    # read the table before P + 12 was inserted. P + 44 is the victim: the step is cut there and the copy
    # [P + 44, P + 50) comes from P + 12
    pattern = [("rand", 3), ("copy", 4), ("rand", 5), ("again", "k", 6), ("rand", 12), ("copy", 4), ("rand", 10),
               ("again", "k", 6)]
    block = craft(oracle, pattern, [(3, 7), (30, 34), (44, 50)], seed=44)
    for hybrid in (False, True):
        hoisted, loop_top = check(oracle, [block], hybrid=hybrid)
        assert hoisted > 0 and loop_top > 0


def test_scan_leaves_stride_one_in_half1(oracle):
    # after the copy [P + 3, P + 7) the scan from P + 8 finds nothing: its 33rd probe, at P + 40, doubles the stride
    block = craft(oracle, [("rand", 3), ("copy", 4), ("rand", 90)], [(3, 7)], forbid=[(7, 64)], seed=33)
    check(oracle, [block])
    check(oracle, [block], hybrid=True)


def test_block_tails(oracle):
    # short blocks, where the fast path ends within the first steps or never runs, and full blocks, whose last
    # steps reach s_limit at every offset
    text = corpus("alice29.txt") + corpus("plrabn12.txt")
    units = [text[n * 7:n * 8] for n in range(17, 201)]
    units += [text[k * 4099:k * 4099 + BLOCK] for k in range(8)]
    hoisted, loop_top = check(oracle, units)
    assert hoisted > 0 and loop_top > 0
    check(oracle, units[:40] + units[-2:], hybrid=True)


def test_steps_per_bench_block(oracle):
    # the bench's text blocks: about 1,100 fast-path steps per 64 KB block (a 32-position step needs about 2,100)
    units = bench_blocks(4) + bench_blocks(4, first=131072)
    hoisted, loop_top = check(oracle, units)
    steps = (hoisted + loop_top) / len(units)
    assert 900 < steps < 1200, steps
