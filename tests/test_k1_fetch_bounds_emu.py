"""K1's parser fetches the sequential words of the next window ahead of time and prefetches the words four windows
ahead into L2. These tests run the K1 body under the CPU warp emulator on blocks whose length puts those fetches
within 0..64 bytes of the block's end, compare the output with the oracle byte for byte, and use the emulator's
counters to show that no sequential-word fetch reached byte n of a block and no probe read a stale table slot.
The L2 prefetch does nothing in the emulator; its address is clamped to n - 1."""
import ctypes as C

import emu_helpers as emu
from conftest import corpus

BLOCK = 65536


def counters():
    return (C.c_ulonglong * 4).in_dll(emu.lib(), "sb_emu_k1_windows")


def check(oracle, units, hybrid=False):
    cnt = counters()
    for i in range(4):
        cnt[i] = 0
    got = emu.compress_units(units, hybrid=hybrid)
    assert [i for i, (g, u) in enumerate(zip(got, units)) if g != oracle.compress(u)] == []
    assert cnt[2] == 0, "a probe read a table slot that changed before its use"
    assert cnt[3] == 0, "a sequential-word fetch reached the end of its block"
    return cnt[0], cnt[1]


def test_fetches_near_the_end_of_full_blocks(oracle):
    # every block length in the last 64 bytes below 64 KiB: the last one-ahead fetch (w + 100 < n) and the L2
    # prefetch (clamped to n - 1) fall at every offset from the end
    text = corpus("lcet10.txt") + corpus("plrabn12.txt")
    units = [text[k * 997:k * 997 + BLOCK - d] for k, d in enumerate(range(0, 65))]
    hoisted, loop_top = check(oracle, units)
    assert hoisted > 0 and loop_top > 0


def test_fetches_near_the_end_of_short_blocks(oracle):
    text = corpus("alice29.txt")
    units = [text[:n] for n in range(1000, 1065)] + [text[:n] for n in range(100, 240, 7)]
    for hybrid in (False, True):
        check(oracle, units, hybrid=hybrid)


def test_copies_ending_in_the_last_windows(oracle):
    # a block that repeats its own text, so long copies run up to the end and their copy-end inserts fall in
    # the last windows, where the next window's words are not fetched ahead
    text = corpus("asyoulik.txt")[:20000]
    units = [(text * 4)[:n] for n in (BLOCK - 1, BLOCK - 33, BLOCK - 64, 40001, 40033)]
    check(oracle, units)
