"""Seek tables: sb_frame_table_build_device_ws once per stream, then sb_frame_table_decode_ranges_device_ws over many
streams, against K12 (sb_frame_decode_ranges_device_ws), which runs the index phase on every call.

  (a) one stream of --gib GiB decoded (frame_range_decode_bench.py's tiled, indexed stream):
      the index phase alone (K12 with no ranges), the table build once, and 1 x 1 GiB, 1,024 x 1 MiB and 1,024 x 4 KiB
      ranges through the table against the same ranges through K12 with the index;
  (b) --streams streams of 16 MiB decoded text, each tabled: 4,096 random 4 KiB ranges over all of them in one table
      call, against one K12 call per stream touched (timed over --subset streams and scaled to all touched streams) and
      against sb_frame_decode_batch_device_ws of every stream;
  (c) the build time of one stream (K7 index, as frame.TableReader builds) across stream sizes.
Every range's bytes are compared with a full decode before and after the timed calls; calls being compared run
alternately, each the median of --reps calls after a warm-up.

    python tools/frame_table_bench.py [--gib 16] [--streams 1024] [--subset 64] [--reps 5] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import random
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from frame_range_decode_bench import GIB, KIB, MIB, UNIT, Ranges, Stream, card, check, device_text, graft  # noqa: E402


def cuda_stream():
    return torch.cuda.current_stream().cuda_stream


def alternating(fns, reps):
    """Median seconds of each callable, the callables run in turn after one warm-up call each."""
    for f in fns:
        f()
    torch.cuda.synchronize()
    ts = [[] for _ in fns]
    for _ in range(reps):
        for i, f in enumerate(fns):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            f()
            b.record()
            b.synchronize()
            ts[i].append(a.elapsed_time(b) / 1e3)
    return [statistics.median(t) for t in ts]


class Table:
    """One stream's seek table, built on the device (with the caller's index when given)."""

    def __init__(self, L, snap, t_in, n, max_chunks, index=None, nchunks=0, fragment=True):
        self.L, self.snap, self.t_in, self.n, self.max_chunks = L, snap, t_in, n, max_chunks
        self.index, self.nchunks, self.flags = index, nchunks, 1 if fragment else 0
        self.tb = L.sb_frame_table_bytes(max_chunks)
        self.table = torch.empty(self.tb, dtype=torch.uint8, device="cuda")
        self.need = L.sb_frame_table_build_scratch_bytes(max_chunks)
        self.scr = torch.empty(self.need, dtype=torch.uint8, device="cuda")
        self.res = torch.zeros(64, dtype=torch.uint8, device="cuda")

    def build(self):
        e = self.snap._lib.SbError()
        check(self.L.sb_frame_table_build_device_ws(self.t_in.data_ptr(), self.n,
                                                    self.index.data_ptr() if self.index is not None else None,
                                                    self.nchunks, self.flags, self.table.data_ptr(), self.tb,
                                                    self.max_chunks, self.res.data_ptr(), self.scr.data_ptr(), self.need,
                                                    cuda_stream(), C.byref(e)), e)

    def result(self):
        r = self.res.cpu()
        return int(r[:4].view(torch.int32)[0]), int(r[32:40].view(torch.int64)[0]), int(r[40:44].view(torch.int32)[0])

    def free_scratch(self):
        del self.scr


class TableRanges:
    """Device descriptors, buffers and scratch of one table call over units [(input, n, table tensor)], allocated once."""

    def __init__(self, L, snap, units, ranges):
        self.L, self.snap, self.units, self.ranges = L, snap, units, ranges
        k = len(ranges)
        self.out = torch.empty(sum(n for _, _, n in ranges) + 1, dtype=torch.uint8, device="cuda")
        offs, at = [], 0
        for _, _, n in ranges:
            offs.append(at)
            at += n
        self.offs = offs
        i64 = lambda v: torch.tensor(v, dtype=torch.int64, device="cuda")
        self.tabs = i64([t.data_ptr() for _, _, t in units])
        self.ins = i64([i.data_ptr() for i, _, _ in units])
        self.lens = i64([n for _, n, _ in units])
        self.unit = torch.tensor([u for u, _, _ in ranges], dtype=torch.int32, device="cuda")
        self.desc = i64([lo for _, lo, _ in ranges] + [n for _, _, n in ranges] + [self.out.data_ptr() + o for o in offs])
        self.res = torch.zeros(5 * k, dtype=torch.int64, device="cuda")
        self.need = L.sb_frame_table_ranges_scratch_bytes(k)
        self.scr = torch.empty(self.need, dtype=torch.uint8, device="cuda")

    def __call__(self):
        k, p, e = len(self.ranges), self.desc.data_ptr(), self.snap._lib.SbError()
        check(self.L.sb_frame_table_decode_ranges_device_ws(self.tabs.data_ptr(), self.ins.data_ptr(), self.lens.data_ptr(),
                                                            len(self.units), self.unit.data_ptr(), p, p + 8 * k,
                                                            p + 16 * k, self.res.data_ptr(), self.res.data_ptr() + 8 * k, k,
                                                            self.scr.data_ptr(), self.need, cuda_stream(), C.byref(e)), e)

    def verify(self, want):
        """want(u, lo, n) -> the expected bytes as a CUDA tensor."""
        back, k = self.res.cpu(), len(self.ranges)
        assert (back[k:5 * k].view(-1, 4)[:, 0] & 0xFFFFFFFF).eq(0).all(), "a range failed"
        for (u, lo, n), o, m in zip(self.ranges, self.offs, back[:k].tolist()):
            assert m == n and torch.equal(self.out[o:o + n], want(u, lo, n)), (u, lo, n)


def part_a(L, snap, text, gib, reps, rows):
    s = Stream(L, snap, text, gib * GIB // UNIT)
    print("(a) stream: %d GiB decoded, %.2f GB compressed, %d chunks, indexed" % (s.total // GIB, s.n / 1e9, s.nchunks),
          flush=True)
    # the full decode every range is compared with
    full = torch.empty(s.total, dtype=torch.uint8, device="cuda")
    fres = torch.zeros(64, dtype=torch.uint8, device="cuda")
    fneed = L.sb_frame_decode_scratch_bytes(s.max_chunks)
    fscr = torch.empty(fneed, dtype=torch.uint8, device="cuda")
    e = snap._lib.SbError()
    check(L.sb_frame_decode_device_ws(s.t.data_ptr(), s.n, full.data_ptr(), s.total, s.idx.data_ptr(), s.nchunks, 1,
                                      fres.data_ptr(), fscr.data_ptr(), fneed, s.max_chunks, cuda_stream(), C.byref(e)), e)
    torch.cuda.synchronize()
    assert int(fres[:4].cpu().view(torch.int32)[0]) == 0 and int(fres[32:40].cpu().view(torch.int64)[0]) == s.total
    del fscr
    want = lambda u, lo, n: full[lo:lo + n]
    idx_only = Ranges(L, snap, s, [])
    tab = Table(L, snap, s.t, s.n, s.max_chunks, index=s.idx, nchunks=s.nchunks)
    tab.build()
    torch.cuda.synchronize()
    assert tab.result() == (0, s.total, s.nchunks), tab.result()
    t_index, t_build = alternating([idx_only, tab.build], reps)
    rows["a_index_phase"] = {"seconds": t_index}
    rows["a_table_build"] = {"seconds": t_build, "table_bytes": L.sb_frame_table_bytes(s.nchunks)}
    print("a_index_phase", json.dumps(rows["a_index_phase"]), "a_table_build", json.dumps(rows["a_table_build"]), flush=True)
    tab.free_scratch()
    rng = random.Random(1)
    cases = {
        "one_1GiB": [(5 * GIB + 12345, GIB)],
        "1024x1MiB": [(rng.randrange(s.total - MIB), MIB) for _ in range(1024)],
        "1024x4KiB": [(rng.randrange(s.total - 4 * KIB), 4 * KIB) for _ in range(1024)],
    }
    units = [(s.t, s.n, tab.table)]
    for name, ranges in cases.items():
        k12 = Ranges(L, snap, s, ranges)
        k13 = TableRanges(L, snap, units, [(0, lo, n) for lo, n in ranges])
        for f in (k12, k13):
            f()
        torch.cuda.synchronize()
        k13.verify(want)
        for (lo, n), o, m in zip(ranges, k12.offs, k12.res[:len(ranges)].tolist()):
            assert m == n and torch.equal(k12.out[o:o + n], want(0, lo, n))
        t12, t13 = alternating([k12, k13], reps)
        k13.verify(want)
        for (lo, n), o, m in zip(ranges, k12.offs, k12.res[:len(ranges)].tolist()):
            assert m == n and torch.equal(k12.out[o:o + n], want(0, lo, n))
        nbytes = sum(n for _, n in ranges)
        rows["a_" + name] = {"ranges": len(ranges), "bytes": nbytes, "k12_seconds": t12, "table_seconds": t13,
                             "k12_over_table": t12 / t13}
        print("a_" + name, json.dumps(rows["a_" + name]), flush=True)
        del k12, k13
    del s, tab, units, full
    torch.cuda.empty_cache()


def encode_with_ident(L, snap, text, n):
    e = snap._lib.SbError()
    cap = L.sb_frame_max_len(n)
    out = torch.empty(cap, dtype=torch.uint8, device="cuda")
    res = torch.zeros(64, dtype=torch.uint8, device="cuda")
    need = L.sb_frame_encode_scratch_bytes(n)
    scr = torch.empty(need, dtype=torch.uint8, device="cuda")
    check(L.sb_frame_encode_device_ws(text.data_ptr(), n, out.data_ptr(), cap, 1, None, res.data_ptr(), scr.data_ptr(), need,
                                      cuda_stream(), C.byref(e)), e)
    torch.cuda.synchronize()
    return out[:int(res[32:40].cpu().view(torch.int64)[0])].clone()


def part_b(L, snap, text, count, subset, reps, rows):
    D = 16 * MIB
    enc = encode_with_ident(L, snap, text, D)
    clen = len(enc)
    big = enc.repeat(count)                                       # every stream its own copy of the bytes
    ins = [big[u * clen:(u + 1) * clen] for u in range(count)]
    cap = D // 65536 + 16
    tables = []
    for t in ins:
        tb = Table(L, snap, t, clen, cap, fragment=False)
        tb.build()
        tables.append(tb)
    torch.cuda.synchronize()
    assert all(t.result() == (0, D, D // 65536) for t in tables[:8])
    for t in tables:
        t.free_scratch()
    units = [(t, clen, tb.table) for t, tb in zip(ins, tables)]
    rng = random.Random(2)
    ranges = [(rng.randrange(count), rng.randrange(D - 4 * KIB), 4 * KIB) for _ in range(4096)]
    k13 = TableRanges(L, snap, units, ranges)
    touched = sorted({u for u, _, _ in ranges})
    sub = touched[:subset]

    class PerStream:
        """One K12 call per stream of the subset, each over that stream's ranges (K7 index phase, as without a table)."""

        def __init__(self):
            self.calls = []
            for u in sub:
                s = type("S", (), {})()
                s.t, s.n, s.max_chunks, s.idx, s.nchunks = ins[u], clen, cap, None, 0
                self.calls.append(K12NoIndex(L, snap, s, [(lo, n) for v, lo, n in ranges if v == u]))

        def __call__(self):
            for c in self.calls:
                c()
    per = PerStream()
    # the batch decode of everything
    out = torch.empty(count * D, dtype=torch.uint8, device="cuda")
    lens = torch.zeros(count, dtype=torch.int32, device="cuda")            # sb_batch out_lens are 32-bit
    sts = torch.zeros(count * 32, dtype=torch.uint8, device="cuda")
    b = snap._lib.SbBatch()
    b.in_base, b.in_stride, b.in_len_uniform = big.data_ptr(), clen, clen
    b.out_base, b.out_stride, b.out_cap_uniform = out.data_ptr(), D, D
    b.out_lens, b.statuses, b.count = lens.data_ptr(), sts.data_ptr(), count
    mc = count * (D // 65536) + 1
    bneed = L.sb_frame_decode_batch_scratch_bytes(count, count * clen, mc)
    bscr = torch.empty(bneed, dtype=torch.uint8, device="cuda")

    def batch():
        e = snap._lib.SbError()
        check(L.sb_frame_decode_batch_device_ws(C.byref(b), count * clen, 0, None, None, mc, None, bscr.data_ptr(), bneed,
                                                cuda_stream(), C.byref(e)), e)
    # the batch decode is the full decode every range is compared with
    batch()
    torch.cuda.synchronize()
    assert bool((lens == D).all()) and bool((sts == 0).all())
    want = lambda u, lo, n: out[u * D + lo:u * D + lo + n]
    k13()
    per()
    torch.cuda.synchronize()
    k13.verify(want)
    for u, c in zip(sub, per.calls):
        c.verify_against(lambda _, lo, n, u=u: want(u, lo, n))
    t13, tper, tbatch = alternating([k13, per, batch], reps)
    k13.verify(want)
    for u, c in zip(sub, per.calls):
        c.verify_against(lambda _, lo, n, u=u: want(u, lo, n))
    scaled = tper * len(touched) / len(sub)
    rows["b_4096x4KiB"] = {"streams": count, "touched": len(touched), "table_seconds": t13,
                           "k12_per_stream_seconds_scaled": scaled, "k12_subset_streams": len(sub),
                           "batch_decode_all_seconds": tbatch, "k12_over_table": scaled / t13,
                           "batch_over_table": tbatch / t13}
    print("b_4096x4KiB", json.dumps(rows["b_4096x4KiB"]), flush=True)
    del out, bscr, big, ins, tables, units, k13, per
    torch.cuda.empty_cache()


class K12NoIndex(Ranges):
    """frame_range_decode_bench's Ranges over a stream with an identifier and no index (K7 builds it per call)."""

    def __call__(self):
        k, p, e = len(self.ranges), self.desc.data_ptr(), self.snap._lib.SbError()
        check(self.L.sb_frame_decode_ranges_device_ws(self.s.t.data_ptr(), self.s.n, None, 0, 0, p, p + 8 * k, p + 16 * k,
                                                      self.res.data_ptr(), self.res.data_ptr() + 8 * k, k,
                                                      self.res.data_ptr() + 40 * k, self.scr.data_ptr(), self.need,
                                                      self.s.max_chunks, cuda_stream(), C.byref(e)), e)

    def verify_against(self, want):
        back, k = self.res.cpu(), len(self.ranges)
        assert (back[k:5 * k].view(-1, 4)[:, 0] & 0xFFFFFFFF).eq(0).all(), "a range failed"
        for (lo, n), o, m in zip(self.ranges, self.offs, back[:k].tolist()):
            assert m == n and torch.equal(self.out[o:o + n], want(0, lo, n)), (lo, n)


def part_c(L, snap, text, reps, rows):
    for d in (64 * KIB, MIB, 16 * MIB, UNIT):
        enc = encode_with_ident(L, snap, text, d)
        tb = Table(L, snap, enc, len(enc), len(enc) // 1024 + 16, fragment=False)
        t = alternating([tb.build], reps)[0]
        assert tb.result() == (0, d, (d + 65535) // 65536)
        rows["c_build_%d" % d] = {"decoded_bytes": d, "compressed_bytes": len(enc), "seconds": t}
        print("c_build_%d" % d, json.dumps(rows["c_build_%d" % d]), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=int, default=16, help="decoded GiB of the stream of (a)")
    ap.add_argument("--streams", type=int, default=1024, help="streams of 16 MiB in (b)")
    ap.add_argument("--subset", type=int, default=64, help="streams of (b) timed one K12 call each")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for frame_table_bench.json (default: print only)")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    snap = graft.load_package()
    L = snap._lib.lib()
    info = {"card": card(), "rows": {}}
    print("card:", info["card"], flush=True)
    text = device_text(UNIT)
    part_c(L, snap, text, args.reps, info["rows"])
    part_a(L, snap, text, args.gib, args.reps, info["rows"])
    part_b(L, snap, text, args.streams, args.subset, args.reps, info["rows"])
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "frame_table_bench.json"), "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
