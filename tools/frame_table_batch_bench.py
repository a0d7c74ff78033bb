"""Seek tables of many streams in one call: sb_frame_table_build_batch_device_ws against one
sb_frame_table_build_device_ws per stream and against sb_frame_decode_batch_device_ws of the same batch.

  (a) --small streams of 64 KiB decoded text (64 distinct encoded slices, each stream its own copy of the bytes);
  (b) --large streams of 16 MiB decoded text;
      for both: one batch build, one single build per stream (timed over --subset streams and scaled to all), and the
      batch decode of everything. Every batch-built table is compared byte for byte with its single build, for all
      streams in (b) and --subset streams in (a), and 4,096 random ranges read through the batch-built tables are
      compared with the batch decode.
  (c) frame.TableReader construction over --readers host-memory streams of 64 KiB, wall clock ending in a synchronise,
      against building the same tables one call per stream.
Compared calls run alternately, each the median of --reps calls after a warm-up.

    python tools/frame_table_batch_bench.py [--small 131072] [--large 1024] [--subset 1024] [--readers 100000]
                                            [--reps 5] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import random
import statistics
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from frame_range_decode_bench import KIB, MIB, card, check, device_text, graft  # noqa: E402
from frame_table_bench import Table, TableRanges, alternating, cuda_stream, encode_with_ident  # noqa: E402

DISTINCT = 64


class BatchSet:
    """`count` framed streams of `d` decoded bytes on the device: DISTINCT encoded slices of the text, tiled so that
    every stream has its own copy of its bytes."""

    def __init__(self, L, snap, text, d, count):
        encs = [encode_with_ident(L, snap, text[k * 9973 % (text.numel() - d):][:d].contiguous(), d)
                for k in range(min(DISTINCT, count))]
        self.texts = [text[k * 9973 % (text.numel() - d):][:d] for k in range(len(encs))]
        block = torch.cat(encs)
        reps = (count + len(encs) - 1) // len(encs)
        self.big = block.repeat(reps)
        at, self.ins, self.lens, self.which = 0, [], [], []
        for r in range(reps):
            for k, e in enumerate(encs):
                if len(self.ins) < count:
                    self.ins.append(self.big[at:at + e.numel()])
                    self.lens.append(e.numel())
                    self.which.append(k)
                at += e.numel()
        self.count, self.d, self.chunks = count, d, (d + 65535) // 65536
        self.in_bytes = sum(self.lens)
        self.max_chunks = count * self.chunks + 1
        i64 = lambda v: torch.tensor(v, dtype=torch.int64, device="cuda")
        self.ptrs = i64([t.data_ptr() for t in self.ins])
        self.t_lens = torch.tensor(self.lens, dtype=torch.int32, device="cuda")


class BatchBuild:
    def __init__(self, L, snap, s):
        self.L, self.snap, self.s = L, snap, s
        b = snap._lib.SbBatch()
        b.in_ptrs, b.in_lens, b.count = s.ptrs.data_ptr(), s.t_lens.data_ptr(), s.count
        self.b = b
        self.tb = L.sb_frame_table_batch_bytes(s.count, s.max_chunks)
        self.tables = torch.empty(self.tb, dtype=torch.uint8, device="cuda")
        self.offs = torch.zeros(s.count + 1, dtype=torch.int64, device="cuda")
        self.rsz = C.sizeof(snap._lib.SbFrameResult)
        self.res = torch.zeros(s.count * self.rsz, dtype=torch.uint8, device="cuda")
        self.need = L.sb_frame_table_build_batch_scratch_bytes(s.count, s.in_bytes, s.max_chunks)
        self.scr = torch.empty(self.need, dtype=torch.uint8, device="cuda")

    def __call__(self):
        e = self.snap._lib.SbError()
        check(self.L.sb_frame_table_build_batch_device_ws(C.byref(self.b), self.s.in_bytes, 0, None, None, self.s.max_chunks,
                                                          self.tables.data_ptr(), self.tb, self.offs.data_ptr(),
                                                          self.res.data_ptr(), self.scr.data_ptr(), self.need,
                                                          cuda_stream(), C.byref(e)), e)

    def table(self, i):
        o = self.offs_host
        return self.tables[o[i]:o[i + 1]]

    def settle(self):
        torch.cuda.synchronize()
        self.offs_host = self.offs.cpu().tolist()
        r = self.res.cpu().view(-1, self.rsz)
        codes = r[:, :4].contiguous().view(torch.int32)[:, 0]
        assert bool((codes == 0).all()), "a unit failed"
        assert bool((r[:, 32:40].contiguous().view(torch.int64)[:, 0] == self.s.d).all())


class BatchDecode:
    def __init__(self, L, snap, s):
        self.L, self.snap, self.s = L, snap, s
        self.out = torch.empty(s.count * s.d, dtype=torch.uint8, device="cuda")
        self.olens = torch.zeros(s.count, dtype=torch.int32, device="cuda")
        self.sts = torch.zeros(s.count * 32, dtype=torch.uint8, device="cuda")
        b = snap._lib.SbBatch()
        b.in_ptrs, b.in_lens, b.count = s.ptrs.data_ptr(), s.t_lens.data_ptr(), s.count
        b.out_base, b.out_stride, b.out_cap_uniform = self.out.data_ptr(), s.d, s.d
        b.out_lens, b.statuses = self.olens.data_ptr(), self.sts.data_ptr()
        self.b = b
        self.need = L.sb_frame_decode_batch_scratch_bytes(s.count, s.in_bytes, s.max_chunks)
        self.scr = torch.empty(self.need, dtype=torch.uint8, device="cuda")

    def __call__(self):
        e = self.snap._lib.SbError()
        check(self.L.sb_frame_decode_batch_device_ws(C.byref(self.b), self.s.in_bytes, 0, None, None, self.s.max_chunks, None,
                                                     self.scr.data_ptr(), self.need, cuda_stream(), C.byref(e)), e)


def part_ab(L, snap, text, name, d, count, subset, reps, rows):
    s = BatchSet(L, snap, text, d, count)
    print("(%s) %d streams of %d bytes decoded, %.2f GB compressed" % (name, count, d, s.in_bytes / 1e9), flush=True)
    bb, dec = BatchBuild(L, snap, s), BatchDecode(L, snap, s)
    sub = list(range(0, count, max(count // subset, 1)))[:subset]
    singles = [Table(L, snap, s.ins[i], s.lens[i], s.lens[i] // 1024 + 16, fragment=False) for i in sub]

    def per_stream():
        for t in singles:
            t.build()
    bb()
    dec()
    per_stream()
    bb.settle()
    assert bool((dec.olens == d).all()) and bool((dec.sts == 0).all())
    for k in range(len(s.texts)):                                         # the batch decode is the reference
        assert torch.equal(dec.out[k * d:(k + 1) * d], s.texts[s.which[k]])

    def compare():
        for i, t in zip(sub, singles):
            assert t.result() == (0, d, s.chunks), (i, t.result())
            exact = L.sb_frame_table_bytes(s.chunks)
            assert torch.equal(bb.table(i), t.table[:exact]), i
    compare()
    rng = random.Random(3)
    ranges = [(rng.randrange(count), rng.randrange(d - 4 * KIB), 4 * KIB) for _ in range(4096)]
    units = [(s.ins[i], s.lens[i], bb.table(i)) for i in range(count)]
    rd = TableRanges(L, snap, units, ranges)
    rd()
    torch.cuda.synchronize()
    want = lambda u, lo, n: dec.out[u * d + lo:u * d + lo + n]
    rd.verify(want)
    t_batch, t_single, t_dec = alternating([bb, per_stream, dec], reps)
    bb.settle()
    compare()
    rd()
    torch.cuda.synchronize()
    rd.verify(want)
    scaled = t_single * count / len(sub)
    rows[name] = {"streams": count, "decoded_bytes_each": d, "compressed_bytes": s.in_bytes,
                  "batch_build_seconds": t_batch, "single_builds_seconds_scaled": scaled, "single_subset": len(sub),
                  "batch_decode_seconds": t_dec, "single_over_batch_build": scaled / t_batch,
                  "decode_over_batch_build": t_dec / t_batch, "tables_compared": len(sub), "ranges_compared": len(ranges)}
    print(name, json.dumps(rows[name]), flush=True)
    del s, bb, dec, singles, units, rd
    torch.cuda.empty_cache()


def part_c(L, snap, text, count, reps, rows):
    d = 64 * KIB
    encs = [encode_with_ident(L, snap, text[k * 9973:k * 9973 + d].contiguous(), d).cpu().numpy().tobytes()
            for k in range(DISTINCT)]
    texts = [text[k * 9973:k * 9973 + d].cpu().numpy().tobytes() for k in range(DISTINCT)]
    streams = [bytes(encs[i % DISTINCT]) for i in range(count)]          # host memory, one object per stream
    rd_holder = []

    def batch():
        rd_holder[:] = [snap.frame.TableReader(streams)]
        torch.cuda.synchronize()

    def single():
        rd = rd_holder[0]
        caps = [min(len(x) // 1024 + 16, snap.frame.MAX_BATCH_CHUNKS) for x in streams]
        rd._build_each(range(count), caps, 0)
        torch.cuda.synchronize()
    batch()
    before = L.sb_launch_count()
    batch()
    launches = L.sb_launch_count() - before
    rd = rd_holder[0]
    assert rd.lengths == [d] * count
    rng = random.Random(4)
    ranges = [(rng.randrange(count), rng.randrange(d), rng.randrange(1, 3 * d)) for _ in range(2000)]
    assert rd.read_ranges(ranges) == [texts[i % DISTINCT][lo:lo + n] for i, lo, n in ranges]
    single()
    tb, ts = [], []
    for _ in range(reps):
        for f, acc in ((batch, tb), (single, ts)):
            t0 = time.perf_counter()
            f()
            acc.append(time.perf_counter() - t0)
    rows["c_reader"] = {"streams": count, "decoded_bytes_each": d, "construct_seconds": statistics.median(tb),
                        "single_builds_seconds": statistics.median(ts), "construct_launches": launches,
                        "single_over_construct": statistics.median(ts) / statistics.median(tb)}
    print("c_reader", json.dumps(rows["c_reader"]), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--small", type=int, default=131072, help="streams of 64 KiB in (a)")
    ap.add_argument("--large", type=int, default=1024, help="streams of 16 MiB in (b)")
    ap.add_argument("--subset", type=int, default=1024, help="streams timed one single build each")
    ap.add_argument("--readers", type=int, default=100000, help="host streams of 64 KiB in (c)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for frame_table_batch_bench.json (default: print only)")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    snap = graft.load_package()
    L = snap._lib.lib()
    info = {"card": card(), "rows": {}}
    print("card:", info["card"], flush=True)
    text = device_text(64 * MIB)
    part_ab(L, snap, text, "a_64KiB", 64 * KIB, args.small, args.subset, args.reps, info["rows"])
    part_ab(L, snap, text, "b_16MiB", 16 * MIB, args.large, args.subset, args.reps, info["rows"])
    part_c(L, snap, text, args.readers, min(args.reps, 3), info["rows"])
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "frame_table_batch_bench.json"), "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
