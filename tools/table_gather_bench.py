"""Gathers: many small ranges over tabled frame and raw streams in one sb_*_table_gather_device_ws call, against the
range calls (sb_*_table_decode_ranges_device_ws) in calls of 4,096 ranges, and against the batch decode of everything.

  (a) 2^20 random 256 B ranges over --streams frame streams of 16 MiB decoded text (each its own copy of one encoded
      stream, tabled by sb_frame_table_build_device_ws): one gather call, the range calls in groups of 4,096, and
      sb_frame_decode_batch_device_ws of every stream;
  (b) as (a) with the streams Zipf-skewed (s = 1.1): the first stream gets about one range in seven, hundreds per chunk;
  (c) (a) and (b) over --streams raw units of 16 MiB (sb_compress_batch_device_ws, tabled by
      sb_raw_table_build_batch_device_ws), against sb_decompress_batch_device_ws;
  (d) 4,096 random 4 KiB ranges, mostly over distinct chunks: the gather against one range call, frame and raw;
  (e) large ranges, where nearly every chunk is interior: one whole stream (16 MiB, one range in the call) and 64 whole
      streams (1 GiB), the gather against one range call, frame and raw.
Every range is compared with the batch decode before and after the timed calls; calls being compared run alternately,
each the median of --reps calls after a warm-up.

    python tools/table_gather_bench.py [--streams 1024] [--only fr] [--reps 5] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import random
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from frame_range_decode_bench import KIB, MIB, card, check, device_text, graft  # noqa: E402
from frame_table_bench import Table, alternating, cuda_stream, encode_with_ident  # noqa: E402
from raw_table_bench import Batch  # noqa: E402

D = 16 * MIB
GROUP = 4096


def i64(v):
    return torch.from_numpy(np.asarray(v, dtype=np.uint64).view(np.int64)).cuda()


class Calls:
    """The ranges of one workload over `count` tabled streams, as one gather call or range calls of GROUP ranges."""

    def __init__(self, L, snap, fmt, t_tables, t_ins, t_lens, count, ranges, gather):
        self.L, self.snap, self.count = L, snap, count
        self.t_tables, self.t_ins, self.t_lens = t_tables, t_ins, t_lens
        self.k = k = len(ranges)
        self.ranges = ranges
        self.n = np.array([n for _, _, n in ranges], dtype=np.int64)
        self.at = np.concatenate([[0], np.cumsum(self.n)]).astype(np.int64)
        self.out = torch.empty(int(self.at[-1]) + 1, dtype=torch.uint8, device="cuda")
        self.t_lo = i64([lo for _, lo, _ in ranges])
        self.t_len = i64(self.n)
        self.t_ptr = i64(self.at[:k] + self.out.data_ptr())
        self.t_unit = torch.from_numpy(np.array([u for u, _, _ in ranges], dtype=np.uint32).view(np.int32)).cuda()
        self.t_ol = torch.zeros(k, dtype=torch.int64, device="cuda")
        self.t_st = torch.zeros(4 * k, dtype=torch.int64, device="cuda")
        name = "gather" if gather else "decode_ranges"
        self.fn = getattr(L, "sb_%s_table_%s_device_ws" % (fmt, name))
        nb = getattr(L, "sb_%s_table_%s_scratch_bytes" % (fmt, "gather" if gather else "ranges"))
        self.parts = [(0, k)] if gather else [(a, min(a + GROUP, k)) for a in range(0, k, GROUP)]
        self.need = max(nb(b - a) for a, b in self.parts)
        self.scr = torch.empty(self.need, dtype=torch.uint8, device="cuda")

    def __call__(self):
        e = self.snap._lib.SbError()
        for a, b in self.parts:
            check(self.fn(self.t_tables.data_ptr(), self.t_ins.data_ptr(), self.t_lens.data_ptr(), self.count,
                          self.t_unit.data_ptr() + 4 * a, self.t_lo.data_ptr() + 8 * a, self.t_len.data_ptr() + 8 * a,
                          self.t_ptr.data_ptr() + 8 * a, self.t_ol.data_ptr() + 8 * a, self.t_st.data_ptr() + 32 * a,
                          b - a, self.scr.data_ptr(), self.need, cuda_stream(), C.byref(e)), e)

    def verify(self, full, base):
        """Every range Ok and equal to full[base[u] + lo:][:n] (all ranges of one workload have one length)."""
        torch.cuda.synchronize()
        assert bool((self.t_st.view(-1, 4)[:, 0] & 0xFFFFFFFF == 0).all()) and torch.equal(self.t_ol.cpu(),
                                                                                           torch.from_numpy(self.n))
        n = int(self.n[0])
        assert (self.n == n).all()
        start = base[self.t_unit.long()] + self.t_lo
        step = max(1, (1 << 24) // n)
        for a in range(0, self.k, step):
            idx = start[a:a + step, None] + torch.arange(n, device="cuda")[None, :]
            assert torch.equal(self.out[a * n:(a + len(idx)) * n].view(-1, n), full[idx]), a


def workloads(count, sizes, rng):
    """(a) uniform 2^20 x 256 B, (b) Zipf 2^20 x 256 B, (d) 4,096 x 4 KiB, (e) 1 and 64 whole streams."""
    nr = 1 << 20
    uni = [(rng.randrange(count), rng.randrange(D - 256), 256) for _ in range(nr)]
    w = 1.0 / np.arange(1, count + 1) ** 1.1
    units = np.random.default_rng(7).choice(count, nr, p=w / w.sum())
    zipf = [(int(u), rng.randrange(D - 256), 256) for u in units]
    small = [(rng.randrange(count), rng.randrange(D - 4 * KIB), 4 * KIB) for _ in range(4096)]
    return {"uniform_2^20x256B": uni, "zipf_2^20x256B": zipf, "4096x4KiB": small, "1x16MiB": [(count // 2, 0, D)],
            "64x16MiB": [(u, 0, D) for u in rng.sample(range(count), 64)]}


def measure(fmt, L, snap, tables, ins, lens, count, full, base, decode_all, reps, rows):
    for name, ranges in workloads(count, [D] * count, random.Random(1)).items():
        g = Calls(L, snap, fmt, tables, ins, lens, count, ranges, True)
        r = Calls(L, snap, fmt, tables, ins, lens, count, ranges, False)
        for c in (g, r):
            c()
            c.verify(full, base)
        fns = [g, r] + ([decode_all] if len(ranges) > GROUP else [])
        ts = alternating(fns, reps)
        g.verify(full, base)
        r.verify(full, base)
        row = {"ranges": len(ranges), "gather_seconds": ts[0], "range_calls_seconds": ts[1], "range_calls": len(r.parts),
               "range_calls_over_gather": ts[1] / ts[0], "gather_scratch_bytes": g.need,
               "range_scratch_bytes_per_call": r.need}
        if len(ts) > 2:
            row.update(batch_decode_seconds=ts[2], gather_over_batch_decode=ts[0] / ts[2])
        rows["%s_%s" % (fmt, name)] = row
        print("%s_%s" % (fmt, name), json.dumps(row), flush=True)
        del g, r
        torch.cuda.empty_cache()


def part_frame(L, snap, count, reps, rows):
    text = device_text(D)
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
    out = torch.empty(count * D, dtype=torch.uint8, device="cuda")
    olens = torch.zeros(count, dtype=torch.int32, device="cuda")
    sts = torch.zeros(count * 32, dtype=torch.uint8, device="cuda")
    b = snap._lib.SbBatch()
    b.in_base, b.in_stride, b.in_len_uniform = big.data_ptr(), clen, clen
    b.out_base, b.out_stride, b.out_cap_uniform = out.data_ptr(), D, D
    b.out_lens, b.statuses, b.count = olens.data_ptr(), sts.data_ptr(), count
    mc = count * (D // 65536) + 1
    bneed = L.sb_frame_decode_batch_scratch_bytes(count, count * clen, mc)
    bscr = torch.empty(bneed, dtype=torch.uint8, device="cuda")

    def decode_all():
        e = snap._lib.SbError()
        check(L.sb_frame_decode_batch_device_ws(C.byref(b), count * clen, 0, None, None, mc, None, bscr.data_ptr(), bneed,
                                                cuda_stream(), C.byref(e)), e)
    decode_all()
    torch.cuda.synchronize()
    assert bool((olens == D).all()) and bool((sts == 0).all()) and torch.equal(out[:D], text)
    print("frame: %d streams of 16 MiB, %.2f GB compressed" % (count, count * clen / 1e9), flush=True)
    measure("frame", L, snap, i64([t.table.data_ptr() for t in tables]), i64([t.data_ptr() for t in ins]),
            i64([clen] * count), count, out, torch.arange(count, device="cuda") * D, decode_all, reps, rows)
    del out, bscr, big, ins, tables
    torch.cuda.empty_cache()


def part_raw(L, snap, count, reps, rows):
    step = 104729
    text = device_text(D + count * step)
    cap = L.sb_max_compress_len(D)
    slots = torch.empty(count * cap, dtype=torch.uint8, device="cuda")
    lens = torch.zeros(count, dtype=torch.int32, device="cuda")
    sts = torch.zeros(32 * count, dtype=torch.uint8, device="cuda")
    b = snap._lib.SbBatch()
    b.in_base, b.in_stride, b.in_len_uniform = text.data_ptr(), step, D
    b.out_base, b.out_stride, b.out_cap_uniform = slots.data_ptr(), cap, cap
    b.out_lens, b.statuses, b.count = lens.data_ptr(), sts.data_ptr(), count
    need = L.sb_compress_batch_scratch_bytes(count, count * D)
    scr = torch.empty(need, dtype=torch.uint8, device="cuda")
    e = snap._lib.SbError()
    check(L.sb_compress_batch_device_ws(C.byref(b), count * D, scr.data_ptr(), need, cuda_stream(), C.byref(e)), e)
    torch.cuda.synchronize()
    assert bool((sts == 0).all())
    del scr
    bt = Batch(L, snap, [slots.data_ptr() + u * cap for u in range(count)], lens.cpu().tolist(), [D] * count)
    bt.build()
    bt.decode_all()
    torch.cuda.synchronize()
    offs = bt.t_res[:8 * (count + 1)].cpu().numpy().view(np.uint64)
    assert all(torch.equal(bt.t_out[u * D:(u + 1) * D], text[u * step:u * step + D]) for u in (0, count - 1))
    print("raw: %d units of 16 MiB, %.2f GB compressed" % (count, bt.in_bytes / 1e9), flush=True)
    measure("raw", L, snap, i64(offs[:count] + bt.t_tab.data_ptr()), bt.t_ip, i64(bt.lens), count, bt.t_out,
            torch.from_numpy(bt.at).cuda(), bt.decode_all, reps, rows)
    del bt, slots, text
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=1024, help="streams of 16 MiB decoded per format")
    ap.add_argument("--only", default="fr", help="f: frame streams, r: raw streams")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for table_gather_bench.json (default: print only)")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    snap = graft.load_package()
    L = snap._lib.lib()
    info = {"card": card(), "rows": {}}
    print("card:", info["card"], flush=True)
    if "f" in args.only:
        part_frame(L, snap, args.streams, args.reps, info["rows"])
    if "r" in args.only:
        part_raw(L, snap, args.streams, args.reps, info["rows"])
    info["card_after"] = card()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "table_gather_bench.json"), "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
