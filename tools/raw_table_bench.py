"""Raw seek tables: sb_raw_table_build_batch_device_ws once per batch, then sb_raw_table_decode_ranges_device_ws, against
sb_decompress_batch_device_ws of everything (which is also the full decode every range is checked against).

  (a) --units raw units of 16 MiB of corpus text from sb_compress_batch_device_ws: the build, then 4,096 random 4 KiB
      ranges over all of them in one call;
  (b) one unit of 4 GiB - 64 KiB of text (assembled on the device as raw_decode_bench.py does): the build, then
      1 x 1 GiB, 1,024 x 1 MiB and 1,024 x 4 KiB ranges;
  (c) 1,024 pages of 1 MiB compressed by pyarrow (Google's C++ snappy), as raw_batch_decode_bench.py builds them, when
      pyarrow is installed: the build, then 4,096 random 4 KiB ranges.
Every range's bytes are compared with the full decode before and after the timed calls; calls being compared run
alternately, each the median of --reps calls after a warm-up.

    python tools/raw_table_bench.py [--units 1024] [--only abc] [--reps 5] [--out DIR]
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
from frame_range_decode_bench import GIB, KIB, MIB, card, check, device_text, graft  # noqa: E402
from frame_table_bench import alternating, cuda_stream  # noqa: E402
from raw_decode_bench import device_stream  # noqa: E402

BLOCK = 65536


class Batch:
    """Units at in_ptrs on the device (lens, decoded sizes), their tables and the full batch decode."""

    def __init__(self, L, snap, ptrs, lens, sizes):
        self.L, self.snap, self.k = L, snap, len(lens)
        self.lens, self.sizes = list(lens), list(sizes)
        self.in_bytes = sum(self.lens)
        i64 = lambda v: torch.from_numpy(np.array(v, dtype=np.uint64).view(np.int64)).cuda()
        self.t_ip, self.t_lens = i64(list(ptrs)), torch.tensor(self.lens, dtype=torch.int64).to(torch.int32).cuda()
        self.ptrs = list(ptrs)
        # the tables
        self.tb = L.sb_raw_table_batch_bytes(self.k, self.in_bytes)
        self.t_tab = torch.empty(self.tb, dtype=torch.uint8, device="cuda")
        self.t_res = torch.zeros(8 * (self.k + 1) + 48 * self.k, dtype=torch.uint8, device="cuda")
        self.need = L.sb_raw_table_build_batch_scratch_bytes(self.k, self.in_bytes)
        self.t_scr = torch.empty(self.need, dtype=torch.uint8, device="cuda")
        # the batch decode of everything
        self.at = np.concatenate([[0], np.cumsum(self.sizes[:-1])]).astype(np.int64)
        self.t_out = torch.empty(sum(self.sizes) + 16, dtype=torch.uint8, device="cuda")
        self.t_op = i64([self.t_out.data_ptr() + int(a) for a in self.at])
        self.t_caps = torch.tensor(self.sizes, dtype=torch.int64).to(torch.int32).cuda()
        self.t_ol = torch.zeros(self.k, dtype=torch.int32, device="cuda")
        self.t_st = torch.zeros(32 * self.k, dtype=torch.uint8, device="cuda")
        self.dneed = L.sb_decompress_batch_scratch_bytes(self.k, self.in_bytes)
        self.t_dscr = torch.empty(self.dneed, dtype=torch.uint8, device="cuda")

    def batch(self, out):
        b = self.snap._lib.SbBatch()
        b.in_ptrs, b.in_lens, b.count = self.t_ip.data_ptr(), self.t_lens.data_ptr(), self.k
        if out:
            b.out_ptrs, b.out_caps = self.t_op.data_ptr(), self.t_caps.data_ptr()
            b.out_lens, b.statuses = self.t_ol.data_ptr(), self.t_st.data_ptr()
        return b

    def build(self):
        e = self.snap._lib.SbError()
        k = self.k
        check(self.L.sb_raw_table_build_batch_device_ws(C.byref(self.batch(False)), self.in_bytes, self.t_tab.data_ptr(),
                                                        self.tb, self.t_res.data_ptr(), self.t_res.data_ptr() + 8 * (k + 1),
                                                        self.t_scr.data_ptr(), self.need, cuda_stream(), C.byref(e)), e)

    def decode_all(self):
        e = self.snap._lib.SbError()
        check(self.L.sb_decompress_batch_device_ws(C.byref(self.batch(True)), self.in_bytes, None, self.t_dscr.data_ptr(),
                                                   self.dneed, cuda_stream(), C.byref(e)), e)

    def verify_build(self):
        torch.cuda.synchronize()
        k = self.k
        r = self.t_res.cpu().numpy()
        self.offs = r[:8 * (k + 1)].view(np.uint64).astype(np.int64)
        res = r[8 * (k + 1):].view(np.uint64).reshape(k, 6)
        assert (res[:, 0] & 0xFFFFFFFF == 0).all(), "a unit is not seekable"
        assert list(res[:, 4]) == self.sizes
        assert bool((self.t_ol.cpu().to(torch.int64) & 0xFFFFFFFF).eq(torch.tensor(self.sizes)).all())
        assert bool((self.t_st == 0).all())
        self.tables = [self.t_tab.data_ptr() + int(o) for o in self.offs[:k]]
        return int(self.offs[k])

    def want(self, u, lo, n):
        a = int(self.at[u])
        return self.t_out[a + lo:a + lo + n]


class Ranges:
    """Device descriptors, buffers and scratch of one table call over a Batch's tables, allocated once."""

    def __init__(self, L, snap, bt, ranges):
        self.L, self.snap, self.bt, self.ranges = L, snap, bt, ranges
        k = len(ranges)
        self.offs = np.concatenate([[0], np.cumsum([n for _, _, n in ranges][:-1])]).astype(np.int64)
        self.out = torch.empty(sum(n for _, _, n in ranges) + 1, dtype=torch.uint8, device="cuda")
        i64 = lambda v: torch.from_numpy(np.array(v, dtype=np.uint64).view(np.int64)).cuda()
        self.tabs, self.ins = i64(bt.tables), i64(bt.ptrs)
        self.lens = i64(bt.lens)
        self.unit = torch.tensor([u for u, _, _ in ranges], dtype=torch.int32, device="cuda")
        self.desc = i64([lo for _, lo, _ in ranges] + [n for _, _, n in ranges] +
                        [self.out.data_ptr() + int(o) for o in self.offs])
        self.res = torch.zeros(5 * k, dtype=torch.int64, device="cuda")
        self.need = L.sb_raw_table_ranges_scratch_bytes(k)
        self.scr = torch.empty(self.need, dtype=torch.uint8, device="cuda")

    def __call__(self):
        k, p, e = len(self.ranges), self.desc.data_ptr(), self.snap._lib.SbError()
        check(self.L.sb_raw_table_decode_ranges_device_ws(self.tabs.data_ptr(), self.ins.data_ptr(), self.lens.data_ptr(),
                                                          self.bt.k, self.unit.data_ptr(), p, p + 8 * k, p + 16 * k,
                                                          self.res.data_ptr(), self.res.data_ptr() + 8 * k, k,
                                                          self.scr.data_ptr(), self.need, cuda_stream(), C.byref(e)), e)

    def verify(self):
        torch.cuda.synchronize()
        back, k = self.res.cpu(), len(self.ranges)
        assert (back[k:5 * k].view(-1, 4)[:, 0] & 0xFFFFFFFF).eq(0).all(), "a range failed"
        for (u, lo, n), o, m in zip(self.ranges, self.offs, back[:k].tolist()):
            assert m == n and torch.equal(self.out[int(o):int(o) + n], self.bt.want(u, lo, n)), (u, lo, n)


def run_batch(name, L, snap, bt, cases, reps, rows):
    """The build against the full decode, then every case of ranges against the full decode."""
    bt.decode_all()
    bt.build()
    packed = bt.verify_build()
    t_build, t_all = alternating([bt.build, bt.decode_all], reps)
    bt.verify_build()
    rows[name + "_build"] = {"units": bt.k, "compressed_bytes": bt.in_bytes, "decoded_bytes": sum(bt.sizes),
                             "tables_bytes": packed, "build_seconds": t_build, "decode_all_seconds": t_all,
                             "build_GBps_compressed": bt.in_bytes / t_build / 1e9}
    print(name + "_build", json.dumps(rows[name + "_build"]), flush=True)
    for case, ranges in cases.items():
        r = Ranges(L, snap, bt, ranges)
        r()
        r.verify()
        t_r, t_all = alternating([r, bt.decode_all], reps)
        r.verify()
        rows[name + "_" + case] = {"ranges": len(ranges), "bytes": sum(n for _, _, n in ranges), "table_seconds": t_r,
                                   "decode_all_seconds": t_all, "decode_all_over_table": t_all / t_r}
        print(name + "_" + case, json.dumps(rows[name + "_" + case]), flush=True)
        del r


def part_a(L, snap, units, reps, rows):
    D, step = 16 * MIB, 104729
    text = device_text(D + units * step)
    cap = L.sb_max_compress_len(D)
    slots = torch.empty(units * cap, dtype=torch.uint8, device="cuda")
    lens = torch.zeros(units, dtype=torch.int32, device="cuda")
    sts = torch.zeros(32 * units, dtype=torch.uint8, device="cuda")
    b = snap._lib.SbBatch()
    b.in_base, b.in_stride, b.in_len_uniform = text.data_ptr(), step, D
    b.out_base, b.out_stride, b.out_cap_uniform = slots.data_ptr(), cap, cap
    b.out_lens, b.statuses, b.count = lens.data_ptr(), sts.data_ptr(), units
    need = L.sb_compress_batch_scratch_bytes(units, units * D)
    scr = torch.empty(need, dtype=torch.uint8, device="cuda")
    e = snap._lib.SbError()
    check(L.sb_compress_batch_device_ws(C.byref(b), units * D, scr.data_ptr(), need, cuda_stream(), C.byref(e)), e)
    torch.cuda.synchronize()
    assert bool((sts == 0).all())
    del scr
    bt = Batch(L, snap, [slots.data_ptr() + u * cap for u in range(units)], lens.cpu().tolist(), [D] * units)
    rng = random.Random(1)
    cases = {"4096x4KiB": [(rng.randrange(units), rng.randrange(D - 4 * KIB), 4 * KIB) for _ in range(4096)]}
    print("(a) %d units of 16 MiB, %.2f GB compressed" % (units, bt.in_bytes / 1e9), flush=True)
    run_batch("a", L, snap, bt, cases, reps, rows)
    # the text every unit came from, against the full decode
    assert all(torch.equal(bt.want(u, 0, D), text[u * step:u * step + D]) for u in (0, units // 2, units - 1))
    del bt, slots, text
    torch.cuda.empty_cache()


def part_b(L, snap, reps, rows):
    D = 4 * GIB - BLOCK
    text = device_text(D)
    s = device_stream(snap, text)
    del text
    torch.cuda.empty_cache()
    bt = Batch(L, snap, [s.data_ptr()], [s.numel()], [D])
    rng = random.Random(2)
    cases = {"one_1GiB": [(0, GIB + 12345, GIB)],
             "1024x1MiB": [(0, rng.randrange(D - MIB), MIB) for _ in range(1024)],
             "1024x4KiB": [(0, rng.randrange(D - 4 * KIB), 4 * KIB) for _ in range(1024)]}
    print("(b) one unit of %d bytes, %.2f GB compressed" % (D, s.numel() / 1e9), flush=True)
    run_batch("b", L, snap, bt, cases, reps, rows)
    del bt, s
    torch.cuda.empty_cache()


def part_c(L, snap, reps, rows):
    try:
        import pyarrow as pa
    except ImportError:
        print("(c) skipped: pyarrow is not installed", flush=True)
        return
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    from raw_batch_decode_bench import text
    count = 1024
    data = text(count * MIB + 104729 * count)
    pages = [data[i * MIB + 104729 * i:(i + 1) * MIB + 104729 * i] for i in range(count)]
    streams = [np.frombuffer(pa.compress(p.tobytes(), codec="snappy", asbytes=True), dtype=np.uint8) for p in pages]
    t_in = torch.from_numpy(np.concatenate(streams)).cuda()
    at = np.concatenate([[0], np.cumsum([s.size for s in streams][:-1])]).astype(np.int64)
    bt = Batch(L, snap, [t_in.data_ptr() + int(a) for a in at], [s.size for s in streams], [MIB] * count)
    rng = random.Random(3)
    cases = {"4096x4KiB": [(rng.randrange(count), rng.randrange(MIB - 4 * KIB), 4 * KIB) for _ in range(4096)]}
    print("(c) %d pyarrow pages of 1 MiB, %.2f GB compressed" % (count, bt.in_bytes / 1e9), flush=True)
    run_batch("c", L, snap, bt, cases, reps, rows)
    assert torch.equal(bt.want(7, 0, MIB).cpu(), torch.from_numpy(pages[7].copy()))
    del bt, t_in
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--units", type=int, default=1024, help="units of 16 MiB in (a)")
    ap.add_argument("--only", default="abc")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for raw_table_bench.json (default: print only)")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    snap = graft.load_package()
    L = snap._lib.lib()
    info = {"card": card(), "rows": {}}
    print("card:", info["card"], flush=True)
    if "a" in args.only:
        part_a(L, snap, args.units, args.reps, info["rows"])
    if "b" in args.only:
        part_b(L, snap, args.reps, info["rows"])
    if "c" in args.only:
        part_c(L, snap, args.reps, info["rows"])
    info["card_after"] = card()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "raw_table_bench.json"), "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
