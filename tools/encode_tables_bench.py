"""Seek tables written by the batch encoders, against building them after the fact.

Three timings per batch, run alternately, each the median of --reps calls after a warm-up:
  plain    the untabled encode (sb_compress_batch_device_ws / sb_frame_encode_batch_device_ws);
  tabled   the tabled encode (sb_compress_batch_tabled_device_ws / sb_frame_encode_batch_tabled_device_ws);
  build    the untabled encode followed by the batch table build over its output (sb_raw_table_build_batch_device_ws /
           sb_frame_table_build_batch_device_ws).
Batches: (a) --raw-units raw units of 16 MiB of corpus text; (b) --frame-units frame units of 1 MiB of corpus text.
Before timing, every output, out_len and status of the tabled call is compared with the untabled call's, and every table,
offset and result with the build's.

    python tools/encode_tables_bench.py [--raw-units 1024] [--frame-units 4096] [--only ab] [--reps 5] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from frame_range_decode_bench import MIB, card, check, device_text, graft  # noqa: E402
from frame_table_bench import alternating, cuda_stream  # noqa: E402

BLOCK = 65536


class Batch:
    """k units of n bytes each, views at distinct offsets into one text buffer; two output buffers (the untabled and
    the tabled call write one each), the tabled call's tables and the build's."""

    def __init__(self, L, snap, frame, k, n):
        self.L, self.snap, self.frame, self.k, self.n = L, snap, frame, k, n
        self.text = device_text(n + 4099 * k + 16)
        i64 = lambda v: torch.from_numpy(np.array(v, dtype=np.uint64).view(np.int64)).cuda()
        self.t_ip = i64([self.text.data_ptr() + 4099 * i for i in range(k)])
        self.cap = L.sb_frame_max_len(n) if frame else L.sb_max_compress_len(n)
        self.in_bytes = n * k if n > BLOCK else 0
        self.outs, self.t_ops, self.t_ols, self.t_sts = [], [], [], []
        for _ in range(2):
            out = torch.zeros(self.cap * k, dtype=torch.uint8, device="cuda")
            self.outs.append(out)
            self.t_ops.append(i64([out.data_ptr() + self.cap * i for i in range(k)]))
            self.t_ols.append(torch.zeros(k, dtype=torch.int32, device="cuda"))
            self.t_sts.append(torch.zeros(32 * k, dtype=torch.uint8, device="cuda"))
        self.need_plain = (L.sb_frame_encode_batch_scratch_bytes if frame else L.sb_compress_batch_scratch_bytes)(
            k, self.in_bytes)
        self.need = (L.sb_frame_encode_batch_tabled_scratch_bytes if frame else L.sb_compress_batch_tabled_scratch_bytes)(
            k, self.in_bytes)
        self.tb = (L.sb_frame_encode_tables_bytes if frame else L.sb_compress_tables_bytes)(k, self.in_bytes)
        self.t_scr = torch.empty(max(self.need, self.need_plain), dtype=torch.uint8, device="cuda")
        self.t_tab = torch.zeros(self.tb, dtype=torch.uint8, device="cuda")
        self.t_res = torch.zeros(8 * (k + 1) + 48 * k, dtype=torch.uint8, device="cuda")
        # the build over the untabled call's output: its compressed bound is that output's total, its chunk table
        # (frame) holds every encoder chunk
        self.plain()
        self.b_in = int(self.t_ols[0].to(torch.int64).sum())
        self.mc = k * ((n + BLOCK - 1) // BLOCK + 1)
        if frame:
            self.btb = L.sb_frame_table_batch_bytes(k, self.mc)
            self.bneed = L.sb_frame_table_build_batch_scratch_bytes(k, self.b_in, self.mc)
        else:
            self.btb = L.sb_raw_table_batch_bytes(k, self.b_in)
            self.bneed = L.sb_raw_table_build_batch_scratch_bytes(k, self.b_in)
        self.b_tab = torch.zeros(self.btb, dtype=torch.uint8, device="cuda")
        self.b_res = torch.zeros(8 * (k + 1) + 48 * k, dtype=torch.uint8, device="cuda")
        self.b_scr = torch.empty(self.bneed, dtype=torch.uint8, device="cuda")

    def batch(self, j):
        b = self.snap._lib.SbBatch()
        b.in_ptrs, b.in_len_uniform, b.count = self.t_ip.data_ptr(), self.n, self.k
        b.out_ptrs, b.out_cap_uniform = self.t_ops[j].data_ptr(), self.cap
        b.out_lens, b.statuses = self.t_ols[j].data_ptr(), self.t_sts[j].data_ptr()
        return b

    def plain(self):
        e, L = self.snap._lib.SbError(), self.L
        f = L.sb_frame_encode_batch_device_ws if self.frame else L.sb_compress_batch_device_ws
        args = (None,) if self.frame else ()
        check(f(C.byref(self.batch(0)), self.in_bytes, *args, self.t_scr.data_ptr(), self.need_plain, cuda_stream(),
                C.byref(e)), e)

    def tabled(self):
        e, L, k = self.snap._lib.SbError(), self.L, self.k
        f = L.sb_frame_encode_batch_tabled_device_ws if self.frame else L.sb_compress_batch_tabled_device_ws
        args = (None,) if self.frame else ()
        p = self.t_res.data_ptr()
        check(f(C.byref(self.batch(1)), self.in_bytes, *args, self.t_tab.data_ptr(), self.tb, p, p + 8 * (k + 1),
                self.t_scr.data_ptr(), self.need, cuda_stream(), C.byref(e)), e)

    def build(self):
        e, L, k = self.snap._lib.SbError(), self.L, self.k
        b = self.snap._lib.SbBatch()
        b.in_ptrs, b.in_lens, b.count = self.t_ops[0].data_ptr(), self.t_ols[0].data_ptr(), k
        p = self.b_res.data_ptr()
        if self.frame:
            rc = L.sb_frame_table_build_batch_device_ws(C.byref(b), self.b_in, 0, None, None, self.mc, self.b_tab.data_ptr(),
                                                        self.btb, p, p + 8 * (k + 1), self.b_scr.data_ptr(), self.bneed,
                                                        cuda_stream(), C.byref(e))
        else:
            rc = L.sb_raw_table_build_batch_device_ws(C.byref(b), self.b_in, self.b_tab.data_ptr(), self.btb, p,
                                                      p + 8 * (k + 1), self.b_scr.data_ptr(), self.bneed, cuda_stream(),
                                                      C.byref(e))
        check(rc, e)

    def plain_then_build(self):
        self.plain()
        self.build()

    def verify(self):
        """Outputs, lengths and statuses of both calls equal; every table, offset and result equals the build's."""
        self.plain()
        self.tabled()
        self.build()
        torch.cuda.synchronize()
        k = self.k
        assert torch.equal(self.outs[0], self.outs[1]), "outputs differ"
        assert torch.equal(self.t_ols[0], self.t_ols[1]) and torch.equal(self.t_sts[0], self.t_sts[1])
        assert bool((self.t_sts[0].view(torch.int64)[0::4] == 0).all()), "a unit failed"
        offs = self.t_res[:8 * (k + 1)].cpu().numpy().view(np.uint64)
        assert torch.equal(self.t_res, self.b_res), "offsets or results differ from the build"
        end = int(offs[k])
        assert torch.equal(self.t_tab[:end], self.b_tab[:end]), "tables differ from the build"
        if not self.frame:
            heads = self.t_tab[:end].cpu().numpy()
            seek = [heads[int(offs[i]) + 32] for i in range(k)]
            assert all(s == 1 for s in seek), "a stream is not seekable"
        return end, int(self.t_ols[0].to(torch.int64).sum())


def part(L, snap, name, frame, k, n, reps, rows):
    bt = Batch(L, snap, frame, k, n)
    tables, comp = bt.verify()
    t_plain, t_tabled, t_build = alternating([bt.plain, bt.tabled, bt.plain_then_build], reps)
    bt.verify()
    row = {"units": k, "unit_bytes": n, "compressed_bytes": comp, "table_bytes": tables,
           "plain_ms": t_plain * 1e3, "tabled_ms": t_tabled * 1e3, "plain_then_build_ms": t_build * 1e3,
           "tabled_over_plain": t_tabled / t_plain, "build_over_plain": t_build / t_plain}
    rows[name] = row
    print(name, json.dumps(row), flush=True)
    del bt
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--raw-units", type=int, default=1024, help="raw units of 16 MiB in (a)")
    ap.add_argument("--frame-units", type=int, default=4096, help="frame units of 1 MiB in (b)")
    ap.add_argument("--only", default="ab")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for encode_tables_bench.json (default: print only)")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    snap = graft.load_package()
    L = snap._lib.lib()
    info = {"card": card(), "rows": {}}
    print("card:", info["card"], flush=True)
    if "a" in args.only:
        part(L, snap, "raw_16mib", False, args.raw_units, 16 * MIB, args.reps, info["rows"])
    if "b" in args.only:
        part(L, snap, "frame_1mib", True, args.frame_units, MIB, args.reps, info["rows"])
    info["card_after"] = card()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "encode_tables_bench.json"), "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
