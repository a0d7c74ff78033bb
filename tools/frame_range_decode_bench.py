"""Byte-range decode of one large frame stream: sb_frame_decode_ranges_device_ws (K5's index phase, then only the chunks
the ranges cover) against sb_frame_decode_device_ws of the whole stream.

The stream is one encoded fragment of corpus text (sb_frame_encode_device_ws) tiled on the device -- frame chunks are
independent -- to --gib GiB decoded, and indexed once by sb_frame_index_device_ws. Every range's bytes are first
compared with the full decode; then each variant is timed by CUDA events, median of --reps calls after a warm-up:
  1  one 1 GiB range
  2  1,024 ranges of 1 MiB at random offsets
  3  1,024 ranges of 4 KiB at random offsets (the staging-dominated case)
  4  sb_frame_decode_device_ws of the whole stream
--window GIB instead walks a tiled stream of GIB GiB decoded -- more than the card holds -- in 1 GiB windows, checks
every window against the text and reports the walk's throughput.

    python tools/frame_range_decode_bench.py [--gib 16] [--reps 5] [--window GIB] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import random
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as graft  # noqa: E402

GIB, MIB, KIB = 1 << 30, 1 << 20, 1 << 10
UNIT = 256 * MIB                                   # decoded bytes of the tiled fragment
DATA = os.path.join(ROOT, "tests", "golden", "data")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def device_text(n):
    base = b""
    for f in ("alice29.txt", "lcet10.txt", "html_x_4", "kppkn.gtb", "urls.10K"):
        with open(os.path.join(DATA, f), "rb") as fh:
            base += fh.read()
    t = torch.frombuffer(bytearray(base), dtype=torch.uint8).cuda()
    return t.repeat(n // t.numel() + 1)[:n].contiguous()


def check(rc, e):
    if rc:
        raise RuntimeError("snapb200 call failed: code %d (%d, %d, %d)" % (e.code, e.a, e.b, e.c))


class Stream:
    """The text's fragment tiled `reps` times on the device, and its K7 index."""

    def __init__(self, L, snap, text, reps):
        st = torch.cuda.current_stream().cuda_stream
        e = snap._lib.SbError()
        cap = L.sb_frame_max_len(UNIT)
        out = torch.empty(cap, dtype=torch.uint8, device="cuda")
        res = torch.zeros(64, dtype=torch.uint8, device="cuda")
        need = L.sb_frame_encode_scratch_bytes(UNIT)
        scr = torch.empty(need, dtype=torch.uint8, device="cuda")
        check(L.sb_frame_encode_device_ws(text.data_ptr(), UNIT, out.data_ptr(), cap, 0, None, res.data_ptr(), scr.data_ptr(),
                                          need, st, C.byref(e)), e)
        flen = int(res[32:40].cpu().view(torch.int64)[0])
        self.frag_len, self.reps = flen, reps
        self.t = out[:flen].repeat(reps)
        del out, scr
        self.n, self.total = flen * reps, UNIT * reps
        self.max_chunks = (UNIT // 65536) * reps + 1
        self.idx = torch.empty(self.max_chunks + 1, dtype=torch.int64, device="cuda")
        cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
        need = L.sb_frame_index_scratch_bytes(self.n, self.max_chunks)
        scr = torch.empty(need, dtype=torch.uint8, device="cuda")
        check(L.sb_frame_index_device_ws(self.t.data_ptr(), self.n, 1, self.idx.data_ptr(), self.max_chunks, cnt.data_ptr(),
                                         scr.data_ptr(), need, st, C.byref(e)), e)
        self.nchunks = int(cnt.cpu()[0])
        assert self.nchunks == self.max_chunks - 1, self.nchunks


class Ranges:
    """Device descriptors, buffers and scratch of one range call, allocated once."""

    def __init__(self, L, snap, s, ranges):
        self.L, self.snap, self.s, self.ranges = L, snap, s, ranges
        k = len(ranges)
        self.out = torch.empty(sum(n for _, n in ranges) + 1, dtype=torch.uint8, device="cuda")
        offs, at = [], 0
        for _, n in ranges:
            offs.append(at)
            at += n
        self.offs = offs
        self.desc = torch.tensor([lo for lo, _ in ranges] + [n for _, n in ranges] + [self.out.data_ptr() + o for o in offs],
                                 dtype=torch.int64, device="cuda")
        self.res = torch.zeros(5 * k + 6, dtype=torch.int64, device="cuda")
        self.need = L.sb_frame_decode_ranges_scratch_bytes(s.max_chunks, k)
        self.scr = torch.empty(self.need, dtype=torch.uint8, device="cuda")

    def __call__(self):
        k, p, e = len(self.ranges), self.desc.data_ptr(), self.snap._lib.SbError()
        check(self.L.sb_frame_decode_ranges_device_ws(self.s.t.data_ptr(), self.s.n, self.s.idx.data_ptr(), self.s.nchunks, 1,
                                                      p, p + 8 * k, p + 16 * k, self.res.data_ptr(), self.res.data_ptr() + 8 * k,
                                                      k, self.res.data_ptr() + 40 * k, self.scr.data_ptr(), self.need,
                                                      self.s.max_chunks, torch.cuda.current_stream().cuda_stream,
                                                      C.byref(e)), e)

    def verify(self, full):
        back, k = self.res.cpu(), len(self.ranges)
        assert (back[k:5 * k].view(-1, 4)[:, 0] & 0xFFFFFFFF).eq(0).all(), "a range failed"
        for (lo, n), o, m in zip(self.ranges, self.offs, back[:k].tolist()):
            assert m == n and torch.equal(self.out[o:o + n], full[lo:lo + n]), (lo, n)


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b) / 1e3)
    return statistics.median(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=int, default=16, help="decoded GiB of the benchmark stream")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--window", type=int, default=0, help="walk a stream of this many decoded GiB in 1 GiB windows")
    ap.add_argument("--out", default=None, help="directory for frame_range_decode_bench.json (default: print only)")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    snap = graft.load_package()
    L = snap._lib.lib()
    info = {"card": card(), "rows": {}}
    print("card:", info["card"], flush=True)
    text = device_text(UNIT)
    if args.window:
        s = Stream(L, snap, text, args.window * GIB // UNIT)
        free, tot = torch.cuda.mem_get_info()
        print("window walk: %d GiB decoded from %.1f GB compressed; device memory %.1f GB" %
              (s.total // GIB, s.n / 1e9, tot / 1e9), flush=True)
        win = Ranges(L, snap, s, [(0, GIB)])
        want = text.repeat(GIB // UNIT)
        desc_lo = win.desc[0:1]
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for w in range(s.total // GIB):
            desc_lo.fill_(w * GIB)
            win()
            assert int(win.res[1]) & 0xFFFFFFFF == 0 and int(win.res[0]) == GIB, w
            assert torch.equal(win.out[:GIB], want), w
        b.record()
        b.synchronize()
        sec = a.elapsed_time(b) / 1e3
        row = {"decoded_gib": s.total // GIB, "compressed_bytes": s.n, "device_bytes": tot, "seconds_with_checks": sec,
               "gb_per_s_with_checks": s.total / sec / 1e9}
        info["rows"]["window"] = row
        print("window", json.dumps(row), flush=True)
    else:
        s = Stream(L, snap, text, args.gib * GIB // UNIT)
        full = torch.empty(s.total, dtype=torch.uint8, device="cuda")
        fres = torch.zeros(64, dtype=torch.uint8, device="cuda")
        fneed = L.sb_frame_decode_scratch_bytes(s.max_chunks)
        fscr = torch.empty(fneed, dtype=torch.uint8, device="cuda")
        e = snap._lib.SbError()

        def full_decode():
            check(L.sb_frame_decode_device_ws(s.t.data_ptr(), s.n, full.data_ptr(), s.total, s.idx.data_ptr(), s.nchunks, 1,
                                              fres.data_ptr(), fscr.data_ptr(), fneed, s.max_chunks,
                                              torch.cuda.current_stream().cuda_stream, C.byref(e)), e)
        full_decode()
        torch.cuda.synchronize()
        assert int(fres[:4].cpu().view(torch.int32)[0]) == 0 and int(fres[32:40].cpu().view(torch.int64)[0]) == s.total
        for t in range(s.total // UNIT):
            assert torch.equal(full[t * UNIT:(t + 1) * UNIT], text), t
        rng = random.Random(1)
        cases = {
            "one_1GiB": [(5 * GIB + 12345, GIB)],
            "1024x1MiB": [(rng.randrange(s.total - MIB), MIB) for _ in range(1024)],
            "1024x4KiB": [(rng.randrange(s.total - 4 * KIB), 4 * KIB) for _ in range(1024)],
        }
        print("stream: %d GiB decoded, %.2f GB compressed, %d chunks, indexed" % (s.total // GIB, s.n / 1e9, s.nchunks),
              flush=True)
        for name, ranges in cases.items():
            r = Ranges(L, snap, s, ranges)
            r()
            torch.cuda.synchronize()
            r.verify(full)
            sec = timed(r, args.reps)
            r.verify(full)
            nbytes = sum(n for _, n in ranges)
            row = {"ranges": len(ranges), "bytes": nbytes, "scratch_bytes": r.need, "seconds": sec,
                   "gb_per_s": nbytes / sec / 1e9}
            info["rows"][name] = row
            print(name, json.dumps(row), flush=True)
            del r
        sec = timed(full_decode, args.reps)
        row = {"bytes": s.total, "seconds": sec, "gb_per_s": s.total / sec / 1e9}
        info["rows"]["full_decode"] = row
        print("full_decode", json.dumps(row), flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "frame_range_decode_bench.json"), "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
