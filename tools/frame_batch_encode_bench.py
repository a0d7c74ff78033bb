"""Frame encode of device-resident batches: sb_frame_encode_batch_device_ws (every unit's chunks in one K1 launch, each
unit a complete framed stream) against a loop of sb_frame_encode_device_ws, one call per unit, and against
sb_compress_batch_device_ws (K9, raw streams of the same units: the ceiling, since frames only add the chunk CRC in
K1's emitter and 8 header bytes per chunk).

The three are alternated in one process; each is timed by CUDA events, median of --reps calls after a warm-up. Every
batch output is compared with the per-unit loop's bytes and chunk index on the device, and every stream is decoded by
sb_frame_decode_device_ws with the batch's index and compared with its input. The per-unit loop takes about a
millisecond per call, so it runs over the first --loop-units units only; its time for the whole batch is that time
scaled by count / loop units (exact for a and b, an extrapolation for c), and only those units are compared with it.
Workloads:
  a  4,096 x 1 MiB units of corpus text
  b  256 x 16 MiB units
  c  131,072 x 64 KB units

    python tools/frame_batch_encode_bench.py [--only abc] [--reps N] [--loop-units N] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as graft  # noqa: E402

BLOCK = 65536
MIB = 1 << 20
DATA = os.path.join(ROOT, "tests", "golden", "data")


def corpus(name):
    with open(os.path.join(DATA, name), "rb") as f:
        return f.read()


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def device_text(n):
    base = b"".join(corpus(f) for f in ("alice29.txt", "lcet10.txt", "html_x_4", "kppkn.gtb", "urls.10K"))
    t = torch.frombuffer(bytearray(base), dtype=torch.uint8).cuda()
    return t.repeat(n // t.numel() + 1)[:n].contiguous()


def chunks(n):
    return (n + BLOCK - 1) // BLOCK


def frame_max_len(n):
    return 10 + chunks(n) * (8 + 76490)


def stream():
    return torch.cuda.current_stream().cuda_stream


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


class Work:
    """count units of `size` bytes back to back in t_data; frame outputs of sb_frame_max_len(size) each for the batch
    and for the loop, raw outputs of max_compress_len(size) for K9."""

    def __init__(self, snap, count, size, loop_units):
        self.snap, self.L = snap, snap._lib.lib()
        self.count, self.size = count, size
        self.nloop = min(count, loop_units)
        self.t_data = device_text(count * size)
        self.cap = frame_max_len(size)
        self.nk = chunks(size) + 1
        self.t_out = torch.zeros(count * self.cap, dtype=torch.uint8, device="cuda")
        self.t_loop = torch.zeros(self.nloop * self.cap, dtype=torch.uint8, device="cuda")
        self.t_idx = torch.zeros(count * self.nk, dtype=torch.int64, device="cuda")
        self.t_lidx = torch.zeros(self.nloop * self.nk, dtype=torch.int64, device="cuda")
        self.t_ol = torch.zeros(count, dtype=torch.int32, device="cuda")
        self.t_st = torch.zeros(count * 32, dtype=torch.uint8, device="cuda")
        self.in_bytes = count * size if size > BLOCK else 0
        b = snap._lib.SbBatch()
        b.in_base, b.in_stride, b.in_len_uniform = self.t_data.data_ptr(), size, size
        b.out_base, b.out_stride, b.out_cap_uniform = self.t_out.data_ptr(), self.cap, self.cap
        b.out_lens, b.statuses, b.count = self.t_ol.data_ptr(), self.t_st.data_ptr(), count
        self.b = b
        self.sb = self.L.sb_frame_encode_batch_scratch_bytes(count, self.in_bytes)
        self.t_scr = torch.empty(self.sb, dtype=torch.uint8, device="cuda")
        self.usb = self.L.sb_frame_encode_scratch_bytes(size)
        self.t_uscr = torch.empty(self.usb, dtype=torch.uint8, device="cuda")
        self.t_res = torch.zeros(count * 64, dtype=torch.uint8, device="cuda")
        # K9 on the same units
        self.rcap = 32 + size + size // 6
        self.t_raw = torch.empty(count * self.rcap, dtype=torch.uint8, device="cuda")
        self.t_rol = torch.zeros(count, dtype=torch.int32, device="cuda")
        r = snap._lib.SbBatch()
        r.in_base, r.in_stride, r.in_len_uniform = self.t_data.data_ptr(), size, size
        r.out_base, r.out_stride, r.out_cap_uniform = self.t_raw.data_ptr(), self.rcap, self.rcap
        r.out_lens, r.count = self.t_rol.data_ptr(), count
        self.r = r
        self.rsb = self.L.sb_compress_batch_scratch_bytes(count, self.in_bytes)
        self.t_rscr = torch.empty(self.rsb, dtype=torch.uint8, device="cuda")

    def batch(self):
        e = self.snap._lib.SbError()
        assert self.L.sb_frame_encode_batch_device_ws(C.byref(self.b), self.in_bytes, self.t_idx.data_ptr(), self.t_scr.data_ptr(),
                                                      self.sb, stream(), C.byref(e)) == 0

    def loop(self):
        e = self.snap._lib.SbError()
        f, st = self.L.sb_frame_encode_device_ws, stream()
        d, o, x, res, s = self.t_data.data_ptr(), self.t_loop.data_ptr(), self.t_lidx.data_ptr(), self.t_res.data_ptr(), self.t_uscr.data_ptr()
        for i in range(self.nloop):
            assert f(d + i * self.size, self.size, o + i * self.cap, self.cap, 1, x + 8 * i * self.nk, res + 64 * i, s, self.usb,
                     st, C.byref(e)) == 0

    def k9(self):
        e = self.snap._lib.SbError()
        assert self.L.sb_compress_batch_device_ws(C.byref(self.r), self.in_bytes, self.t_rscr.data_ptr(), self.rsb, stream(),
                                                  C.byref(e)) == 0

    def check(self):
        """The batch equals the loop (bytes and index) and every stream decodes to its unit."""
        torch.cuda.synchronize()
        assert bool((self.t_st == 0).all()), "a unit failed"
        m, k = self.nloop * self.cap, self.nloop * self.nk
        assert torch.equal(self.t_out[:m], self.t_loop[:m]) and torch.equal(self.t_idx[:k], self.t_lidx[:k]), "batch differs from the loop"
        L, snap = self.L, self.snap
        ol = self.t_ol.cpu().numpy().astype(np.int64)
        assert np.array_equal(ol, self.t_idx.view(self.count, self.nk)[:, -1].cpu().numpy())
        t_dec = torch.zeros(self.count * self.size, dtype=torch.uint8, device="cuda")
        maxc = self.nk
        dsb = L.sb_frame_decode_scratch_bytes(maxc)
        t_dscr = torch.empty(dsb, dtype=torch.uint8, device="cuda")
        t_dres = torch.zeros(self.count * 64, dtype=torch.uint8, device="cuda")
        e = snap._lib.SbError()
        o, x, dd, dr, ds = self.t_out.data_ptr(), self.t_idx.data_ptr(), t_dec.data_ptr(), t_dres.data_ptr(), t_dscr.data_ptr()
        for i in range(self.count):
            assert L.sb_frame_decode_device_ws(o + i * self.cap, int(ol[i]), dd + i * self.size, self.size, x + 8 * i * self.nk,
                                               self.nk - 1, 0, dr + 64 * i, ds, dsb, maxc, stream(), C.byref(e)) == 0
        torch.cuda.synchronize()
        assert bool((t_dres.view(self.count, 64)[:, :4] == 0).all()), "a decode failed"
        assert torch.equal(t_dec, self.t_data), "decoded bytes differ from the input"
        return int(ol.sum())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="abc")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--loop-units", type=int, default=4096, help="units the per-unit loop encodes (default 4096)")
    ap.add_argument("--out", default=None, help="directory for frame_batch_encode_bench.json (default: print only)")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    snap = graft.load_package()
    info = {"card": card(), "torch": torch.__version__, "reps": args.reps, "workloads": {}}
    print("card:", info["card"], flush=True)
    shapes = {"a": (4096, MIB), "b": (256, 16 * MIB), "c": (131072, BLOCK)}
    for name in args.only:
        w = Work(snap, *shapes[name], args.loop_units)
        w.batch()
        w.loop()
        w.k9()
        out_bytes = w.check()
        print(name, "checked, timing", flush=True)
        total = w.count * w.size
        times = {"batch": [], "loop": [], "k9": []}
        for _ in range(args.reps):
            for k in ("batch", "loop", "k9"):
                times[k].append(timed(getattr(w, k)) * (w.count / w.nloop if k == "loop" else 1))
            print(name, {k: round(v[-1], 3) for k, v in times.items()}, flush=True)
        w.check()
        row = {"units": w.count, "unit_bytes": w.size, "loop_units": w.nloop, "in_bytes": total, "frame_bytes": out_bytes,
               "raw_bytes": int(w.t_rol.to(torch.int64).sum())}
        for k, v in times.items():
            row[k + "_ms"] = round(statistics.median(v), 3)
            row[k + "_spread_ms"] = [round(min(v), 3), round(max(v), 3)]
            row[k + "_gbps"] = round(total / row[k + "_ms"] / 1e6, 2)
        info["workloads"][name] = row
        print(name, json.dumps(row), flush=True)
        del w
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "frame_batch_encode_bench.json"), "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
