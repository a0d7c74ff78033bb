"""Frame decode of device-resident batches: sb_frame_decode_batch_device_ws (every unit's chunk index built by K7 or
checked against the encoder's, every unit's chunks decoded in one grid) against a loop of sb_frame_decode_device_ws, one
call per unit, and against sb_decompress_batch_device_ws over the same data as raw streams (the ceiling: no chunk
index, no CRC).

The streams are made on the device by sb_frame_encode_batch_device_ws (and its chunk index), the raw streams by
sb_compress_batch_device_ws. The variants are alternated in one process; each is timed by CUDA events, median of --reps
calls after a warm-up. Every output is compared with the input after the warm-up and again after the timed calls. The
per-unit loop takes several launches per call, so it runs over the first --loop-units units only and its time is
scaled by count / loop units. Workloads:
  a  4,096 x 1 MiB units of corpus text, without and with the encoder's index
  b  131,072 x 64 KB units, one chunk each (per-call overhead dominates a loop)
  c  4,096 x 1 MiB units with a skippable chunk appended to every 16th unit (K7 declines those: they are walked)

    python tools/frame_batch_decode_bench.py [--only abc] [--reps N] [--loop-units N] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys

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
    """count units of `size` bytes of text, frame-encoded by K10 at a stride of sb_frame_max_len(size); `skip`: every
    16th stream gets an 8-byte skippable chunk appended."""

    def __init__(self, snap, count, size, loop_units, skip=False):
        self.snap, self.L = snap, snap._lib.lib()
        L, e = self.L, snap._lib.SbError()
        self.count, self.size = count, size
        self.nloop = min(count, loop_units)
        self.t_data = device_text(count * size)
        self.fcap = 10 + chunks(size) * (8 + 76490)
        self.nk = chunks(size) + 1
        self.t_frames = torch.zeros(count * self.fcap, dtype=torch.uint8, device="cuda")
        self.t_flens = torch.zeros(count, dtype=torch.int32, device="cuda")
        self.t_idx = torch.zeros(count * self.nk, dtype=torch.int64, device="cuda")
        self.t_at = torch.arange(0, count * self.nk + 1, self.nk, dtype=torch.int64, device="cuda")
        b = snap._lib.SbBatch()
        b.in_base, b.in_stride, b.in_len_uniform = self.t_data.data_ptr(), size, size
        b.out_base, b.out_stride, b.out_cap_uniform = self.t_frames.data_ptr(), self.fcap, self.fcap
        b.out_lens, b.count = self.t_flens.data_ptr(), count
        in_bytes = count * size if size > BLOCK else 0
        esb = L.sb_frame_encode_batch_scratch_bytes(count, in_bytes)
        t = torch.empty(esb, dtype=torch.uint8, device="cuda")
        assert L.sb_frame_encode_batch_device_ws(C.byref(b), in_bytes, self.t_idx.data_ptr(), t.data_ptr(), esb, stream(),
                                                 C.byref(e)) == 0
        torch.cuda.synchronize()
        del t
        if skip:
            sel = torch.arange(0, count, 16, device="cuda")
            at = sel * self.fcap + self.t_flens[sel].to(torch.int64)
            for k, v in enumerate((0x80, 4, 0, 0, 0, 0, 0, 0)):
                self.t_frames[at + k] = v
            self.t_flens[sel] += 8
        self.in_bytes = int(self.t_flens.to(torch.int64).sum())
        self.max_chunks = count * (self.nk - 1)
        # the batch decode
        self.t_dec = torch.zeros(count * size, dtype=torch.uint8, device="cuda")
        self.t_ol = torch.zeros(count, dtype=torch.int32, device="cuda")
        self.t_st = torch.zeros(count * 32, dtype=torch.uint8, device="cuda")
        self.t_uc = torch.zeros(count, dtype=torch.int32, device="cuda")
        d = snap._lib.SbBatch()
        d.in_base, d.in_stride, d.in_lens = self.t_frames.data_ptr(), self.fcap, self.t_flens.data_ptr()
        d.out_base, d.out_stride, d.out_cap_uniform = self.t_dec.data_ptr(), size, size
        d.out_lens, d.statuses, d.count = self.t_ol.data_ptr(), self.t_st.data_ptr(), count
        self.d = d
        self.sb = L.sb_frame_decode_batch_scratch_bytes(count, self.in_bytes, self.max_chunks)
        self.t_scr = torch.empty(self.sb, dtype=torch.uint8, device="cuda")
        # the per-unit loop
        self.t_ldec = torch.zeros(self.nloop * size, dtype=torch.uint8, device="cuda")
        self.usb = L.sb_frame_decode_scratch_bytes(self.nk + 1)
        self.t_uscr = torch.empty(self.usb, dtype=torch.uint8, device="cuda")
        self.t_res = torch.zeros(self.nloop * 48, dtype=torch.uint8, device="cuda")
        self.flens = self.t_flens.cpu().tolist()
        # the same units as raw streams (K9) for sb_decompress_batch_device_ws
        self.rcap = 32 + size + size // 6
        self.t_raw = torch.empty(count * self.rcap, dtype=torch.uint8, device="cuda")
        self.t_rol = torch.zeros(count, dtype=torch.int32, device="cuda")
        r = snap._lib.SbBatch()
        r.in_base, r.in_stride, r.in_len_uniform = self.t_data.data_ptr(), size, size
        r.out_base, r.out_stride, r.out_cap_uniform = self.t_raw.data_ptr(), self.rcap, self.rcap
        r.out_lens, r.count = self.t_rol.data_ptr(), count
        csb = L.sb_compress_batch_scratch_bytes(count, in_bytes)
        t = torch.empty(csb, dtype=torch.uint8, device="cuda")
        assert L.sb_compress_batch_device_ws(C.byref(r), in_bytes, t.data_ptr(), csb, stream(), C.byref(e)) == 0
        torch.cuda.synchronize()
        del t
        self.raw_bytes = int(self.t_rol.to(torch.int64).sum())
        self.t_rdec = torch.zeros(count * size, dtype=torch.uint8, device="cuda")
        self.t_rdol = torch.zeros(count, dtype=torch.int32, device="cuda")
        self.t_rst = torch.zeros(count * 32, dtype=torch.uint8, device="cuda")
        rd = snap._lib.SbBatch()
        rd.in_base, rd.in_stride, rd.in_lens = self.t_raw.data_ptr(), self.rcap, self.t_rol.data_ptr()
        rd.out_base, rd.out_stride, rd.out_cap_uniform = self.t_rdec.data_ptr(), size, size
        rd.out_lens, rd.statuses, rd.count = self.t_rdol.data_ptr(), self.t_rst.data_ptr(), count
        self.rd = rd
        self.rsb = L.sb_decompress_batch_scratch_bytes(count, self.raw_bytes)
        self.t_rscr = torch.empty(self.rsb, dtype=torch.uint8, device="cuda")

    def batch(self, index=False):
        e = self.snap._lib.SbError()
        assert self.L.sb_frame_decode_batch_device_ws(
            C.byref(self.d), self.in_bytes, 0, self.t_idx.data_ptr() if index else None, self.t_at.data_ptr() if index else None,
            self.max_chunks, self.t_uc.data_ptr(), self.t_scr.data_ptr(), self.sb, stream(), C.byref(e)) == 0

    def batch_index(self):
        self.batch(True)

    def loop(self):
        e = self.snap._lib.SbError()
        f, st = self.L.sb_frame_decode_device_ws, stream()
        fr, o, res, s = self.t_frames.data_ptr(), self.t_ldec.data_ptr(), self.t_res.data_ptr(), self.t_uscr.data_ptr()
        for i in range(self.nloop):
            assert f(fr + i * self.fcap, self.flens[i], o + i * self.size, self.size, None, 0, 0, res + 48 * i, s, self.usb,
                     self.nk + 1, st, C.byref(e)) == 0

    def raw(self):
        e = self.snap._lib.SbError()
        assert self.L.sb_decompress_batch_device_ws(C.byref(self.rd), self.raw_bytes, None, self.t_rscr.data_ptr(), self.rsb,
                                                    stream(), C.byref(e)) == 0

    def check(self, skip):
        torch.cuda.synchronize()
        assert bool((self.t_st == 0).all()) and bool((self.t_ol == self.size).all()), "a unit failed"
        assert torch.equal(self.t_dec, self.t_data), "batch output differs from the input"
        walked = int((self.t_uc == 0).sum())
        assert walked == (len(range(0, self.count, 16)) if skip else 0), walked
        assert bool((self.t_res.view(self.nloop, 48)[:, :4] == 0).all()), "a loop decode failed"
        assert torch.equal(self.t_ldec, self.t_data[:self.nloop * self.size]), "loop output differs from the input"
        assert bool((self.t_rst == 0).all()) and torch.equal(self.t_rdec, self.t_data), "raw batch output differs"
        self.t_dec.zero_()
        return walked


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="abc")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--loop-units", type=int, default=1024, help="units the per-unit loop decodes (default 1024)")
    ap.add_argument("--out", default=None, help="directory for frame_batch_decode_bench.json (default: print only)")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    snap = graft.load_package()
    info = {"card": card(), "torch": torch.__version__, "reps": args.reps, "workloads": {}}
    print("card:", info["card"], flush=True)
    shapes = {"a": (4096, MIB, False), "b": (131072, BLOCK, False), "c": (4096, MIB, True)}
    for name in args.only:
        count, size, skip = shapes[name]
        w = Work(snap, count, size, args.loop_units, skip)
        kinds = ["batch", "batch_index", "loop", "raw"] if name == "a" else ["batch", "loop", "raw"]
        w.loop()                                                       # warm-up, then check every output
        w.raw()
        for k in kinds[::-1]:
            if k.startswith("batch"):
                getattr(w, k)()
                walked = w.check(skip)
        print(name, "checked, timing", flush=True)
        total = w.count * w.size
        times = {k: [] for k in kinds}
        for _ in range(args.reps):
            for k in kinds:
                times[k].append(timed(getattr(w, k)) * (w.count / w.nloop if k == "loop" else 1))
            print(name, {k: round(v[-1], 3) for k, v in times.items()}, flush=True)
        for k in kinds:                                                # the timed calls' outputs too
            if k.startswith("batch"):
                getattr(w, k)()
                w.check(skip)
        row = {"units": w.count, "unit_bytes": w.size, "loop_units": w.nloop, "out_bytes": total, "frame_bytes": w.in_bytes,
               "raw_bytes": w.raw_bytes, "walked_units": walked}
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
        with open(os.path.join(args.out, "frame_batch_decode_bench.json"), "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
