"""Validation against decoding on device-resident batches: sb_validate_batch_device_ws against
sb_decompress_batch_device_ws (raw) and sb_frame_validate_batch_device_ws against sb_frame_decode_batch_device_ws (frame),
on the same inputs, the two calls alternating after a warm-up, timed by CUDA events. Reports the median and the spread
(min, max) of each, and the device bytes each call needs: its scratch plus its outputs (decoded bytes, out_lens,
statuses, per-unit counts). Every run compares the two calls' statuses, out_lens and d_unit_blocks / d_unit_chunks; the
decode's output is compared with the input once. Workloads (corpus text, encoded on the device by this library):
  r64k   131,072 x 64 KiB raw units         r1m   4,096 x 1 MiB raw units        r4g   one raw stream of 4 GiB - 64 KiB
  f1m    4,096 x 1 MiB frame units, without the encoder's index        f1mi   the same with it
  f64k   131,072 x 64 KiB frame units, without the encoder's index     f64ki  the same with it

    python tools/validate_bench.py [--only r64k,r1m,...] [--reps N] [--warmup N] [--out DIR]
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
from raw_decode_bench import device_stream  # noqa: E402

BLOCK = 65536
MIB = 1 << 20
SLOT = 76544
DATA = os.path.join(ROOT, "tests", "golden", "data")
WORKLOADS = ("r64k", "r1m", "r4g", "f1m", "f1mi", "f64k", "f64ki")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def text_base():
    names = ("alice29.txt", "lcet10.txt", "html_x_4", "kppkn.gtb", "urls.10K", "plrabn12.txt")
    raw = b"".join(open(os.path.join(DATA, n), "rb").read() for n in names)
    return torch.frombuffer(bytearray(raw), dtype=torch.uint8).cuda()


def stream():
    return torch.cuda.current_stream().cuda_stream


def check_rc(rc, e, what):
    if rc:
        raise RuntimeError("%s failed: code %d a=%d b=%d" % (what, e.code, e.a, e.b))


def source(L, snap, base, count, size):
    """count units of `size` text bytes, back to back on the device (for one unit: the text tiled)."""
    if count == 1:
        return base.repeat(size // base.numel() + 1)[:size].contiguous()
    t = torch.empty(count * size, dtype=torch.uint8, device="cuda")
    e = snap._lib.SbError()
    check_rc(L.sb_generate_blocks_device(base.data_ptr(), base.numel(), t.data_ptr(), size, size, 0, count, 7919, stream(),
                                         C.byref(e)), e, "sb_generate_blocks_device")
    return t


def encode(L, snap, src, count, size, frame, index):
    """The units of src encoded by the batch encoder: (streams tensor, stride, lengths tensor, chunk index or None). A raw
    stream too large for the encoder's worst-case bound is assembled from its blocks compressed as independent units."""
    if not frame and count == 1 and L.sb_max_compress_len(size) == 0:
        out = device_stream(snap, src)
        return out, out.numel(), torch.tensor([out.numel()], dtype=torch.int32, device="cuda"), None
    stride = (L.sb_frame_max_len(size) if frame else L.sb_max_compress_len(size)) + 1 | 1
    out = torch.empty(count * stride + 16, dtype=torch.uint8, device="cuda")
    lens = torch.zeros(count, dtype=torch.int32, device="cuda")
    b = snap._lib.SbBatch()
    b.in_base, b.in_stride, b.in_len_uniform = src.data_ptr(), size, size
    b.out_base, b.out_stride, b.out_cap_uniform, b.out_lens, b.count = out.data_ptr(), stride, stride - 1, lens.data_ptr(), count
    e = snap._lib.SbError()
    big = size * count if size > BLOCK else 0
    idx = None
    if frame:
        per = (size + BLOCK - 1) // BLOCK
        idx = torch.empty(count * (per + 1) + 1, dtype=torch.int64, device="cuda") if index else None
        need = L.sb_frame_encode_batch_scratch_bytes(count, big)
        scr = torch.empty(need, dtype=torch.uint8, device="cuda")
        check_rc(L.sb_frame_encode_batch_device_ws(C.byref(b), big, idx.data_ptr() if index else None, scr.data_ptr(), need,
                                                   stream(), C.byref(e)), e, "frame encode")
    elif size <= BLOCK:
        check_rc(L.sb_compress_batch_device(C.byref(b), stream(), C.byref(e)), e, "compress")
    else:
        need = L.sb_compress_batch_scratch_bytes(count, big)
        scr = torch.empty(need, dtype=torch.uint8, device="cuda")
        check_rc(L.sb_compress_batch_device_ws(C.byref(b), big, scr.data_ptr(), need, stream(), C.byref(e)), e, "compress")
    torch.cuda.synchronize()
    return out, stride, lens, idx


class Pair:
    """One workload: the decode call and the validation call over the same device-resident units."""

    def __init__(self, snap, name, src, count, size):
        L = self.L = snap._lib.lib()
        self.snap, self.name, self.count, self.size = snap, name, count, size
        self.frame, index = name.startswith("f"), name.endswith("i")
        self.t_in, stride, self.t_len, self.idx = encode(L, snap, src, count, size, self.frame, index)
        self.in_bytes = int(self.t_len.to(torch.int64).sum())
        self.per = (size + BLOCK - 1) // BLOCK
        self.t_at = torch.arange(count + 1, dtype=torch.int64, device="cuda") * (self.per + 1) if index else None
        self.max_chunks = count * self.per if self.frame else 0
        self.t_out = torch.empty(count * size + 16, dtype=torch.uint8, device="cuda")
        self.t_res = [torch.zeros(count * 40 + 8, dtype=torch.uint8, device="cuda") for _ in range(2)]   # out_lens, statuses
        self.t_extra = [torch.zeros(count, dtype=torch.int32, device="cuda") for _ in range(2)]
        if self.frame:
            self.sb = [L.sb_frame_decode_batch_scratch_bytes(count, self.in_bytes, self.max_chunks),
                       L.sb_frame_validate_batch_scratch_bytes(count, self.in_bytes, self.max_chunks)]
        else:
            self.sb = [L.sb_decompress_batch_scratch_bytes(count, self.in_bytes)] * 2
        self.t_scr = torch.empty(max(self.sb), dtype=torch.uint8, device="cuda")
        self.b = []
        for k in range(2):
            b = snap._lib.SbBatch()
            b.in_base, b.in_stride, b.in_lens = self.t_in.data_ptr(), stride, self.t_len.data_ptr()
            if k == 0:
                b.out_base, b.out_stride, b.out_cap_uniform = self.t_out.data_ptr(), size, size
            b.out_lens, b.statuses, b.count = self.t_res[k].data_ptr(), self.t_res[k].data_ptr() + 8 * count, count
            self.b.append(b)

    def call(self, k):
        """k = 0: the decode, 1: the validation."""
        L, e = self.L, self.snap._lib.SbError()
        args = (self.t_extra[k].data_ptr(), self.t_scr.data_ptr(), self.sb[k], stream(), C.byref(e))
        if self.frame:
            f = L.sb_frame_validate_batch_device_ws if k else L.sb_frame_decode_batch_device_ws
            rc = f(C.byref(self.b[k]), self.in_bytes, 0, self.idx.data_ptr() if self.idx is not None else None,
                   self.t_at.data_ptr() if self.t_at is not None else None, self.max_chunks, *args)
        else:
            f = L.sb_validate_batch_device_ws if k else L.sb_decompress_batch_device_ws
            rc = f(C.byref(self.b[k]), self.in_bytes, *args)
        check_rc(rc, e, self.name)

    def compare(self):
        torch.cuda.synchronize()
        r0, r1 = self.t_res
        assert torch.equal(r0, r1), "%s: statuses or out_lens differ" % self.name
        assert torch.equal(self.t_extra[0], self.t_extra[1]), "%s: per-unit counts differ" % self.name
        assert bool((r0[8 * self.count:40 * self.count].view(-1, 32)[:, :4] == 0).all()), "%s: a unit failed" % self.name
        assert bool((r0[:4 * self.count].view(torch.int32) == self.size).all())

    def device_bytes(self, k):
        results = self.count * (4 + 32 + 4)
        return self.sb[k] + results + (self.count * self.size if k == 0 else 0)


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def run(snap, name, base, reps, warmup):
    L = snap._lib.lib()
    count, size = {"r64k": (131072, BLOCK), "r1m": (4096, MIB), "r4g": (1, 4 * 1024 * MIB - BLOCK),
                   "f1m": (4096, MIB), "f1mi": (4096, MIB), "f64k": (131072, BLOCK), "f64ki": (131072, BLOCK)}[name]
    src = source(L, snap, base, count, size)
    p = Pair(snap, name, src, count, size)
    p.call(0)
    torch.cuda.synchronize()
    assert torch.equal(p.t_out[:count * size], src), "%s: decoded output differs from the input" % name
    del src
    for _ in range(warmup):
        p.call(0)
        p.call(1)
    p.compare()
    times = [[], []]
    for _ in range(reps):
        for k in (0, 1):
            times[k].append(timed(lambda: p.call(k)))
        p.compare()
    res = {"workload": name, "units": count, "unit_bytes": size, "compressed_bytes": p.in_bytes}
    for k, tag in ((0, "decode"), (1, "validate")):
        t = times[k]
        res[tag] = {"median_ms": statistics.median(t), "min_ms": min(t), "max_ms": max(t),
                    "gb_per_s": count * size / statistics.median(t) / 1e6, "device_bytes": p.device_bytes(k)}
    res["validate_over_decode"] = res["validate"]["median_ms"] / res["decode"]["median_ms"]
    del p
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default=",".join(WORKLOADS))
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "validate_bench.py needs the GPU"
    torch.cuda.set_device(0)
    graft.build_cuda()
    snap = graft.load_package()
    info = {"card": card()}
    print(json.dumps(info), flush=True)
    base = text_base()
    results = []
    for name in a.only.split(","):
        r = run(snap, name, base, a.reps, a.warmup)
        results.append(r)
        print(json.dumps(r), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "validate_bench.json"), "w") as f:
            json.dump({"info": info, "results": results}, f, indent=1)


if __name__ == "__main__":
    main()
