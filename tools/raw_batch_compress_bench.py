"""Raw compress of batches with units over 64 KB: sb_compress_batch_device_ws (every unit cut into its 64 KB blocks, all
blocks of the batch in one K1 launch, each unit assembled in its output) on device-resident batches.

Each workload is timed by CUDA events, median of --reps timed calls after a warm-up. Every output is decoded by
sb_decompress_batch_device_ws and compared with the input, and the first and last unit are compared with host
sb_compress. The ceiling is the same data as independent 64 KB units through sb_compress_batch_device (K1 alone).
Workloads:
  a  4,096 x 1 MiB units of corpus text
  b  256 x 16 MiB units
  c  131,072 x 64 KB units (nothing multi-block), against sb_compress_batch_device on the same batch, alternating
  d  one 256 MiB unit among 65,536 units of 64 KB
  e  one 1 GiB unit, against host sb_compress on the same data (host clock: it copies in, compresses, copies back)

    python tools/raw_batch_compress_bench.py [--only abcde] [--reps N] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import __graft_entry__ as graft  # noqa: E402

BLOCK = 65536
MIB = 1 << 20
SLOT = 76544
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


def max_compress_len(n):
    return 32 + n + n // 6


def host_compress(L, snap, arr):
    cap = L.sb_max_compress_len(arr.size)
    out = np.empty(cap, dtype=np.uint8)
    n, e = C.c_size_t(0), snap._lib.SbError()
    assert L.sb_compress(arr.ctypes.data, arr.size, out.ctypes.data, cap, C.byref(n), C.byref(e)) == 0
    return out[:n.value]


def stream():
    return torch.cuda.current_stream().cuda_stream


class Batch:
    """Units of t_data at offs with lengths lens; outputs of max_compress_len(len) back to back in one buffer."""

    def __init__(self, snap, t_data, offs, lens):
        self.snap, self.L, self.t_data = snap, snap._lib.lib(), t_data
        offs, lens = np.asarray(offs, dtype=np.int64), np.asarray(lens, dtype=np.int64)
        self.n, self.lens, self.offs = len(lens), lens, offs
        caps = max_compress_len(lens)
        self.ooffs = np.concatenate([[0], np.cumsum(caps)[:-1]])
        self.t_out = torch.empty(int(caps.sum()) + 16, dtype=torch.uint8, device="cuda")
        self.t_ip = torch.tensor(offs + t_data.data_ptr(), device="cuda")
        self.t_op = torch.tensor(self.ooffs + self.t_out.data_ptr(), device="cuda")
        self.t_len = torch.tensor(lens, dtype=torch.int32, device="cuda")
        self.t_cap = torch.tensor(caps, dtype=torch.int32, device="cuda")
        self.t_ol = torch.zeros(self.n, dtype=torch.int32, device="cuda")
        self.t_st = torch.zeros(self.n * 32, dtype=torch.uint8, device="cuda")
        self.in_bytes = int(lens[lens > BLOCK].sum())
        self.sb = self.L.sb_compress_batch_scratch_bytes(self.n, self.in_bytes)
        self.t_scr = torch.empty(self.sb, dtype=torch.uint8, device="cuda")
        b = snap._lib.SbBatch()
        b.in_ptrs, b.in_lens, b.out_ptrs, b.out_caps = self.t_ip.data_ptr(), self.t_len.data_ptr(), self.t_op.data_ptr(), self.t_cap.data_ptr()
        b.out_lens, b.statuses, b.count = self.t_ol.data_ptr(), self.t_st.data_ptr(), self.n
        self.b = b

    def ws(self):
        e = self.snap._lib.SbError()
        assert self.L.sb_compress_batch_device_ws(C.byref(self.b), self.in_bytes, self.t_scr.data_ptr(), self.sb, stream(),
                                                  C.byref(e)) == 0

    def k1_batch(self):
        e = self.snap._lib.SbError()
        assert self.L.sb_compress_batch_device(C.byref(self.b), stream(), C.byref(e)) == 0

    def check(self):
        """Decode every unit block-parallel and compare with the input; first and last unit against host sb_compress."""
        torch.cuda.synchronize()
        assert bool((self.t_st.view(-1, 32)[:, :4] == 0).all()), "a unit failed"
        ol = self.t_ol.cpu().numpy().astype(np.int64)
        L, snap = self.L, self.snap
        t_dec = torch.zeros(int(self.lens.sum()) + 16, dtype=torch.uint8, device="cuda")
        doffs = np.concatenate([[0], np.cumsum(self.lens)[:-1]])
        t_dp = torch.tensor(doffs + t_dec.data_ptr(), device="cuda")
        t_dl = torch.zeros(self.n, dtype=torch.int32, device="cuda")
        t_blk = torch.zeros(self.n, dtype=torch.int32, device="cuda")
        t_st = torch.zeros(self.n * 32, dtype=torch.uint8, device="cuda")
        b = snap._lib.SbBatch()
        b.in_ptrs, b.in_lens, b.out_ptrs, b.out_caps = self.t_op.data_ptr(), self.t_ol.data_ptr(), t_dp.data_ptr(), self.t_len.data_ptr()
        b.out_lens, b.statuses, b.count = t_dl.data_ptr(), t_st.data_ptr(), self.n
        sb = L.sb_decompress_batch_scratch_bytes(self.n, int(ol.sum()))
        t_scr = torch.empty(sb, dtype=torch.uint8, device="cuda")
        e = snap._lib.SbError()
        assert L.sb_decompress_batch_device_ws(C.byref(b), int(ol.sum()), t_blk.data_ptr(), t_scr.data_ptr(), sb, stream(),
                                               C.byref(e)) == 0
        torch.cuda.synchronize()
        assert bool((t_st == 0).all()) and torch.equal(t_dl.to(torch.int64), self.t_len.to(torch.int64))
        multi = self.lens > BLOCK
        assert np.array_equal(t_blk.cpu().numpy()[multi], (self.lens[multi] + BLOCK - 1) // BLOCK), "not block-parallel"
        assert np.array_equal(self.offs, doffs)                       # every workload's units lie back to back
        assert torch.equal(t_dec[:int(self.lens.sum())], self.t_data[:int(self.lens.sum())])
        for i in (0, self.n - 1):
            unit = self.t_data[self.offs[i]:self.offs[i] + self.lens[i]].cpu().numpy()
            assert torch.equal(t_dec[doffs[i]:doffs[i] + self.lens[i]].cpu(), torch.from_numpy(unit))
            got = self.t_out[self.ooffs[i]:self.ooffs[i] + ol[i]].cpu().numpy()
            assert np.array_equal(got, host_compress(L, snap, unit)), "differs from host sb_compress"
        return int(ol.sum())


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def ceiling_ms(snap, t_data, reps):
    """t_data as independent 64 KB units through sb_compress_batch_device."""
    L = snap._lib.lib()
    nb = t_data.numel() // BLOCK
    slots = torch.empty(nb * SLOT, dtype=torch.uint8, device="cuda")
    lens = torch.zeros(nb, dtype=torch.int32, device="cuda")
    b = snap._lib.SbBatch()
    b.in_base, b.in_stride, b.in_len_uniform = t_data.data_ptr(), BLOCK, BLOCK
    b.out_base, b.out_stride, b.out_cap_uniform, b.out_lens, b.count = slots.data_ptr(), SLOT, SLOT, lens.data_ptr(), nb
    e = snap._lib.SbError()
    run = lambda: L.sb_compress_batch_device(C.byref(b), stream(), C.byref(e))  # noqa: E731
    run()
    return statistics.median(timed(run) for _ in range(reps))


def workload(name, snap):
    if name in "ab":
        count, size = (4096, MIB) if name == "a" else (256, 16 * MIB)
        t_data = device_text(count * size)
        return Batch(snap, t_data, np.arange(count) * size, [size] * count)
    if name == "c":
        t_data = device_text(131072 * BLOCK)
        return Batch(snap, t_data, np.arange(131072) * BLOCK, [BLOCK] * 131072)
    if name == "d":
        t_data = device_text(256 * MIB + 65535 * BLOCK)
        at = 40000
        lens = [BLOCK] * at + [256 * MIB] + [BLOCK] * (65535 - at)
        return Batch(snap, t_data, np.concatenate([[0], np.cumsum(lens)[:-1]]), lens)
    t_data = device_text(1 << 30)
    return Batch(snap, t_data, [0], [1 << 30])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="abcde")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for raw_batch_compress_bench.json (default: print only)")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    snap = graft.load_package()
    L = snap._lib.lib()
    info = {"card": card(), "torch": torch.__version__, "reps": args.reps, "workloads": {}}
    print("card:", info["card"], flush=True)
    for name in args.only:
        bt = workload(name, snap)
        bt.ws()
        out_bytes = bt.check()
        total = int(bt.lens.sum())
        row = {"units": bt.n, "in_bytes": total, "out_bytes": out_bytes}
        new, old = [], []
        for _ in range(args.reps):
            new.append(timed(bt.ws))
            if name == "c":
                old.append(timed(bt.k1_batch))
        bt.check()                                                    # (c): the last call was sb_compress_batch_device
        row["ws_ms"] = round(statistics.median(new), 3)
        row["ws_spread_ms"] = [round(min(new), 3), round(max(new), 3)]
        if old:
            row["batch_device_ms"] = round(statistics.median(old), 3)
            row["batch_device_spread_ms"] = [round(min(old), 3), round(max(old), 3)]
        if name == "e":
            host = bt.t_data.cpu().numpy()
            host_compress(L, snap, host)
            ts = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                host_compress(L, snap, host)
                ts.append((time.perf_counter() - t0) * 1e3)
            row["host_sb_compress_ms"] = round(statistics.median(ts), 3)
        row["ceiling_ms"] = round(ceiling_ms(snap, bt.t_data, args.reps), 3)
        for k in ("ws", "batch_device", "host_sb_compress", "ceiling"):
            if k + "_ms" in row:
                row[k + "_gbps"] = round(total / row[k + "_ms"] / 1e6, 2)
        info["workloads"][name] = row
        print(name, json.dumps(row), flush=True)
        del bt
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "raw_batch_compress_bench.json"), "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
