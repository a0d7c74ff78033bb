"""Batches of raw streams over 64 KB: sb_decompress_batch_device_ws (K8 over the batch: every multi-block unit split into
its blocks, all blocks decoded in one grid) against sb_decompress_batch_device (one warp per unit) on the same
device-resident batches.

Each workload is timed by CUDA events, the two calls alternating, median of --reps timed calls after a warm-up, and
every output is checked against the input. The ceiling is the same data compressed as independent 64 KB units and
decoded by sb_decompress_batch_device. Workloads:
  a  4,096 x 1 MiB units of corpus text compressed by sb_compress
  b  256 x 16 MiB units (sb_compress)
  c  131,072 x 64 KB text units (one block each: the split has nothing to do)
  d  1,024 x 1 MiB pages compressed by pyarrow (Google's C++ snappy)
  e  one 256 MiB unit among 65,536 units of 64 KB

    python tools/raw_batch_decode_bench.py [--only abcde] [--reps N] [--out DIR]
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
SLOT = 76544
DATA = os.path.join(ROOT, "tests", "golden", "data")


def corpus(name):
    with open(os.path.join(DATA, name), "rb") as f:
        return f.read()


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def text(n):
    base = np.frombuffer(corpus("alice29.txt") + corpus("lcet10.txt") + corpus("html_x_4") + corpus("kppkn.gtb") +
                         corpus("urls.10K"), dtype=np.uint8)
    return np.resize(base, n)


def host_compress(L, snap, arr):
    cap = L.sb_max_compress_len(arr.size)
    out = np.empty(cap, dtype=np.uint8)
    n, e = C.c_size_t(0), snap._lib.SbError()
    assert L.sb_compress(arr.ctypes.data, arr.size, out.ctypes.data, cap, C.byref(n), C.byref(e)) == 0
    return out[:n.value]


def block_compress(L, snap, t_data):
    """Every 64 KB block of t_data as its own unit, compressed on the device: (slots, lens)."""
    nb = t_data.numel() // BLOCK
    slots = torch.empty(nb * SLOT, dtype=torch.uint8, device="cuda")
    lens = torch.zeros(nb, dtype=torch.int32, device="cuda")
    b = snap._lib.SbBatch()
    b.in_base, b.in_stride, b.in_len_uniform = t_data.data_ptr(), BLOCK, BLOCK
    b.out_base, b.out_stride, b.out_cap_uniform, b.out_lens, b.count = slots.data_ptr(), SLOT, SLOT, lens.data_ptr(), nb
    e = snap._lib.SbError()
    assert L.sb_compress_batch_device(C.byref(b), torch.cuda.current_stream().cuda_stream, C.byref(e)) == 0
    torch.cuda.synchronize()
    return slots, lens


class Batch:
    """Units at device pointers (t_in + offs), outputs back to back in one buffer, per-unit lengths and caps."""

    def __init__(self, snap, t_in, offs, lens, sizes):
        self.snap, self.L = snap, snap._lib.lib()
        n = len(offs)
        self.n, self.total = n, int(sum(sizes))
        self.in_bytes = int(np.asarray(lens, dtype=np.int64).sum())
        ooffs = np.concatenate([[0], np.cumsum(np.asarray(sizes, dtype=np.int64))[:-1]])
        self.t_out = torch.empty(self.total + 16, dtype=torch.uint8, device="cuda")
        self.t_ip = torch.tensor(np.asarray(offs, dtype=np.int64) + t_in.data_ptr(), device="cuda")
        self.t_op = torch.tensor(ooffs + self.t_out.data_ptr(), device="cuda")
        self.t_len = torch.tensor(np.asarray(lens, dtype=np.int64), dtype=torch.int32, device="cuda")
        self.t_cap = torch.tensor(np.asarray(sizes, dtype=np.int64), dtype=torch.int32, device="cuda")
        self.t_ol = torch.zeros(n, dtype=torch.int32, device="cuda")
        self.t_st = torch.zeros(n * 32, dtype=torch.uint8, device="cuda")
        self.t_blk = torch.zeros(n, dtype=torch.int32, device="cuda")
        self.sb = self.L.sb_decompress_batch_scratch_bytes(n, self.in_bytes)
        self.t_scr = torch.empty(self.sb, dtype=torch.uint8, device="cuda")
        b = snap._lib.SbBatch()
        b.in_ptrs, b.in_lens, b.out_ptrs, b.out_caps = self.t_ip.data_ptr(), self.t_len.data_ptr(), self.t_op.data_ptr(), self.t_cap.data_ptr()
        b.out_lens, b.statuses, b.count = self.t_ol.data_ptr(), self.t_st.data_ptr(), n
        self.b = b
        self._t_in = t_in

    def ws(self):
        e = self.snap._lib.SbError()
        assert self.L.sb_decompress_batch_device_ws(C.byref(self.b), self.in_bytes, self.t_blk.data_ptr(), self.t_scr.data_ptr(),
                                                    self.sb, torch.cuda.current_stream().cuda_stream, C.byref(e)) == 0

    def one_warp(self):
        e = self.snap._lib.SbError()
        assert self.L.sb_decompress_batch_device(C.byref(self.b), torch.cuda.current_stream().cuda_stream, C.byref(e)) == 0

    def check(self, t_data):
        torch.cuda.synchronize()
        assert bool((self.t_st.view(-1, 32)[:, :4] == 0).all()), "a unit failed"
        assert torch.equal(self.t_ol.to(torch.int64), self.t_cap.to(torch.int64))
        assert torch.equal(self.t_out[:self.total], t_data), "output differs from the input"
        self.t_out.fill_(0)


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def ceiling_ms(snap, t_data, reps):
    L = snap._lib.lib()
    slots, lens = block_compress(L, snap, t_data)
    nb = lens.numel()
    out = torch.empty(nb * BLOCK, dtype=torch.uint8, device="cuda")
    olens = torch.zeros(nb, dtype=torch.int32, device="cuda")
    st = torch.zeros(nb * 32, dtype=torch.uint8, device="cuda")
    b = snap._lib.SbBatch()
    b.in_base, b.in_stride, b.in_lens = slots.data_ptr(), SLOT, lens.data_ptr()
    b.out_base, b.out_stride, b.out_cap_uniform, b.out_lens, b.statuses, b.count = \
        out.data_ptr(), BLOCK, BLOCK, olens.data_ptr(), st.data_ptr(), nb
    e = snap._lib.SbError()
    run = lambda: L.sb_decompress_batch_device(C.byref(b), torch.cuda.current_stream().cuda_stream, C.byref(e))  # noqa: E731
    run()
    ms = statistics.median(timed(run) for _ in range(reps))
    assert torch.equal(out, t_data)
    return ms


def from_host_streams(snap, streams, sizes):
    """Compressed streams (numpy) uploaded back to back: a Batch over them."""
    offs = np.concatenate([[0], np.cumsum([s.size for s in streams])[:-1]]).astype(np.int64)
    t_in = torch.from_numpy(np.concatenate(streams)).cuda()
    return Batch(snap, t_in, offs, [s.size for s in streams], sizes)


def from_blocks(snap, slots, lens):
    n = lens.numel()
    return Batch(snap, slots, np.arange(n, dtype=np.int64) * SLOT, lens.cpu().numpy(), [BLOCK] * n)


def workload(name, snap):
    L = snap._lib.lib()
    if name in "ab":
        count, size = (4096, MIB) if name == "a" else (256, 16 * MIB)
        data = text(count * size + 7919 * count)
        units = [data[i * size + 7919 * i:(i + 1) * size + 7919 * i] for i in range(count)]
        streams = [host_compress(L, snap, u) for u in units]
        t_data = torch.from_numpy(np.concatenate(units)).cuda()
        return from_host_streams(snap, streams, [size] * count), t_data
    if name == "c":
        t_data = torch.from_numpy(text(131072 * BLOCK)).cuda()
        slots, lens = block_compress(L, snap, t_data)
        return from_blocks(snap, slots, lens), t_data
    if name == "d":
        import pyarrow as pa
        count = 1024
        data = text(count * MIB + 104729 * count)
        units = [data[i * MIB + 104729 * i:(i + 1) * MIB + 104729 * i] for i in range(count)]
        streams = [np.frombuffer(pa.compress(u.tobytes(), codec="snappy", asbytes=True), dtype=np.uint8) for u in units]
        t_data = torch.from_numpy(np.concatenate(units)).cuda()
        return from_host_streams(snap, streams, [MIB] * count), t_data
    # e: the 256 MiB unit at position 40,000 of 65,536 units of 64 KB
    big = text(256 * MIB + 12345)[12345:]
    t_small = torch.from_numpy(text(65535 * BLOCK + 999)[999:]).cuda()
    slots, lens = block_compress(L, snap, t_small)
    s_big = host_compress(L, snap, big)
    at = 40000
    lens_h = lens.cpu().numpy().astype(np.int64)
    t_in = torch.cat([slots, torch.from_numpy(s_big).cuda()])
    offs = list(np.arange(65535, dtype=np.int64) * SLOT)
    offs.insert(at, 65535 * SLOT)
    ulens = list(lens_h)
    ulens.insert(at, s_big.size)
    sizes = [BLOCK] * 65536
    sizes[at] = 256 * MIB
    t_data = torch.cat([t_small[:at * BLOCK], torch.from_numpy(big).cuda(), t_small[at * BLOCK:]])
    return Batch(snap, t_in, offs, ulens, sizes), t_data


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="abcde")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for raw_batch_decode_bench.json (default: print only)")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    snap = graft.load_package()
    info = {"card": card(), "torch": torch.__version__, "reps": args.reps, "workloads": {}}
    print("card:", info["card"], flush=True)
    for name in args.only:
        bt, t_data = workload(name, snap)
        bt.ws()
        bt.check(t_data)
        blocks = bt.t_blk.cpu().numpy()
        bt.one_warp()
        bt.check(t_data)
        new, old = [], []
        reps_old = args.reps if name != "e" else min(args.reps, 3)     # e's one-warp call takes seconds
        for r in range(args.reps):
            new.append(timed(bt.ws))
            if r < reps_old:
                old.append(timed(bt.one_warp))
        bt.check(t_data)
        ceil = ceiling_ms(snap, t_data, args.reps)
        row = {"units": bt.n, "out_bytes": bt.total, "in_bytes": bt.in_bytes,
               "split_units": int((blocks > 0).sum()), "blocks": int(blocks.sum()),
               "ws_ms": round(statistics.median(new), 3), "one_warp_ms": round(statistics.median(old), 3),
               "ws_spread_ms": [round(min(new), 3), round(max(new), 3)],
               "one_warp_spread_ms": [round(min(old), 3), round(max(old), 3)],
               "ceiling_ms": round(ceil, 3)}
        row["ws_gbps"] = round(bt.total / row["ws_ms"] / 1e6, 2)
        row["one_warp_gbps"] = round(bt.total / row["one_warp_ms"] / 1e6, 2)
        row["ceiling_gbps"] = round(bt.total / row["ceiling_ms"] / 1e6, 2)
        info["workloads"][name] = row
        print(name, json.dumps(row), flush=True)
        del bt, t_data
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "raw_batch_decode_bench.json"), "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
