"""Gathers over streams in pinned host memory (sb_*_table_gather_host_streams_ws) against the other ways a user can read
ranges of a corpus that lives in host memory. --streams copies of one 16 MiB text stream, frame and raw, each tabled by
the batch encoders, in one pinned buffer allocated after the thread is bound to the GPU's NUMA node. Workloads:
  loader   4,096 random 4 KiB ranges per call;
  small    65,536 random 256 B ranges, uniform over the streams;
  zipf     65,536 random 256 B ranges, Zipf-skewed (s = 1.1) over the streams;
  whole    one whole 16 MiB stream;
  million  2^20 uniform 256 B ranges: nearly every chunk is touched, where host residency stops paying.
Each runs through
  host     the host-stream gather over the pinned streams;
  device   the device gather over device-resident copies (the ceiling);
  zcopy    the device gather handed the pinned addresses directly (zero copy: the kernels read across PCIe);
  upload   every stream copied to the device, then the device gather.
The four run alternately, medians of --reps after a warm-up. Per call: the compressed bytes the call decodes (computed
from the table on the host: each edge once per work item of 256 ranges, each interior chunk once per range) and that
over the host call's time, beside a pinned-to-device cudaMemcpyAsync rate measured in the same run. Every range of
every mode is checked against the device gather before and after the timed calls.
--host-gib G: the loader workload over G GiB of compressed streams in host memory (more than the card holds), host mode
only, when MemAvailable allows it.

    python tools/host_gather_bench.py [--streams 1024] [--reps 5] [--only frame,raw] [--host-gib 0] [--out DIR]
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
from frame_table_bench import alternating  # noqa: E402

D = 16 * MIB
GROUP = 256


def i64(v):
    return torch.from_numpy(np.asarray(v, dtype=np.uint64).view(np.int64)).cuda()


def mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


class Corpus:
    """`count` copies of one encoded stream back to back in pinned host memory, their device copies (when asked) and
    one shared seek table (tables hold no pointers). spans: per chunk or block (decoded offset, decoded length,
    compressed bytes)."""

    def __init__(self, snap, fmt, text, count, device=True):
        enc = snap.frame.encode_batch if fmt == "frame" else snap.raw.compress_batch
        (s,), (t,) = enc([text], tables=True)
        self.fmt, self.count, self.n = fmt, count, len(s)
        self.host = torch.empty(count * self.n + 16, dtype=torch.uint8, pin_memory=True)
        one = torch.frombuffer(bytearray(s), dtype=torch.uint8)
        self.host[:count * self.n].view(count, self.n).copy_(one.expand(count, self.n))
        self.dev = self.host.cuda() if device else None
        self.table = torch.frombuffer(bytearray(t), dtype=torch.uint8).cuda()
        self.t_tables = i64([self.table.data_ptr()] * count + [0])
        self.t_lens = i64([self.n] * count + [0])
        self.t_host = i64([self.host.data_ptr() + i * self.n for i in range(count)] + [0])
        self.t_dev = i64([self.dev.data_ptr() + i * self.n for i in range(count)] + [0]) if device else None
        w = np.frombuffer(t[:64], dtype=np.uint64)
        if fmt == "frame":
            nch = int(w[3]) & 0xFFFFFFFF
            r = np.frombuffer(t[64:64 + 32 * nch], dtype=np.uint64).reshape(nch, 4)
            self.spans = np.stack([r[:, 3], r[:, 1] >> 32, r[:, 1] & 0xFFFFFFFF], axis=1).astype(np.int64)
            self.dn = int(w[2])
        else:
            self.dn, nb = int(w[2]), int(w[3]) >> 32
            offs = np.frombuffer(t[64:64 + 8 * nb], dtype=np.uint32).reshape(nb, 2)[:, 0].astype(np.int64)
            body = np.diff(np.append(offs, self.n))
            j = np.arange(nb, dtype=np.int64)
            self.spans = np.stack([j << 16, np.minimum(65536, self.dn - (j << 16)), body], axis=1)

    def fetched(self, ranges):
        """Compressed bytes a gather of `ranges` decodes: edges once per work item of GROUP ranges, interiors once per
        range (all ranges inside the streams)."""
        off, dl, body = self.spans[:, 0], self.spans[:, 1], self.spans[:, 2]
        u = np.array([r[0] for r in ranges], dtype=np.int64)
        lo = np.array([r[1] for r in ranges], dtype=np.int64)
        end = np.minimum(lo + np.array([r[2] for r in ranges], dtype=np.int64), self.dn)
        first = np.searchsorted(off + dl, lo, side="right")              # the run: off + dlen > lo and off < end
        last = np.searchsorted(off, end, side="left") - 1
        has = last >= first
        pre = np.concatenate([[0], np.cumsum(body)])
        f, l = first[has], last[has]
        total = int(np.where(l > f + 1, pre[np.maximum(l, 0)] - pre[np.minimum(f + 1, len(off))], 0).sum())
        keys = {}
        for k, ok in ((f, np.ones(len(f), dtype=bool)), (l, l > f)):      # the middle of a run is always inside
            kk, lk, ek, uk = k[ok], lo[has][ok], end[has][ok], u[has][ok]
            ins = (off[kk] >= lk) & (off[kk] + dl[kk] <= ek)
            total += int(body[kk[ins]].sum())
            for key in zip(uk[~ins].tolist(), kk[~ins].tolist()):
                keys[key] = keys.get(key, 0) + 1
        return total + sum((c + GROUP - 1) // GROUP * int(body[k]) for (_, k), c in keys.items())


class Calls:
    """One gather call of `ranges` over a corpus, in one of the four modes."""

    def __init__(self, L, snap, corpus, ranges, mode):
        self.L, self.snap, self.c, self.mode = L, snap, corpus, mode
        self.k = k = len(ranges)
        n = np.array([r[2] for r in ranges], dtype=np.int64)
        at = np.concatenate([[0], np.cumsum(n)])
        self.out = torch.empty(int(at[-1]) + 1, dtype=torch.uint8, device="cuda")
        self.t_lo = i64([r[1] for r in ranges])
        self.t_len = i64(n)
        self.t_ptr = i64(at[:k] + self.out.data_ptr())
        self.t_unit = torch.from_numpy(np.array([r[0] for r in ranges], dtype=np.uint32).view(np.int32)).cuda()
        self.t_ol = torch.zeros(k, dtype=torch.int64, device="cuda")
        self.t_st = torch.zeros(4 * k, dtype=torch.int64, device="cuda")
        host = mode == "host"
        kind = "gather_host_streams" if host else "gather"
        self.fn = getattr(L, "sb_%s_table_%s" % (corpus.fmt, kind + ("_ws" if host else "_device_ws")))
        self.need = getattr(L, "sb_%s_table_%s_scratch_bytes" % (corpus.fmt, kind))(k)
        self.scr = torch.empty(self.need, dtype=torch.uint8, device="cuda")
        self.t_ins = corpus.t_dev if mode in ("device", "upload") else corpus.t_host

    def __call__(self):
        c = self.c
        if self.mode == "upload":
            c.dev.copy_(c.host, non_blocking=True)
        e = self.snap._lib.SbError()
        check(self.fn(c.t_tables.data_ptr(), self.t_ins.data_ptr(), c.t_lens.data_ptr(), c.count, self.t_unit.data_ptr(),
                      self.t_lo.data_ptr(), self.t_len.data_ptr(), self.t_ptr.data_ptr(), self.t_ol.data_ptr(),
                      self.t_st.data_ptr(), self.k, self.scr.data_ptr(), self.need,
                      torch.cuda.current_stream().cuda_stream, C.byref(e)), e)

    def result(self):
        torch.cuda.synchronize()
        return self.t_ol.cpu(), self.t_st.cpu(), self.out[:-1].cpu()


def workloads(count, dn, rng):
    uni = lambda k, size: [(rng.randrange(count), lo, size) for lo in (rng.randrange(dn - size) for _ in range(k))]
    w = 1.0 / np.arange(1, count + 1) ** 1.1
    zu = np.random.default_rng(rng.randrange(1 << 30)).choice(count, 65536, p=w / w.sum())
    return [("loader 4096 x 4 KiB", uni(4096, 4 * KIB)), ("small 65536 x 256 B", uni(65536, 256)),
            ("zipf 65536 x 256 B", [(int(u), rng.randrange(dn - 256), 256) for u in zu]),
            ("whole 1 x 16 MiB", [(rng.randrange(count), 0, dn)]), ("million 2^20 x 256 B", uni(1 << 20, 256))]


def copy_rate(corpus, reps):
    """Pinned-to-device cudaMemcpyAsync of up to 1 GiB of the corpus: bytes per second (the PCIe ceiling)."""
    n = min(GIB, corpus.count * corpus.n)
    dst = torch.empty(n, dtype=torch.uint8, device="cuda")
    (t,) = alternating([lambda: dst.copy_(corpus.host[:n], non_blocking=True)], reps)
    return n / t


def run_format(L, snap, fmt, text, args, info):
    rng = random.Random(7)
    c = Corpus(snap, fmt, text, args.streams)
    rate = copy_rate(c, args.reps)
    print("%s: %d streams of %.2f MB compressed (%.1f GB), pinned-to-device copy %.1f GB/s" %
          (fmt, c.count, c.n / 1e6, c.count * c.n / 1e9, rate / 1e9), flush=True)
    rows = {"copy_gbps": rate / 1e9, "stream_bytes": c.n, "workloads": {}}
    modes = ("host", "device", "zcopy", "upload")
    for name, ranges in workloads(c.count, c.dn, rng):
        calls = [Calls(L, snap, c, ranges, m) for m in modes]
        for f in calls:
            f()
        want = calls[1].result()
        for f in calls:
            got = f.result()
            assert all(torch.equal(a, b) for a, b in zip(got, want)), (fmt, name, f.mode)
        ts = alternating(calls, args.reps)
        for f in calls:
            got = f.result()
            assert all(torch.equal(a, b) for a, b in zip(got, want)), (fmt, name, f.mode)
        fetched = c.fetched(ranges)
        row = {m: t * 1e3 for m, t in zip(modes, ts)}
        row.update(fetched_mb=fetched / 1e6, host_gbps=fetched / ts[0] / 1e9)
        rows["workloads"][name] = row
        print("  %-22s host %8.3f ms  device %8.3f ms  zcopy %8.3f ms  upload %8.3f ms | fetched %7.1f MB, %5.1f GB/s" %
              (name, row["host"], row["device"], row["zcopy"], row["upload"], row["fetched_mb"], row["host_gbps"]),
              flush=True)
        del calls
    info["formats"][fmt] = rows
    del c
    torch.cuda.empty_cache()


def run_large(L, snap, text, gib, args, info):
    """The loader workload, host mode only, over gib GiB of compressed frame streams in pinned host memory."""
    (s,), _ = snap.frame.encode_batch([text[:MIB]], tables=True)
    enc_n = len(s) * 16                                                  # about a 16 MiB stream's compressed size
    count = int(gib * GIB // enc_n)
    need = count * enc_n * 1.1 + 4 * GIB
    if mem_available() < need:
        msg = "skipped: %.1f GiB wanted, MemAvailable %.1f GiB" % (need / GIB, mem_available() / GIB)
        print("host-gib %g: %s" % (gib, msg), flush=True)
        info["large"] = msg
        return
    c = Corpus(snap, "frame", text, count, device=False)
    ranges = workloads(c.count, c.dn, random.Random(3))[0][1]
    f = Calls(L, snap, c, ranges, "host")
    (t,) = alternating([f], args.reps)
    fetched = c.fetched(ranges)
    info["large"] = {"gib": c.count * c.n / GIB, "ms": t * 1e3, "fetched_mb": fetched / 1e6}
    print("host-gib: %.1f GiB of frame streams in host memory, loader call %.3f ms, fetched %.1f MB (%.1f GB/s)" %
          (c.count * c.n / GIB, t * 1e3, fetched / 1e6, fetched / t / 1e9), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=1024)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", default="frame,raw")
    ap.add_argument("--host-gib", type=float, default=0)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    snap = graft.load_package()
    L = snap._lib.lib()
    node = L.sb_bind_host_thread_to_device_numa(torch.cuda.current_device())
    info = {"card": card(), "numa_node": node, "mem_available_gib": mem_available() / GIB, "formats": {}}
    print("card: %s | NUMA node %d | MemAvailable %.1f GiB" % (info["card"], node, info["mem_available_gib"]), flush=True)
    text = device_text(D).cpu().numpy().tobytes()
    for fmt in args.only.split(","):
        run_format(L, snap, fmt, text, args, info)
    if args.host_gib:
        run_large(L, snap, text, args.host_gib, args, info)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "host_gather_bench.json"), "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
