"""Raw-stream decode on the GPU: K8's parallel block decode against its ceiling and the one-warp path.

For each stream it reports the median of timed sb_decompress_device_ws calls (CUDA events, after a warm-up), K8's split
and block-decode kernel times from torch.profiler in a separate call, the ceiling (the same 64 KB blocks compressed as
independent units and decoded by sb_decompress_batch_device), and checks every output against the input. It also
times the one-warp path (the whole stream as one unit of sb_decompress_batch_device) on a prefix, host sb_decompress
of the 100 MB stream for this library against another build (--parent), alternating, and sweeps SNAPB200_K8_SEG.

    python tools/raw_decode_bench.py [--parent path/to/libsnapb200.so] [--out DIR]
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
DATA = os.path.join(ROOT, "tests", "golden", "data")


def corpus(name):
    with open(os.path.join(DATA, name), "rb") as f:
        return f.read()


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def ev_time(fn, reps, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ts.append(a.elapsed_time(b))
    return statistics.median(ts)


class Raw:
    def __init__(self, snap, t_in, n, dn):
        self.snap, self.L = snap, snap._lib.lib()
        self.t_in, self.n, self.dn = t_in, n, dn
        self.t_out = torch.empty(dn + 16, dtype=torch.uint8, device="cuda")
        self.sb = self.L.sb_decompress_scratch_bytes(n)
        self.t_scr = torch.empty(self.sb, dtype=torch.uint8, device="cuda")
        self.t_res = torch.zeros(64, dtype=torch.uint8, device="cuda")

    def __call__(self):
        e = self.snap._lib.SbError()
        rc = self.L.sb_decompress_device_ws(self.t_in.data_ptr(), self.n, self.t_out.data_ptr(), self.dn, self.t_res.data_ptr(),
                                            self.t_scr.data_ptr(), self.sb, torch.cuda.current_stream().cuda_stream, C.byref(e))
        assert rc == 0, rc

    def result(self):
        torch.cuda.synchronize()
        return self.snap._lib.SbFrameResult.from_buffer_copy(bytes(self.t_res.cpu().numpy()[:48]))


def device_compress(snap, t_data):
    """Every 64 KB block of t_data (a multiple of 65536 bytes) compressed as its own unit: (slots, lens)."""
    L = snap._lib.lib()
    nb = t_data.numel() // BLOCK
    slots = torch.empty(nb * 76544, dtype=torch.uint8, device="cuda")
    lens = torch.zeros(nb, dtype=torch.int32, device="cuda")
    b = snap._lib.SbBatch()
    b.in_base, b.in_stride, b.in_len_uniform = t_data.data_ptr(), BLOCK, BLOCK
    b.out_base, b.out_stride, b.out_cap_uniform, b.out_lens, b.count = slots.data_ptr(), 76544, 76544, lens.data_ptr(), nb
    e = snap._lib.SbError()
    assert L.sb_compress_batch_device(C.byref(b), torch.cuda.current_stream().cuda_stream, C.byref(e)) == 0
    torch.cuda.synchronize()
    return slots, lens


def ceiling_ms(snap, t_data, reps):
    L = snap._lib.lib()
    slots, lens = device_compress(snap, t_data)
    nb = lens.numel()
    out = torch.empty(nb * BLOCK, dtype=torch.uint8, device="cuda")
    olens = torch.zeros(nb, dtype=torch.int32, device="cuda")
    st = torch.zeros(nb * 32, dtype=torch.uint8, device="cuda")
    b = snap._lib.SbBatch()
    b.in_base, b.in_stride, b.in_lens = slots.data_ptr(), 76544, lens.data_ptr()
    b.out_base, b.out_stride, b.out_cap_uniform, b.out_lens, b.statuses, b.count = \
        out.data_ptr(), BLOCK, BLOCK, olens.data_ptr(), st.data_ptr(), nb
    e = snap._lib.SbError()
    ms = ev_time(lambda: L.sb_decompress_batch_device(C.byref(b), torch.cuda.current_stream().cuda_stream, C.byref(e)), reps)
    assert torch.equal(out, t_data)
    del slots, out, st
    return ms


def one_warp_ms(snap, stream_np, dn):
    """The whole stream as one unit of sb_decompress_batch_device: one warp."""
    L = snap._lib.lib()
    t_in = torch.from_numpy(stream_np).cuda()
    out = torch.empty(dn + 16, dtype=torch.uint8, device="cuda")
    olens = torch.zeros(1, dtype=torch.int32, device="cuda")
    st = torch.zeros(32, dtype=torch.uint8, device="cuda")
    b = snap._lib.SbBatch()
    b.in_base, b.in_len_uniform = t_in.data_ptr(), stream_np.size
    b.out_base, b.out_cap_uniform, b.out_lens, b.statuses, b.count = out.data_ptr(), dn, olens.data_ptr(), st.data_ptr(), 1
    e = snap._lib.SbError()
    return ev_time(lambda: L.sb_decompress_batch_device(C.byref(b), torch.cuda.current_stream().cuda_stream, C.byref(e)), 2, 1)


def device_stream(snap, t_data):
    """One raw stream of t_data (a multiple of 65536 bytes) assembled on the device from its blocks compressed as
    independent units: exactly what sb_compress writes, also where the input is too large for sb_compress's
    worst-case bound."""
    slots, lens = device_compress(snap, t_data)
    nb, head = lens.numel(), varint(t_data.numel())
    body = lens.to(torch.int64) - 3                                  # each unit's varint of 65536 is 3 bytes
    offs = torch.cumsum(body, 0) - body + len(head)
    n = int(offs[-1] + body[-1])
    out = torch.empty(n, dtype=torch.uint8, device="cuda")
    out[:len(head)] = torch.tensor(list(head), dtype=torch.uint8)
    for c0 in range(0, nb, 2048):
        b = body[c0:c0 + 2048]
        rep = torch.repeat_interleave(torch.arange(b.numel(), device="cuda"), b)
        within = torch.arange(rep.numel(), device="cuda") - (torch.cumsum(b, 0) - b)[rep]
        out[offs[c0:c0 + 2048][rep] + within] = slots[(c0 + rep) * 76544 + 3 + within]
    del slots
    return out


def varint(v):
    out = b""
    while v >= 0x80:
        out += bytes([v & 0x7F | 0x80])
        v >>= 7
    return out + bytes([v])


def host_compress(snap, arr):
    L = snap._lib.lib()
    cap = L.sb_max_compress_len(arr.size)
    out = np.empty(cap, dtype=np.uint8)
    n, e = C.c_size_t(0), snap._lib.SbError()
    assert L.sb_compress(arr.ctypes.data, arr.size, out.ctypes.data, cap, C.byref(n), C.byref(e)) == 0
    return out[:n.value]


def kernel_split(raw):
    """K8 split (every k8_* kernel but the block decode and the fallback) and block-decode time of one call, from
    torch.profiler (microseconds)."""
    from torch.profiler import ProfilerActivity, profile
    raw()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        raw()
        torch.cuda.synchronize()
    per = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        t = ev.cuda_time_total if t is None else t
        if t and ("k8_" in ev.key or "emset" in ev.key):
            name = ev.key.split("k8_")[1].split("_kernel")[0] if "k8_" in ev.key else "memset"
            per[name] = per.get(name, 0.0) + t
    blocks = per.get("blocks", 0.0)
    split = sum(v for k, v in per.items() if k not in ("blocks", "fallback"))
    return split, blocks, {k: round(v / 1e3, 3) for k, v in per.items()}


def bench_stream(snap, name, stream_np, t_data, reps, ceiling=True):
    dn = t_data.numel()
    t_in = torch.from_numpy(stream_np).cuda()
    raw = Raw(snap, t_in, stream_np.size, dn)
    ms = ev_time(raw, reps)
    r = raw.result()
    assert r.status.code == 0 and r.bytes == dn, (name, r.status.code)
    ok = torch.equal(raw.t_out[:dn], t_data)
    split_us, blocks_us, per = kernel_split(raw)
    row = {"stream": name, "compressed": int(stream_np.size), "bytes": dn, "parallel_blocks": int(r.nchunks),
           "output_matches": bool(ok), "ws_ms": round(ms, 3), "ws_GBps": round(dn / ms / 1e6, 2),
           "k8_split_ms": round(split_us / 1e3, 3), "block_decode_ms": round(blocks_us / 1e3, 3), "kernels_ms": per}
    if ceiling and dn % BLOCK == 0:
        c = ceiling_ms(snap, t_data, reps)
        row.update(ceiling_ms=round(c, 3), ceiling_GBps=round(dn / c / 1e6, 2))
    del raw, t_in
    torch.cuda.empty_cache()
    print(json.dumps(row), flush=True)
    return row


def seg_sweep(snap, name, stream_np, t_data, segs, reps):
    rows = []
    t_in = torch.from_numpy(stream_np).cuda()
    raw = Raw(snap, t_in, stream_np.size, t_data.numel())
    for s in segs:
        os.environ["SNAPB200_K8_SEG"] = str(s)
        ms = ev_time(raw, reps)
        r = raw.result()
        ok = r.status.code == 0 and torch.equal(raw.t_out[:t_data.numel()], t_data)
        rows.append({"stream": name, "seg": s, "ws_ms": round(ms, 3), "ok": bool(ok), "parallel_blocks": int(r.nchunks)})
        print(json.dumps(rows[-1]), flush=True)
    os.environ.pop("SNAPB200_K8_SEG", None)
    return rows


def host_ab(snap, parent, stream, data, reps):
    """Host sb_decompress of one stream with this library and with `parent`, alternating (seconds)."""
    libs = {"this": snap._lib.lib(), "parent": C.CDLL(parent)}
    out = np.empty(len(data) + 64, dtype=np.uint8)
    src = np.frombuffer(stream, dtype=np.uint8)
    times = {k: [] for k in libs}
    for _ in range(reps):
        for k, L in libs.items():
            n, e = C.c_size_t(0), snap._lib.SbError()
            t0 = time.perf_counter()
            rc = L.sb_decompress(C.c_void_p(src.ctypes.data), src.size, C.c_void_p(out.ctypes.data), out.size, C.byref(n), C.byref(e))
            times[k].append(time.perf_counter() - t0)
            assert rc == 0 and n.value == len(data) and out[:n.value].tobytes() == data, k
    return {k: [round(x, 4) for x in v] for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent", default=None, help="another libsnapb200.so for the host sb_decompress comparison")
    ap.add_argument("--out", default=None, help="directory for raw_decode_bench.json (default: print only)")
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--text-blocks", type=int, default=65535, help="64 KB blocks of the text stream")
    args = ap.parse_args()
    torch.cuda.set_device(0)
    snap = graft.load_package()
    rep = {"card": card(), "rows": [], "sweep": []}
    print("card:", rep["card"], flush=True)
    text = corpus("alice29.txt") + corpus("lcet10.txt") + corpus("html_x_4") + corpus("kppkn.gtb") + corpus("urls.10K")

    # 100 MB pyarrow stream (and the host A/B on it)
    import pyarrow as pa
    base = corpus("alice29.txt") + corpus("html") + corpus("kppkn.gtb") + corpus("urls.10K")
    pdata = (base * (100 * 1000 * 1000 // len(base) + 1))[:100 * 1000 * 1000]
    pstream = pa.compress(pdata, codec="snappy", asbytes=True)
    t_p = torch.frombuffer(bytearray(pdata), dtype=torch.uint8).cuda()
    rep["rows"].append(bench_stream(snap, "pyarrow 100 MB", np.frombuffer(pstream, dtype=np.uint8), t_p, args.reps, False))
    rep["sweep"] += seg_sweep(snap, "pyarrow 100 MB", np.frombuffer(pstream, dtype=np.uint8), t_p,
                              [128 << 10, 256 << 10, 512 << 10, 1 << 20], args.reps)
    ceil_n = len(pdata) // BLOCK * BLOCK
    c = ceiling_ms(snap, t_p[:ceil_n], args.reps)
    rep["rows"][-1].update(ceiling_ms_prefix=round(c, 3), ceiling_GBps=round(ceil_n / c / 1e6, 2))
    del t_p
    if args.parent:
        rep["host_ab_100mb_s"] = host_ab(snap, args.parent, pstream, pdata, 2)
        print(json.dumps({"host_ab_100mb_s": rep["host_ab_100mb_s"]}), flush=True)

    # one warp: a 16 MiB prefix of the text as one stream
    pre = np.resize(np.frombuffer(text, dtype=np.uint8), 16 << 20)
    ow = one_warp_ms(snap, host_compress(snap, pre), pre.size)
    rep["one_warp_16MiB"] = {"ms": round(ow, 2), "GBps": round(pre.size / ow / 1e6, 4)}
    print(json.dumps(rep["one_warp_16MiB"]), flush=True)

    for name, src, nb in (("fireworks.jpeg 1 GiB", corpus("fireworks.jpeg"), 16384), ("zeros 1 GiB", b"\0", 16384),
                          ("text %d x 64 KiB" % args.text_blocks, text, args.text_blocks)):
        t_d = torch.from_numpy(np.resize(np.frombuffer(src, dtype=np.uint8), nb * BLOCK)).cuda()
        stream = device_stream(snap, t_d).cpu().numpy()
        rep["rows"].append(bench_stream(snap, name, stream, t_d, args.reps))
        if not name.startswith("zeros"):
            rep["sweep"] += seg_sweep(snap, name, stream, t_d, [128 << 10, 256 << 10, 512 << 10, 1 << 20], 3)
        del t_d
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "raw_decode_bench.json"), "w") as f:
            json.dump(rep, f, indent=1)
    print(json.dumps(rep))


if __name__ == "__main__":
    main()
