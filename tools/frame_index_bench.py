"""Frame decode with and without a chunk index, and the K7 indexer alone, on one GPU.

Two streams:
  big    >= 4 GiB of synthetic text (bench.py's generator) frame-encoded on the device, 64 KB chunks, with the
         encoder's chunk index;
  small  >= 65,536 chunks of <= 4 KB, prepared on the host (the oracle's frame_encode of 4000-byte writes).
For each, sb_frame_decode_device_ws is timed with CUDA events three ways:
  (a) with the encoder's index, (b) without an index (K7 builds it on the device), (c) without an index on the same
  stream with one padding chunk after the identifier (K7 declines, one thread walks the headers; same output bytes),
and sb_frame_index_device_ws alone. Every decode is compared with the input. Prints one JSON line per stream, with the
card's name and power limit.

  python tools/frame_index_bench.py [--gib 4] [--small-chunks 65536] [--reps 3]
"""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import __graft_entry__ as graft  # noqa: E402

TEXT_FILES = ["alice29.txt", "asyoulik.txt", "lcet10.txt", "plrabn12.txt"]
BLOCK, MUL = 65536, 65521
PADDING = b"\xfe\x00\x00\x00"          # an empty padding chunk


def card():
    name, limit_w = torch.cuda.get_device_name(0), None
    try:
        import pynvml
        pynvml.nvmlInit()
        h = pynvml.nvmlDeviceGetHandleByIndex(torch.cuda.current_device())
        limit_w = pynvml.nvmlDeviceGetPowerManagementLimit(h) / 1000.0
    except Exception:  # noqa: BLE001
        pass
    return name, limit_w


class Runner:
    def __init__(self):
        self.snap = graft.load_package()
        self.L = self.snap._lib.lib()
        self.err = self.snap._lib.SbError()
        self.st = torch.cuda.current_stream().cuda_stream
        self.dev = torch.device("cuda:0")

    def ck(self, rc):
        if rc:
            raise self.snap.error.from_c(self.err)

    def timed(self, fn, reps):
        ms = []
        for _ in range(reps + 1):                          # first call warms up
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            ms.append(a.elapsed_time(b))
        return sorted(ms[1:])

    def decode(self, t_stream, m, t_out, n, t_idx, nidx, maxc, t_scr, t_res):
        self.ck(self.L.sb_frame_decode_device_ws(t_stream.data_ptr(), m, t_out.data_ptr(), n,
                                                 t_idx.data_ptr() if t_idx is not None else None, nidx, 0, t_res.data_ptr(),
                                                 t_scr.data_ptr(), t_scr.numel(), maxc, self.st, C.byref(self.err)))

    def measure(self, label, t_stream, m, t_in, n, t_idx, nchunks, reps):
        """(a), (b), (c) and K7 alone over the stream t_stream[:m] whose decode is t_in[:n]."""
        dev = self.dev
        maxc = nchunks + 1024
        t_scr = torch.empty(self.L.sb_frame_decode_scratch_bytes(maxc), dtype=torch.uint8, device=dev)
        t_res = torch.zeros(64, dtype=torch.uint8, device=dev)
        t_out = torch.empty(n + 16, dtype=torch.uint8, device=dev)
        t_pad = torch.cat([t_stream[:10], torch.tensor(list(PADDING), dtype=torch.uint8, device=dev), t_stream[10:m]])
        res_t = self.snap._lib.SbFrameResult

        def check(nbytes_expected):
            r = res_t.from_buffer_copy(bytes(t_res.cpu().numpy()[:C.sizeof(res_t)]))
            assert r.status.code == 0 and r.bytes == nbytes_expected and r.nchunks == nchunks, (label, r.status.code, r.bytes)
            assert torch.equal(t_out[:n], t_in[:n]), label
            t_out.fill_(0)

        out = {"stream": label, "uncompressed_bytes": n, "stream_bytes": m, "chunks": nchunks}
        for key, fn in (("a_with_index_ms", lambda: self.decode(t_stream, m, t_out, n, t_idx, nchunks, maxc, t_scr, t_res)),
                        ("b_no_index_ms", lambda: self.decode(t_stream, m, t_out, n, None, 0, maxc, t_scr, t_res)),
                        ("c_walk_ms", lambda: self.decode(t_pad, m + len(PADDING), t_out, n, None, 0, maxc, t_scr, t_res))):
            ms = self.timed(fn, reps)
            check(n)
            out[key] = round(ms[len(ms) // 2], 3)
            out[key.replace("_ms", "_gbs")] = round(n / (ms[len(ms) // 2] * 1e-3) / 1e9, 2)
        # K7 alone, into its own scratch; the index must equal the encoder's
        t_kidx = torch.empty(maxc + 1, dtype=torch.int64, device=dev)
        t_cnt = torch.zeros(1, dtype=torch.int32, device=dev)
        sb = self.L.sb_frame_index_scratch_bytes(m, maxc)
        t_kscr = torch.empty(sb, dtype=torch.uint8, device=dev)
        ms = self.timed(lambda: self.ck(self.L.sb_frame_index_device_ws(t_stream.data_ptr(), m, 0, t_kidx.data_ptr(), maxc,
                                                                        t_cnt.data_ptr(), t_kscr.data_ptr(), sb, self.st,
                                                                        C.byref(self.err))), reps)
        assert int(t_cnt.item()) == nchunks and torch.equal(t_kidx[:nchunks + 1], t_idx[:nchunks + 1]), label
        out["k7_alone_ms"] = round(ms[len(ms) // 2], 3)
        return out


def big_stream(r, gib):
    dev = r.dev
    text = b"".join(open(os.path.join(ROOT, "tests", "golden", "data", f), "rb").read() for f in TEXT_FILES)
    blocks = int(gib * (1 << 30)) // BLOCK
    n = blocks * BLOCK
    t_text = torch.frombuffer(bytearray(text), dtype=torch.uint8).to(dev)
    t_in = torch.empty(n + 16, dtype=torch.uint8, device=dev)
    r.ck(r.L.sb_generate_blocks_device(t_text.data_ptr(), len(text), t_in.data_ptr(), BLOCK, BLOCK, 0, blocks, MUL, r.st,
                                       C.byref(r.err)))
    cap = r.L.sb_frame_max_len(n)
    t_out = torch.empty(cap + 16, dtype=torch.uint8, device=dev)
    t_idx = torch.zeros(blocks + 1, dtype=torch.int64, device=dev)
    t_res = torch.zeros(64, dtype=torch.uint8, device=dev)
    sb = r.L.sb_frame_encode_scratch_bytes(n)
    t_scr = torch.empty(sb, dtype=torch.uint8, device=dev)
    r.ck(r.L.sb_frame_encode_device_ws(t_in.data_ptr(), n, t_out.data_ptr(), cap, 1, t_idx.data_ptr(), t_res.data_ptr(),
                                       t_scr.data_ptr(), sb, r.st, C.byref(r.err)))
    torch.cuda.synchronize()
    del t_scr
    res = r.snap._lib.SbFrameResult.from_buffer_copy(bytes(t_res.cpu().numpy()[:C.sizeof(r.snap._lib.SbFrameResult)]))
    assert res.status.code == 0 and res.nchunks == blocks
    return t_out, res.bytes, t_in, n, t_idx, blocks


def small_stream(r, nchunks):
    """Host-prepared: 4000-byte writes, each its own chunk (the oracle's frame_encode, identifier once)."""
    from oracle import oracle as orc
    text = b"".join(open(os.path.join(ROOT, "tests", "golden", "data", f), "rb").read() for f in TEXT_FILES)
    piece, parts, offs, at, data = 4000, [orc.frame_encode(b"x")[:10]], [], 10, []
    for i in range(nchunks):
        o = (i * 7919 * 13) % (len(text) - piece)
        d = text[o:o + piece]
        c = orc.frame_encode(d)[10:]
        assert len(c) <= 4096
        data.append(d); parts.append(c); offs.append(at)
        at += len(c)
    offs.append(at)
    stream, plain = b"".join(parts), b"".join(data)
    dev = r.dev
    t_stream = torch.frombuffer(bytearray(stream) + bytearray(16), dtype=torch.uint8).to(dev)
    t_in = torch.frombuffer(bytearray(plain) + bytearray(16), dtype=torch.uint8).to(dev)
    t_idx = torch.tensor(offs, dtype=torch.int64, device=dev)
    return t_stream, len(stream), t_in, len(plain), t_idx, nchunks


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=4.0)
    ap.add_argument("--small-chunks", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    torch.cuda.set_device(0)
    r = Runner()
    name, limit_w = card()
    for build in (lambda: big_stream(r, a.gib), lambda: small_stream(r, a.small_chunks)):
        t_stream, m, t_in, n, t_idx, nchunks = build()
        res = r.measure("big" if nchunks * 65536 == n else "small", t_stream, m, t_in, n, t_idx, nchunks, a.reps)
        res.update({"card": name, "power_limit_w": limit_w})
        print(json.dumps(res), flush=True)
        del t_stream, t_in, t_idx
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
