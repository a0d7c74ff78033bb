#!/bin/bash
# Builds a separate library with parser phase timers (-DK1_PROFILE) and prints where the parser
# warp's cycles go. Diagnostic only; the product library is never built with K1_PROFILE.
set -e
cd "$(dirname "$0")/.."
mkdir -p gpurun_out
nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -shared -Xcompiler -fPIC -DK1_PROFILE \
     -o gpurun_out/libsnapb200_prof.so rust-snappy_b200/csrc/snapb200.cu
SNAPB200_LIB=$PWD/gpurun_out/libsnapb200_prof.so python - <<'PY'
import ctypes as C, json, os, sys
sys.path.insert(0, os.getcwd())
import torch
import __graft_entry__ as graft
from bench import load_text, BLOCK, MUL, STRIDE
snap = graft.load_package(); L = snap._lib.lib(); err = snap._lib.SbError()
torch.cuda.set_device(0); dev = torch.device("cuda:0"); st = torch.cuda.current_stream().cuda_stream
n = 16576
text = load_text()
t_text = torch.frombuffer(bytearray(text), dtype=torch.uint8).to(dev)
t_in = torch.empty(n * BLOCK, dtype=torch.uint8, device=dev); t_c = torch.empty(n * STRIDE, dtype=torch.uint8, device=dev)
cl = torch.zeros(n, dtype=torch.int32, device=dev)
L.sb_generate_blocks_device(t_text.data_ptr(), len(text), t_in.data_ptr(), BLOCK, BLOCK, 0, n, MUL, st, C.byref(err))
b = snap._lib.SbBatch(); b.in_base, b.in_stride, b.in_len_uniform = t_in.data_ptr(), BLOCK, BLOCK
b.out_base, b.out_stride, b.out_cap_uniform, b.out_lens, b.count = t_c.data_ptr(), STRIDE, STRIDE, cl.data_ptr(), n
L.sb_compress_batch_device(C.byref(b), st, C.byref(err)); torch.cuda.synchronize()
out = (C.c_ulonglong * 16)()
L.sb_debug_k1_profile(out, 1)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(); L.sb_compress_batch_device(C.byref(b), st, C.byref(err)); e1.record(); torch.cuda.synchronize()
L.sb_debug_k1_profile(out, 0)
if os.environ.get("SNAPB200_K1_X", "1") != "0":
    names = ["byte ring upkeep", "chunk pipeline (complete+issue)", "event ring space", "own bytes/hash/slot/info", "moved slots",
             "match.any + dynamic lanes", "walk", "commit", "exit state/publish/loop", "serial path", "block end", "windows"]
    wins = out[11]
    tot = sum(out[i] for i in range(11))
    print("kernel %.2f ms, %.2f GB/s; windows %d (%.1f bytes each); parser cycles per window: %.0f" % (e0.elapsed_time(e1), n * BLOCK / e0.elapsed_time(e1) / 1e6, wins, n * BLOCK / max(1, wins), tot / max(1, wins)))
    for i in range(11):
        print("  [%2d] %-34s %6.1f%%  %7.0f cyc/window" % (i, names[i], 100.0 * out[i] / tot, out[i] / max(1, wins)))
    sys.exit(0)
names = ["loop top/prefetch", "probe (hash,table,cand,compare)", "pointer doubling", "entry->taken copies", "interiors/inserted mask",
         "commit+verify(+clash)", "event ring", "exit state/copy-end insert", "(pre-serial)", "serial path", "block end", ""]
tot = sum(out[i] for i in range(11))
windows = n * 2048
print("kernel %.2f ms, %.2f GB/s; parser cycles per 32-byte window: %.0f" % (e0.elapsed_time(e1), n * BLOCK / e0.elapsed_time(e1) / 1e6, tot / windows))
for i in range(11):
    print("  [%2d] %-34s %6.1f%%  %7.0f cyc/window" % (i, names[i], 100.0 * out[i] / tot, out[i] / windows))
PY
