#!/bin/bash
# Builds a separate library with parser phase timers (-DK1_PROFILE) and prints where the parser
# warp's cycles go, plus the census of parser warps per warp scheduler (%warpid & 3) as the hardware
# placed them. Diagnostic only; the product library is never built with K1_PROFILE.
# usage: tools/k1_phase_profile.sh [profile library]   (given: use it instead of building one from the tree)
# The built library goes to $OUT (default build/k1_exp, kept out of git).
set -e
cd "$(dirname "$0")/.."
OUT=${OUT:-build/k1_exp}
mkdir -p "$OUT"
LIB=${1:-$(cd "$OUT" && pwd)/libsnapb200_prof.so}
if [ -z "$1" ]; then
  nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -shared -Xcompiler -fPIC -DK1_PROFILE \
       -o "$LIB" rust-snappy_b200/csrc/snapb200.cu
fi
SNAPB200_LIB=$LIB python - <<'PY'
import ctypes as C, os, sys
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
out = (C.c_ulonglong * 18)()
L.sb_debug_k1_profile(out, 1)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record(); L.sb_compress_batch_device(C.byref(b), st, C.byref(err)); e1.record(); torch.cuda.synchronize()
L.sb_debug_k1_profile(out, 0)
names = ["loop top/prefetch", "probe: candidate wait, compare", "pointer doubling", "entry->taken copies", "interiors/inserted mask",
         "commit+verify(+clash)", "probe issue + event ring", "exit state/copy-end insert", "(pre-serial)", "serial path",
         "block end", "probe issue at the loop top"]
tot = sum(out[i] for i in range(12))
windows = n * (BLOCK // 32)
fw = out[16] + out[17]
print("lib %s: kernel %.2f ms, %.2f GB/s; parser cycles per 32 input bytes: %.0f, per fast-path step: %.0f"
      % (os.path.basename(os.environ["SNAPB200_LIB"]), e0.elapsed_time(e1), n * BLOCK / e0.elapsed_time(e1) / 1e6,
         tot / windows, tot / max(fw, 1)))
for i in range(12):
    print("  [%2d] %-34s %6.1f%%  %7.0f cyc/32 B" % (i, names[i], 100.0 * out[i] / tot, out[i] / windows))
print("parser warps per scheduler (%%warpid & 3 = 0..3): %s" % [out[12 + s] for s in range(4)])
print("fast-path steps: %d (%.0f per block); probe issued by the previous step (hoisted): %d (%.1f%%), at the loop top: %d"
      % (fw, fw / n, out[16], 100.0 * out[16] / max(fw, 1), out[17]))
PY
