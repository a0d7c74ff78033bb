#!/bin/bash
# Static instruction census of K1's parser loops; needs no GPU. Compiles snapb200.cu to an sm_90a cubin with the
# product's flags, disassembles k1_m7_kernel<NG> (NG=0 by default), finds its loops (the natural loops of its backward
# branches, so the cold blocks ptxas places after a loop count as part of it) and prints, per loop, the instruction
# count and the counts of the instructions that cost more than an issue slot (SHFL, VOTE, REDUX, MATCH, FLO, shared
# and global loads/stores, BSSY = divergent regions to reconverge from), plus every K1 kernel's registers and spills
# from -Xptxas -v. In k1_m7_kernel<0> the first large loop is the emitter's, the largest the chain's loop over units;
# nested in that one are the parse loop of k1_parse, in it the loop of windows whose probe the previous window issued
# (k1_probe_complete + k1_finish), and beside that the serial path.
# A static count is a rehearsal metric: it is not a time and says nothing about which instructions a window executes.
# WAITS=1 adds the scoreboard table of one loop (HEAD=0x..., default the largest loop at depth 2: the loop of windows
# whose probe was issued early). Every instruction's control bits are decoded from the high word of its 128-bit
# encoding (bits 41..44 stall cycles, 45 yield, 46..48 write scoreboard, 49..51 read scoreboard, 7 = none, 52..57 wait
# mask); the per-instruction listing goes to $OUT/census.ctrl. For every instruction of the loop that sets a scoreboard
# the table gives the first later instruction that waits on it and the distance in instructions, reading the loop as
# laid out: through conditional branches (so a rare block placed inline is read, as a reader of the listing would),
# along unconditional ones, once through nested loops, past the BRA.DIV fallbacks (taken only by a diverged warp), and
# across the back edge into the next iteration. A wait a few instructions after a long-latency load is a stall.
# usage: tools/k1_sass_census.sh [extra nvcc flags, e.g. -DK1_PROFILE]
#   NG=5|7 picks the kernel, MIN=n hides loops under n instructions, SASS=1 reuses the listing already in $OUT
# The cubin, the SASS listing and the ptxas log go to $OUT (default build/k1_exp, kept out of git).
set -e
cd "$(dirname "$0")/.."
OUT=${OUT:-build/k1_exp}
NG=${NG:-0}
MIN=${MIN:-40}     # loops shorter than this many instructions are not listed
mkdir -p "$OUT"
[ -n "$SASS" ] || nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xptxas -v "$@" -cubin \
     -o "$OUT/census.cubin" rust-snappy_b200/csrc/snapb200.cu 2> "$OUT/census.ptxas.log"
[ -n "$SASS" ] || cuobjdump -sass "$OUT/census.cubin" > "$OUT/census.sass"
python3 - "$OUT/census.sass" "$OUT/census.ptxas.log" "$NG" "$MIN" "${WAITS:-0}" "${HEAD:-}" "$OUT/census.ctrl" <<'PY'
import re, sys
sass, log, ng, minlen = sys.argv[1], sys.argv[2], sys.argv[3], int(sys.argv[4])
waits, head_arg, ctrl_out = sys.argv[5] == "1", sys.argv[6], sys.argv[7]
# registers and spills of every K1 kernel
lines = open(log).read().splitlines()
for i, l in enumerate(lines):
    m = re.search(r"Compiling entry function '\w*k1_m7_kernelILi(\d+)E\w*'", l)
    if m:
        info = " ".join(x.split(":", 1)[-1].strip() for x in lines[i + 1:i + 4] if "bytes stack" in x or "Used" in x)
        print("k1_m7_kernel<%s>: %s" % (m.group(1), info))
# instructions of k1_m7_kernel<NG>: [address, opcode, branch target or None, predicated, text]; hi[k] = high
# 64 bits of the encoding, which cuobjdump prints alone on the line after the instruction; raw[k] = text with predicate
ins, hi, raw, on = [], [], [], False
for l in open(sass):
    if "Function :" in l:
        on = ("k1_m7_kernelILi%sE" % ng) in l
        continue
    if not on:
        continue
    m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);", l)
    if not m:
        h = re.match(r"\s*/\* (0x[0-9a-f]{16}) \*/\s*$", l)
        if h and len(hi) < len(ins):
            hi.append(int(h.group(1), 16))
        continue
    text = m.group(2).strip()
    raw.append(text)
    pred = text.startswith("@")
    text = re.sub(r"^@!?U?P\w+\s+", "", text)
    op = text.split()[0]
    t = re.search(r"\b0x([0-9a-f]+)\s*$", text)
    ins.append((int(m.group(1), 16), op, int(t.group(1), 16) if t else None, pred, text))
if not ins:
    sys.exit("k1_m7_kernel<%s> not found in %s" % (ng, sass))
print("k1_m7_kernel<%s>: %d SASS instructions" % (ng, sum(1 for a in ins if a[1] != "NOP")))
# control-flow graph over instructions. BSYNC Bx continues at the target the last BSSY Bx on the way set: the possible
# targets per barrier register are propagated forward along the edges until nothing changes.
idx = {a[0]: k for k, a in enumerate(ins)}
def breg(text):
    return text.split()[1].rstrip(",")
state = [None] * len(ins)            # per instruction: {barrier register: set of targets} on entry
succ = [set() for _ in ins]
state[0] = {}
todo = [0]
while todo:
    k = todo.pop()
    ad, op, t, pred, text = ins[k]
    base, out = op.split(".")[0], {b: set(v) for b, v in state[k].items()}
    nxt, fall = [], True
    if base == "BSSY" and t in idx:
        out[breg(text)] = {idx[t]}
    elif base in ("BRA", "JMP") and t in idx:
        nxt.append(idx[t]); fall = pred or ".DIV" in op
    elif base == "BSYNC":
        nxt += sorted(state[k].get(breg(text), ())); fall = pred
    elif base in ("EXIT", "RET", "BRX", "JMX"):
        fall = pred
    if fall and k + 1 < len(ins):
        nxt.append(k + 1)
    for x in nxt:
        succ[k].add(x)
        if state[x] is None:
            state[x] = {b: set(v) for b, v in out.items()}; todo.append(x)
        else:
            grew = False
            for b, v in out.items():
                have = state[x].setdefault(b, set())
                if not v <= have:
                    have |= v; grew = True
            if grew:
                todo.append(x)
pred_of = [[] for _ in ins]
for k, ss in enumerate(succ):
    for x in ss:
        pred_of[x].append(k)
# natural loop of a backward edge a -> t: everything that reaches a without passing through t. When that includes the
# kernel's entry, t does not dominate a: the edge is a cold block placed after the loop jumping back, not a loop.
loops = {}
for k, ss in enumerate(succ):
    for h in ss:
        if h > k:
            continue
        body, todo = {h, k}, [k]
        while todo:
            for q in pred_of[todo.pop()]:
                if q not in body:
                    body.add(q); todo.append(q)
        if 0 not in body or h == 0:
            loops.setdefault(h, set()).update(body)
cols = ["SHFL", "VOTE", "REDUX", "MATCH", "FLO", "BREV", "LDS", "STS", "LD", "ST", "BSSY", "BRA"]
fam = {"LDG": "LD", "STG": "ST"}     # global accesses through a generic pointer are LD / ST
print("%-10s %5s %6s " % ("loop head", "depth", "instr") + " ".join("%5s" % c for c in cols))
for h in sorted(loops):
    body = [ins[k][1] for k in sorted(loops[h]) if ins[k][1] != "NOP"]
    if len(body) < minlen:
        continue
    depth = sum(1 for h2 in loops if h2 != h and loops[h] < loops[h2])
    cnt = [sum(1 for op in body if fam.get(op.split(".")[0], op.split(".")[0]) == c) for c in cols]
    print("0x%05x    %5d %6d " % (ins[h][0], depth, len(body)) + " ".join("%5d" % c for c in cnt))
if not waits:
    sys.exit(0)
if len(hi) != len(ins):
    sys.exit("control words: %d of %d instructions" % (len(hi), len(ins)))
def ctrl(k):
    c = hi[k] >> 41
    return {"stall": c & 15, "yield": (c >> 4) & 1, "wr": (c >> 5) & 7, "rd": (c >> 8) & 7, "wait": (c >> 11) & 63}
if head_arg:
    h0 = idx[int(head_arg, 16)]
else:
    depth2 = [h for h in loops if sum(1 for h2 in loops if h2 != h and loops[h] < loops[h2]) == 2]
    h0 = max(depth2, key=lambda h: len(loops[h]))
body = loops[h0]
order = sorted(body)
with open(ctrl_out, "w") as f:
    f.write("loop 0x%05x: address  stall yield wr rd wait  instruction\n" % ins[h0][0])
    for k in order:
        c = ctrl(k)
        f.write("0x%05x  %2d %d %s %s %s  %s\n" % (ins[k][0], c["stall"], c["yield"], "-" if c["wr"] == 7 else c["wr"],
                "-" if c["rd"] == 7 else c["rd"], "".join(str(b) for b in range(6) if c["wait"] >> b & 1) or "-", raw[k]))
def layout_next(k):
    ad, op, t, pred, text = ins[k]
    if op.split(".")[0] in ("BRA", "JMP") and not pred and ".DIV" not in op and t in idx:
        if idx[t] > k or idx[t] == h0:
            return idx[t]
    elif op.split(".")[0] in ("EXIT", "RET") and not pred:
        return None
    return k + 1
def nearest_wait(k, sb):
    j, d = layout_next(k), 1
    while j is not None and j in body and j != k:
        if ctrl(j)["wait"] >> sb & 1:
            return j, d
        j, d = layout_next(j), d + 1
    return None, None
print("scoreboards of loop 0x%05x (%d instructions): setter -> first waiter as laid out" % (ins[h0][0], len(body)))
print("%-8s %-30s %-3s %-8s %-30s %5s" % ("set at", "instruction", "sb", "wait at", "instruction", "dist"))
short = lambda x: " ".join(raw[x].split()[:4])[:30]
for k in order:
    c = ctrl(k)
    for kind in ("wr", "rd"):
        sb = c[kind]
        if sb == 7:
            continue
        j, d = nearest_wait(k, sb)
        print("0x%05x  %-30s %s%d  %-8s %-30s %5s" % (ins[k][0], short(k), kind[0], sb,
              "0x%05x" % ins[j][0] if j is not None else "-", short(j) if j is not None else "(no wait in the loop)",
              d if j is not None else "-"))
PY
