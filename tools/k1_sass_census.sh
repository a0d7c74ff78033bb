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
python3 - "$OUT/census.sass" "$OUT/census.ptxas.log" "$NG" "$MIN" <<'PY'
import re, sys
sass, log, ng, minlen = sys.argv[1], sys.argv[2], sys.argv[3], int(sys.argv[4])
# registers and spills of every K1 kernel
lines = open(log).read().splitlines()
for i, l in enumerate(lines):
    m = re.search(r"Compiling entry function '\w*k1_m7_kernelILi(\d+)E\w*'", l)
    if m:
        info = " ".join(x.split(":", 1)[-1].strip() for x in lines[i + 1:i + 4] if "bytes stack" in x or "Used" in x)
        print("k1_m7_kernel<%s>: %s" % (m.group(1), info))
# instructions of k1_m7_kernel<NG>: [address, opcode, branch target or None, predicated]
ins, on = [], False
for l in open(sass):
    if "Function :" in l:
        on = ("k1_m7_kernelILi%sE" % ng) in l
        continue
    if not on:
        continue
    m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);", l)
    if not m:
        continue
    text = m.group(2).strip()
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
PY
