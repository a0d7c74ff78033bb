#!/bin/bash
# K1 launch sweep, one bench run per setting:
#   CAPS: SNAPB200_K1_CHAINS = chains per SM (shared-memory-table chains fill first, so a cap <= 7 runs that many
#         shared-memory chains and no L2-table chain), each with SNAPB200_K1_NG = 0
#   NGS:  SNAPB200_K1_NG = L2-table chains per SM next to the 7 shared-memory ones, no cap
# LIBS="name=path ..." runs the sweep for each library (default: the one in the tree); a library that predates
# SNAPB200_K1_CHAINS ignores it, so give it CAPS="" or read its cap rows as repeats of the uncapped one.
# Each run's JSON line and stderr go to $OUT (default build/k1_exp, kept out of git).
cd "$(dirname "$0")/.."
OUT=${OUT:-build/k1_exp}
mkdir -p "$OUT"
BLOCKS=${BLOCKS:-262144}
for spec in ${LIBS:-tree=}; do
  name=${spec%%=*}; lib=${spec#*=}
  runs=""
  for cap in ${CAPS-5 6}; do runs="$runs $cap:0"; done
  for ng in ${NGS-0 2 4 5 7}; do runs="$runs 0:$ng"; done
  for r in $runs; do
    cap=${r%%:*}; ng=${r#*:}; tag=${name}_c${cap}_ng${ng}
    SNAPB200_LIB=$lib SNAPB200_K1_CHAINS=$cap SNAPB200_K1_NG=$ng timeout 300 python bench.py --blocks $BLOCKS --wave 65536 \
        --steps 2 --no-e2e --no-cpu-baseline --no-parity > "$OUT/sweep_$tag.json" 2> "$OUT/sweep_$tag.err"
    python - "$OUT" "$tag" "$cap" "$ng" <<'PY'
import json, sys
out, tag, cap, ng = sys.argv[1:]
try:
    d = json.loads(open("%s/sweep_%s.json" % (out, tag)).read().strip().splitlines()[-1])
    print("%-22s chains cap %s NG %s: compress %.2f decompress %.2f value %.2f" % (tag, cap or "-", ng, d["compress_gbs"], d["decompress_gbs"], d["value"]))
except Exception as e:
    print(tag, "FAILED", e); print(open("%s/sweep_%s.err" % (out, tag)).read()[-800:])
PY
  done
done
