mkdir -p gpurun_out
for k in 4 8 10 16 30 64 1024; do   # 1024: one warp per unit, the default
  SNAPB200_K2_CTAS=$k timeout 200 python bench.py --blocks 65536 --wave 32768 --steps 2 --no-e2e --no-cpu-baseline --no-parity > gpurun_out/k2c_$k.json 2> gpurun_out/k2c_$k.err
  python -c "
import json
d=json.load(open('gpurun_out/k2c_$k.json')); print('CTAS/SM=$k decompress', round(d['decompress_gbs'],2))"
done
