# A/B of wide-kernel variants (fma + 4*style) on the saturation workload; prints kernel ms per step.
for v in ${VARIANTS:-0 8 9 11}; do
  DM_KERNEL_VARIANT=$v,0 python bench.py --workload saturate_135168x112KiB --steps 3 --no-e2e --no-cpu ${EXTRA} 2>&1 | python -c "
import sys,json
d=json.loads(sys.stdin.read().strip().split('\n')[-1]); r=d['roofline']
print('variant $v fma=%d style=%d kernel_ms=%.3f hash_GBps=%.1f frac=%.4f' % ($v%4, $v//4, r['kernel_ms_per_step'], r['achieved']/r['algorithmic_bytes_per_blob_byte'], r['frac']))"
done
