# usage: scripts/ab_variants.sh LIB1.so LIB2.so ...   one short bench.py run per built library, e.g. the parent commit's
# libggrmcp_b200.so next to this one's ("base" = the library of this tree)
for lib in "$@"; do
  if [ "$lib" = base ]; then path=""; else path=$(realpath "$lib"); fi
  GGR_LIB_PATH=$path python bench.py --steps 8 --warmup 3 --no-cpu-baseline --e2e-steps 1 --no-side-configs --no-parity 2>/dev/null | python -c "
import json,sys
d=json.loads(sys.stdin.read().strip().splitlines()[-1])
k=d['roofline']['kernels']
print('$lib', round(d['value']), round(d['ms_per_step'],3), {a:round(b['avg_ms'],3) for a,b in k.items() if b['avg_ms']>0.05})
"
done
