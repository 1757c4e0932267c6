#!/bin/bash
# Round evidence in one GPU call: sanitizer, ncu raw page + launch list, bench lines (both arms, configs 1 / 2 / 4).
# Usage (on the GPU box): bash tools/collect_evidence.sh <tag>      e.g. r02_v14
TAG=${1:-r02}
OUT=gpurun_out
mkdir -p $OUT
{
  echo "compute-sanitizer (CUDA 12.9) on $(nvidia-smi --query-gpu=name --format=csv,noheader | head -1), command: compute-sanitizer --tool <tool> python tools/sanitize_smoke.py"
  for tool in memcheck racecheck initcheck synccheck; do
    echo "== $tool"
    timeout 600 compute-sanitizer --tool $tool python tools/sanitize_smoke.py 2>&1 | grep -E "^ok|SUMMARY|Error|error|hazard|Invalid|Race" | head -20
  done
} > $OUT/${TAG}_sanitizer.txt 2>&1
timeout 600 ncu --set full --clock-control none -s 10 -c 5 -o $OUT/${TAG}_step python tools/ncu_step.py > $OUT/ncu_step.log 2>&1
ncu -i $OUT/${TAG}_step.ncu-rep --page raw --csv > $OUT/${TAG}_ncu_raw_B65536.csv 2>/dev/null
rm -f $OUT/${TAG}_step.ncu-rep
timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -s 200 -c 300 --csv --log-file $OUT/launches_${TAG}.csv python bench.py --streams 4096 --steps 2 --warmup 3 --no-cpu-baseline --no-legacy > /dev/null 2>&1
python bench.py > $OUT/${TAG}_bench_B65536.json 2> $OUT/bench_default.err
python bench.py --impl reference > $OUT/${TAG}_bench_reference_arm.json 2>> $OUT/bench_default.err
python bench.py --streams 4096 > $OUT/${TAG}_bench_B4096.json 2>> $OUT/bench_default.err
python bench.py --model tests/golden/sh.rnnn --total-streams 65536 --no-cpu-baseline --no-legacy > $OUT/${TAG}_bench_config4_sh_1gpu.json 2>> $OUT/bench_default.err
tail -c 400 $OUT/bench_default.err
head -c 600 $OUT/${TAG}_sanitizer.txt
python - <<PY
import json
for f in ("${TAG}_bench_B65536","${TAG}_bench_B4096","${TAG}_bench_config4_sh_1gpu","${TAG}_bench_reference_arm"):
    try:
        d=json.load(open("$OUT/"+f+".json"))
        print(f, "%.4g"%d["value"], "e2e %.4g"%d["e2e"]["value"], d.get("roofline",{}).get("frac"), d["config"]["workload"][:60])
        if d.get("cpu_baseline"): print("   cpu", {k:(round(v,1) if isinstance(v,float) else v) for k,v in d["cpu_baseline"].items() if k!="sample" and k!="sin_note"})
        if d.get("legacy_abi"): print("   legacy", d["legacy_abi"])
    except Exception as e: print(f, "ERR", e)
PY
