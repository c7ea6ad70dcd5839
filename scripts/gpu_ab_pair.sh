# A/B of the warp-kernel variants on one H100: parity tests, bench per variant, one ncu capture
set -x
python -m pytest tests -m gpu -x -q 2>&1 | tail -4
run() {  # label, env...
  local label=$1; shift
  env "$@" python bench.py --steps 100 --warmup 5 --no-cpu-baseline --no-extras --e2e-steps 5 2>&1 | tail -1 > gpurun_out/bench_ab_$label.json
  python -c "import sys,json; d=json.loads(open('gpurun_out/bench_ab_$label.json').read()); print('== $label %.3e steps/s'%d['value'], d['per_kind_ms'], 'frac %.3f'%d['roofline']['frac'], 'e2e %.3e'%d['e2e']['value'], d['clocks'])"
}
run pair REDNOSE_B200_WARP_KERNEL=pair
for d in rednose_b200/generated_g*; do run $(basename $d) REDNOSE_B200_GENERATED_DIR=$PWD/$d; done
run single REDNOSE_B200_WARP_KERNEL=single
run pair2 REDNOSE_B200_WARP_KERNEL=pair
ncu --set full --clock-control none --import-source on -k regex:ekf_step_pair -s 3 -c 2 -o gpurun_out/prof_ab python bench.py --steps 4 --warmup 3 --no-cpu-baseline --no-extras --e2e-steps 0 > gpurun_out/b_ncu_ab.log 2>&1
ncu -i gpurun_out/prof_ab.ncu-rep --page raw --csv > gpurun_out/raw_ab.csv 2>/dev/null
