# validation on one H100: parity tests, smoke, default bench, launch list
python -m pytest tests -m gpu -x -q 2>&1 | tail -3
python -c "import __graft_entry__ as g; g.smoke()" 2>&1 | tail -2
S=$(date +%s); python bench.py > gpurun_out/bench_final_r1.json 2> gpurun_out/bench_final_r1.err; E=$(date +%s); echo "default bench wall $((E-S)) s"
tail -c 4500 gpurun_out/bench_final_r1.json; tail -3 gpurun_out/bench_final_r1.err
ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file gpurun_out/launches_r1h.csv python bench.py --steps 6 --warmup 3 --no-cpu-baseline --no-extras --e2e-steps 3 > gpurun_out/b_launches_r1h.log 2>&1
wc -l gpurun_out/launches_r1h.csv
