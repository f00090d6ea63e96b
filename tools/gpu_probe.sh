# one GPU visit: smoke, stage times, all GPU tests, the bench at every config, ncu captures
timeout 90 python -c "import __graft_entry__ as g; g.smoke()" 2>&1 | tail -1 || { echo "SMOKE FAILED OR HUNG"; exit 1; }
timeout 200 python tools/stage_probe.py 128 stats 2>&1 | grep -E "images:|tiers"; timeout 100 python tools/stage_probe.py 1 2>&1 | grep -E "images:"
timeout 900 python -m pytest tests -m gpu -q > gpurun_out/gpu_tests.log 2>&1; tail -4 gpurun_out/gpu_tests.log
for CFG in 2 3 4; do
timeout 400 python bench.py --steps 6 --warmup 3 --no-cpu-baseline --config $CFG > gpurun_out/bench_c$CFG.json 2> gpurun_out/bench_c$CFG.err
python - $CFG <<'PY'
import json, sys
try:
    j = json.loads(open(f"gpurun_out/bench_c{sys.argv[1]}.json").read().strip().splitlines()[-1])
    print("BENCH config", sys.argv[1], j["run"].get("matcher_stats"), round(j["value"], 2), round(j["e2e"]["value"], 2), round(j["ms_per_step"], 3), {k: (round(v, 3) if v else v) for k, v in j["roofline"].get("stage_ms", {}).items()}, j.get("run", {}).get("single_frame_latency_ms"))
except Exception as e:
    print("bench failed", sys.argv[1], e)
PY
done
