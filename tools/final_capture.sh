# profiling evidence on one GPU (the H100 the library targets): ncu --set full of one bench step AT THE BENCH BATCH (128 frames x 3 cameras), launch list, the
# default bench run of every config and the reference arm.  Reports come back in gpurun_out/, summaries are made from them with
# tools/profile_summary.py / ncu_lines.py / ncu_phases.py / make_k1_traffic.py and committed under profiles/.
#   tools/final_capture.sh r3            config 2 in full + bench lines of configs 3 and 4
#   FULL=1 tools/final_capture.sh r3     ... + ncu of config 4's kernels and the reference arm of configs 3 and 4
set -x
R=${1:-r3}
mkdir -p gpurun_out
# kernels per step: 8 x K1, K2, K3, lists, acceptance = 12; bench.py --warmup 3 runs 3 warm-up steps first
ncu --set full --clock-control none --import-source on -k regex:"pyr_fast|octree|describe|hamming_stream|stream_replay" -s 36 -c 12 -f -o gpurun_out/${R}_step python bench.py --steps 1 --warmup 3 --no-cpu-baseline > gpurun_out/ncu_${R}_step.log 2>&1
tail -2 gpurun_out/ncu_${R}_step.log
ncu --metrics gpu__time_duration.sum --clock-control none -c 400 --csv --log-file gpurun_out/${R}_launches.csv python bench.py --steps 2 --warmup 3 --no-cpu-baseline > gpurun_out/b.log 2>&1
if [ -n "$FULL" ]; then
ncu --set full --clock-control none --import-source on -k regex:"hamming_topk|bruteforce_replay" -s 2 -c 2 -f -o gpurun_out/${R}_cfg4 python bench.py --config 4 --steps 1 --warmup 3 --no-cpu-baseline > gpurun_out/ncu_${R}_cfg4.log 2>&1
fi
python bench.py > gpurun_out/${R}_bench_c2.json 2> gpurun_out/${R}_bench_c2.err
python bench.py --impl reference --steps 2 --warmup 1 > gpurun_out/${R}_bench_reference_c2.json 2> gpurun_out/${R}_bench_reference_c2.err
for C in 3 4; do
  python bench.py --config $C --no-cpu-baseline > gpurun_out/${R}_bench_c$C.json 2> gpurun_out/${R}_bench_c$C.err
  if [ -n "$FULL" ]; then python bench.py --config $C --impl reference --steps 2 --warmup 1 > gpurun_out/${R}_bench_reference_c$C.json 2> gpurun_out/${R}_bench_reference_c$C.err; fi
done
tail -c 700 gpurun_out/${R}_bench_c2.json; tail -c 500 gpurun_out/${R}_bench_reference_c2.json; tail -c 400 gpurun_out/${R}_bench_c3.json; tail -c 400 gpurun_out/${R}_bench_c4.json
