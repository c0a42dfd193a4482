# One GPU session (bash tools/gpu_call.sh <tag> under gpurun)
tag=${1:-r02}
set -x
mkdir -p gpurun_out
timeout 900 python -m pytest tests -m gpu -x -q > gpurun_out/${tag}_pytest_gpu.log 2>&1; tail -5 gpurun_out/${tag}_pytest_gpu.log
timeout 300 python tools/bench_extra.py > gpurun_out/${tag}_secondary_kernels.json 2> gpurun_out/${tag}_secondary.err; cut -c1-300 gpurun_out/${tag}_secondary_kernels.json; tail -3 gpurun_out/${tag}_secondary.err
timeout 900 python bench.py --config c4 --no-cpu-baseline --no-e2e > gpurun_out/${tag}_bench_c4.json 2> gpurun_out/${tag}_bench_c4.err; tail -5 gpurun_out/${tag}_bench_c4.err
timeout 600 python bench.py --config c2 --no-cpu-baseline --no-e2e > gpurun_out/${tag}_bench_c2.json 2> gpurun_out/${tag}_bench_c2.err; tail -5 gpurun_out/${tag}_bench_c2.err
timeout 300 ncu --set full --clock-control none --import-source on -k regex:median_filter_merge -c 1 -f -o gpurun_out/${tag}_prof_mfmerge python tools/bench_extra.py > /dev/null 2>&1
timeout 300 ncu --set full --clock-control none --import-source on -k regex:viterbi_fast -s 3 -c 1 -f -o gpurun_out/${tag}_prof_vfast python bench.py --config c2 --no-cpu-baseline --no-e2e --steps 2 --warmup 1 > /dev/null 2>&1
ls -la gpurun_out | tail -6
