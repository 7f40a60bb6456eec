#!/bin/bash
# One gpurun call that produces the evidence of a round: final bench line, ncu launch list of the same command, `ncu --set full` of the
# largest kernels (one capture each), and the secondary workloads (configs[3] shape, configs[4] ANS1 block-size sweep, -l 1 / -l 4).
# usage (on the GPU box, from the repo root): bash tools/profile_round.sh r02
tag=${1:-r02}
out=gpurun_out
mkdir -p $out
python bench.py --steps 5 --warmup 3 > $out/${tag}_bench_final.json 2> $out/${tag}_bench_final.err
echo "bench rc=$?"
timeout 600 ncu --metrics gpu__time_duration.sum --clock-control none -c 20000 --csv --log-file $out/${tag}_launches_final.csv \
    python bench.py --steps 1 --warmup 1 --no-cpu-baseline --no-e2e > $out/${tag}_launch_bench.log 2>&1
echo "launch list rc=$?"
for k in sbrt_inverse_multi lzi_parse_kernel sbrt_rank_kernel lzp_spec_kernel lzp_junction_kernel bwtu_keys_kernel lzp_derive_kernel tp_round_eval_kernel; do
    timeout 400 ncu --set full --import-source on --clock-control none -k regex:$k -c 1 -f -o $out/${tag}_full_$k \
        python bench.py --steps 1 --warmup 1 --no-cpu-baseline --no-e2e > $out/${tag}_full_$k.log 2>&1
    echo "full $k rc=$?"
done
for w in enwik_l5 l1 l4 ans1_1m ans1_2m ans1_4m ans1_8m ans1_16m ans1_32m ans1_64m; do
    timeout 400 python bench.py --workload $w --steps 3 --warmup 3 --no-e2e > $out/${tag}_bench_workload_$w.json 2> $out/${tag}_bench_workload_$w.err
    echo "workload $w rc=$?"
done
