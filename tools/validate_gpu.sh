#!/bin/bash
mkdir -p gpurun_out
rm -f gpurun_out/summary.txt
timeout -s KILL 1500 python -m pytest tests -q -m gpu > gpurun_out/t_gpu_all.log 2>&1
echo "pytest gpu exit $?" >> gpurun_out/summary.txt
timeout -s KILL 300 python __graft_entry__.py --smoke > gpurun_out/smoke.log 2>&1
echo "smoke exit $?" >> gpurun_out/summary.txt
timeout -s KILL 900 python bench.py > gpurun_out/bench_r1.json 2> gpurun_out/bench_r1.err
echo "bench exit $?" >> gpurun_out/summary.txt
timeout -s KILL 900 python bench.py --impl reference --steps 2 --warmup 1 > gpurun_out/bench_r1_reference.json 2>> gpurun_out/bench_r1.err
echo "bench ref exit $?" >> gpurun_out/summary.txt
timeout -s KILL 300 python tools/mega_timeline.py 1 > gpurun_out/mega_timeline_r1.txt 2>&1
timeout -s KILL 900 ncu --metrics gpu__time_duration.sum --clock-control none -k "regex:attention|cast_f32|embed_merge|k_attn|k_mega|k_sample|k_set_state|k_stream|layer_norm|mrope_kv|rms_norm|swiglu_kernel|vision_rope|gemm|k_pack" -c 3000 --csv --log-file gpurun_out/launches_request_r1.csv python tools/profile_decode.py 3 > gpurun_out/prof.log 2>&1
echo "ncu list exit $?" >> gpurun_out/summary.txt
timeout -s KILL 900 ncu --set full --clock-control none --import-source on -k "regex:k_mega" -s 2 -c 1 -o gpurun_out/prof_mega_r1 -f python tools/profile_decode.py 3 > gpurun_out/prof2.log 2>&1
echo "ncu full exit $?" >> gpurun_out/summary.txt
cat gpurun_out/summary.txt
grep -E "passed|failed" gpurun_out/t_gpu_all.log | tail -3
tail -2 gpurun_out/smoke.log
cut -c1-900 gpurun_out/bench_r1.json
cut -c1-300 gpurun_out/bench_r1_reference.json
tail -5 gpurun_out/bench_r1.err
