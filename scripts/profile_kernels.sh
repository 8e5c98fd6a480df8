#!/usr/bin/env bash
# ncu evidence of one bench step (one GPU; run under gpurun):   bash scripts/profile_kernels.sh [tag]
#   gpurun_out/<tag>_launches.csv          launch list of `bench.py --steps 1 --warmup 1` (cold-cache, serialised: shares)
#   gpurun_out/<tag>_gemm.json             ncu --set full summary of one ViT layer's four F16 GEMMs + two BF16X3 conv GEMMs
#   gpurun_out/<tag>_kernels.{ncu-rep,json} attention_f16, LayerNorm, conv0 stats/apply, positional conv, long-key attention
#   gpurun_out/<tag>_fusion.{ncu-rep,json}  the two kernels of one fusion training step (graph replay)
# Three profiled processes instead of one per kernel: the capture windows are set with MER_CUPROF (runtime.cu).  The
# GEMM report (source pages of 6 large kernels, ~40 MB) is summarised on the box and dropped: gpurun_out/ comes back only
# below 64 MiB.  Environment switches (MER_ATT_SHORT=...) are inherited.
set -u
tag=${1:-r2}
out=gpurun_out
mkdir -p "$out"
ncu --metrics gpu__time_duration.sum --clock-control none -s 200 -c 900 --csv --log-file "$out/${tag}_launches.csv" \
    python bench.py --steps 1 --warmup 1 --cpu-clips 2 --no-extras > "$out/${tag}_launches.log" 2>&1
echo "launch list: exit $?"
full="ncu --set full --clock-control none --import-source on --profile-from-start off -f"
MER_CUPROF="2:21:4,1:0:2" $full -o "$out/${tag}_gemm" python scripts/profile_step.py > "$out/${tag}_gemm.log" 2>&1
echo "gemm: exit $?"
python scripts/ncu_hotspots.py "$out/${tag}_gemm.ncu-rep" > "$out/${tag}_gemm.json" 2>> "$out/${tag}_gemm.log" && rm -f "$out/${tag}_gemm.ncu-rep"
MER_CUPROF="10:2:1,12:8:1,14:0:1,13:0:1,15:0:1" $full -o "$out/${tag}_kernels" python scripts/profile_step.py --long-audio \
    > "$out/${tag}_kernels.log" 2>&1
echo "kernels: exit $?"
python scripts/ncu_hotspots.py "$out/${tag}_kernels.ncu-rep" > "$out/${tag}_kernels.json" 2>> "$out/${tag}_kernels.log"
$full -o "$out/${tag}_fusion" python scripts/bench_fusion_step.py --no-cpu --batches 32 --iters 1 --profile \
    > "$out/${tag}_fusion.log" 2>&1
echo "fusion: exit $?"
python scripts/ncu_hotspots.py "$out/${tag}_fusion.ncu-rep" > "$out/${tag}_fusion.json" 2>> "$out/${tag}_fusion.log"
ls -la "$out" | grep "${tag}_"
du -sh "$out"
