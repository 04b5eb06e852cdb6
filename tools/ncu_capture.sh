#!/bin/bash
# ncu captures of one matcher(batch) step (tools/profile_step.py: batch 8 x 640x480, thr 0).  Usage:
#   tools/ncu_capture.sh <tag>            -> gpurun_out/<tag>_launches.csv      (every launch, durations only)
#                                            gpurun_out/<tag>_tf.ncu-rep         (--set full, transformer + SIMT kernels)
#                                            gpurun_out/<tag>_conv.ncu-rep       (--set full, backbone kernels)
#                                            gpurun_out/<tag>_match.ncu-rep      (--set full, score / fine kernels)
tag="${1:-r2}"
mkdir -p gpurun_out
cd "$(dirname "$0")/.."
NCU="ncu --clock-control none --profile-from-start off --kernel-name-base demangled"
timeout 600 $NCU --metrics gpu__time_duration.sum --csv --log-file gpurun_out/${tag}_launches.csv \
  python tools/profile_step.py > gpurun_out/${tag}_launches.out 2>&1
FULL="--set full --import-source on"
# first self layer + first cross pass of the coarse transformer (every kernel kind once or twice)
timeout 900 $NCU $FULL -k regex:"EpiActStore|EpiLayerNorm|EpiPlanes|EpiKv|EpiAttn|kv_tile_merge|coarse_prep" -c "${NCU_TF_COUNT:-16}" \
  -f -o gpurun_out/${tag}_tf python tools/profile_step.py > gpurun_out/${tag}_tf.out 2>&1
timeout 900 $NCU $FULL -k regex:"EpiConv|stem" -c 23 -f -o gpurun_out/${tag}_conv python tools/profile_step.py \
  > gpurun_out/${tag}_conv.out 2>&1
timeout 900 $NCU $FULL -k regex:"EpiScore|fine_|match_|kv_window|lse_merge|argmax_merge" -c 12 -f -o gpurun_out/${tag}_match \
  python tools/profile_step.py > gpurun_out/${tag}_match.out 2>&1
ls -la gpurun_out/${tag}_*
