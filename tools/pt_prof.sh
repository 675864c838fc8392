#!/bin/bash
# per-warp phase profile of the one-wave physics launch
#   bash tools/pt_prof.sh build   (build container) compiles vid2player3d_b200/lib/ab_prof.so with -DPT_PROF=1
#   bash tools/pt_prof.sh [steps] (GPU box) runs tools/pt_prof.py with it
cd "$(dirname "$0")/.."
D=$PWD/vid2player3d_b200/lib
if [ "$1" = "build" ]; then
  /usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 --shared -Xcompiler -fPIC -diag-suppress 177,550 \
    -DPT_PROF=1 -o $D/ab_prof.so vid2player3d_b200/csrc/b200env.cu vid2player3d_b200/csrc/b200env_v2p.cu && ls -la $D/ab_prof.so
  exit $?
fi
B200ENV_LIB=$D/ab_prof.so python tools/pt_prof.py "$@"
