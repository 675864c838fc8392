#!/bin/bash
# Build ablated variants of the step kernel (-DABL=n, see b200env.cu) and time each with tools/perf_step.py.
# Usage (on the GPU box): bash tools/ablate.sh run      |  (build container): bash tools/ablate.sh build
set -e
cd "$(dirname "$0")/.."
D=vid2player3d_b200/lib
if [ "$1" = "build" ]; then
  for v in ${ABLS:-1 2 3 4 5}; do
    /usr/local/cuda/bin/nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 --shared -Xcompiler -fPIC -diag-suppress 177,550 \
      -DABL=$v ${EXTRA} -o $D/abl_$v.so vid2player3d_b200/csrc/b200env.cu vid2player3d_b200/csrc/b200env_v2p.cu &
  done
  wait
else
  python tools/perf_step.py 8192 320
  for f in $D/abl_*.so; do B200ENV_LIB=$PWD/$f python tools/perf_step.py 8192 320; done
fi
