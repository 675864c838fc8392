#!/bin/bash
# Experiment: what would 2x the resident warps cost?  (PK_SHADOW, csrc/b200env.cu)
#   bash tools/shadow.sh build    compiles vid2player3d_b200/lib/ab_w{5,6,7}_{r128,shadow}.so
#   bash tools/shadow.sh          (GPU box) parity subset with the shadow build, then tools/perf_step.py / perf_federer.py per variant
cd "$(dirname "$0")/.."
D=$PWD/vid2player3d_b200/lib
if [ "$1" = "build" ]; then
  FL="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 --shared -Xcompiler -fPIC -diag-suppress 177,550"
  S="vid2player3d_b200/csrc/b200env.cu vid2player3d_b200/csrc/b200env_v2p.cu"
  for w in 5 6 7; do
    /usr/local/cuda/bin/nvcc $FL -DPK_WARPS=$w -DPK_BOUND_WARPS=14 -o $D/ab_w${w}_r128.so $S &
    /usr/local/cuda/bin/nvcc $FL -DPK_WARPS=$w -DPK_SHADOW=1 -DPK_BOUND_WARPS=14 -o $D/ab_w${w}_shadow.so $S &
  done
  wait
  ls -la $D
  exit 0
fi
echo "== parity with the shadow build"; B200ENV_LIB=$D/ab_w7_shadow.so python -m pytest tests/test_gpu_parity.py -m gpu -x -q 2>&1 | tail -2
for r in 1 2; do
  python tools/perf_step.py 8192 160
  for f in $D/ab_w*.so; do B200ENV_LIB=$f python tools/perf_step.py 8192 160; done
done
for f in $D/libb200env.so $D/ab_w7_r128.so $D/ab_w7_shadow.so; do
  echo "== federer $f"; B200ENV_LIB=$f python tools/perf_federer.py 2>&1 | tail -12
done
