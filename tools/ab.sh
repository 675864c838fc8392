#!/bin/bash
# A/B of step-kernel variants.
#   bash tools/ab.sh build     (build container) compiles the prepared variants into vid2player3d_b200/lib/ab_*.so:
#                              ab_nocc.so = -DPK_CONTACT_COMPACT=0 (the in-place ground contact; the compacted phase is the default since r2a),
#                              ab_p3.so = -DB200ENV_WITH_PACKED3=1 (tools/variants/packed3.cuh, run with B200ENV_KERNEL=packed3)
#   bash tools/ab.sh           (GPU box, e.g. `gpurun -- 'bash tools/ab.sh > gpurun_out/ab.log 2>&1'`): parity subset for every variant,
#                              then tools/perf_step.py for the product build and every variant, each also with B200ENV_SORT=1
#                              (envs handed out by ground-contact load) and, for the product build, B200ENV_KERNEL=packed3.
cd "$(dirname "$0")/.."
D=$PWD/vid2player3d_b200/lib
if [ "$1" = "build" ]; then
  FL="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 --shared -Xcompiler -fPIC -diag-suppress 177,550"
  /usr/local/cuda/bin/nvcc $FL -DPK_CONTACT_COMPACT=0 ${EXTRA} -o $D/ab_nocc.so vid2player3d_b200/csrc/b200env.cu vid2player3d_b200/csrc/b200env_v2p.cu
  /usr/local/cuda/bin/nvcc $FL -DB200ENV_WITH_PACKED3=1 ${EXTRA} -o $D/ab_p3.so vid2player3d_b200/csrc/b200env.cu vid2player3d_b200/csrc/b200env_v2p.cu
  ls -la $D
  exit 0
fi
python -m pytest tests -m gpu -x -q 2>&1 | tail -4
for f in $D/ab_*.so; do
  [ -e "$f" ] || continue
  echo "== parity $f"; B200ENV_LIB=$f python -m pytest tests/test_gpu_parity.py tests/test_zz_sort_gpu.py -m gpu -x -q 2>&1 | tail -2
done
for r in 1 2; do
  python tools/perf_step.py 8192 320
  B200ENV_SORT=1 python tools/perf_step.py 8192 320 | sed 's/^/SORT=1 /'
  [ -e $D/ab_p3.so ] && B200ENV_LIB=$D/ab_p3.so B200ENV_KERNEL=packed3 python tools/perf_step.py 8192 320
  for f in $D/ab_*.so; do
    [ -e "$f" ] || continue
    B200ENV_LIB=$f python tools/perf_step.py 8192 320
    B200ENV_LIB=$f B200ENV_SORT=1 python tools/perf_step.py 8192 320 | sed 's/^/SORT=1 /'
  done
done
