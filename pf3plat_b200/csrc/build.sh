#!/bin/sh
# Builds libgsplat_b200.so (sm_90a only, H100) in-tree.  Usage: sh build.sh [extra nvcc flags]
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
ARCH="-gencode arch=compute_90a,code=sm_90a"
FLAGS="$ARCH -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xcompiler -fvisibility=hidden --expt-relaxed-constexpr"
OBJS=""
PIDS=""
for f in gs_capi gs_preprocess gs_binning gs_composite_fwd gs_composite_bwd gs_preprocess_bwd gs_metrics gs_losses gs_pose_loss gs_lpips gs_adapter gs_cameras gs_costvolume gs_poses gs_encoder_depth gs_gaussian_head gs_sh_rotation; do
  stale=0
  for dep in "$f.cu" gs_common.cuh gs_bin_policy.h gs_det.cuh gs_tile_sort.cuh gs_inverse.cuh gs_adapter_math.cuh gs_sh_fit.h ../../include/gsplat_b200.h build.sh; do
    if [ ! -f "$f.o" ] || [ "$dep" -nt "$f.o" ]; then stale=1; fi
  done
  if [ "$stale" = 1 ]; then
    rm -f "$f.o"
    $NVCC $FLAGS "$@" -c "$f.cu" -o "$f.o" &
    PIDS="$PIDS $!"
  fi
  OBJS="$OBJS $f.o"
done
# a failed compile must fail the build (a bare `wait` returns 0 whatever its jobs returned); every job is waited for
# first, so that none is still running when the script exits
failed=0
for p in $PIDS; do wait "$p" || failed=1; done
if [ "$failed" = 1 ]; then echo "build.sh: compilation failed" >&2; exit 1; fi
$NVCC $ARCH -shared -o libgsplat_b200.so $OBJS -lcudart
echo "built $(pwd)/libgsplat_b200.so"
