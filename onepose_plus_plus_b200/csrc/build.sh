#!/bin/bash
# Builds libopp_b200.so (sm_90a only) next to the Python package. Usage: build.sh [extra nvcc flags]
set -e
HERE="$(cd "$(dirname "$0")" && pwd)"
OUT="${OPP_OUT:-$HERE/../libopp_b200.so}"
OBJ="${OPP_OBJ:-$HERE/obj}"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-std=c++17 -O3 -lineinfo -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC -Xcompiler -Wall --expt-relaxed-constexpr"
mkdir -p "$OBJ"
pids=()
for f in opp_gemm opp_stages opp_pnp opp_metrics opp_image opp_train opp_train_fine opp_train_coarse_tf opp_train_backbone opp_train_kpt opp_train_batch opp_sfm_points opp_sfm_refine; do
  $NVCC $FLAGS "$@" -c "$HERE/$f.cu" -o "$OBJ/$f.o" &
  pids+=($!)
done
for p in "${pids[@]}"; do wait $p; done
$NVCC -shared -gencode arch=compute_90a,code=sm_90a -o "$OUT" "$OBJ/opp_gemm.o" "$OBJ/opp_stages.o" "$OBJ/opp_pnp.o" \
  "$OBJ/opp_metrics.o" "$OBJ/opp_image.o" "$OBJ/opp_train.o" "$OBJ/opp_train_fine.o" \
  "$OBJ/opp_train_coarse_tf.o" "$OBJ/opp_train_backbone.o" "$OBJ/opp_train_kpt.o" \
  "$OBJ/opp_train_batch.o" "$OBJ/opp_sfm_points.o" "$OBJ/opp_sfm_refine.o"
echo "built $OUT"
