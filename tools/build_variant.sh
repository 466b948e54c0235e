#!/bin/bash
# tools/build_variant.sh NAME "EXTRA_NVCC_FLAGS"  -> tools/variants/libdfk_NAME.so (A/B kernel variants, loaded with DFK_LIB=...)
set -e
NAME=$1; EXTRA=$2
ROOT=$(cd "$(dirname "$0")/.." && pwd)
OUT=$ROOT/tools/variants; mkdir -p $OUT/obj_$NAME
cd $ROOT/deepfactors_b200/csrc
ARCH="-gencode arch=compute_90a,code=sm_90a"
for f in dfk_api dfk_sfm_fp32 dfk_sfm_tc dfk_sfm_wide dfk_sfm_rays dfk_sfm_finalize dfk_simple dfk_window dfk_depth dfk_sparse; do
  if [ "$f" = "dfk_sfm_tc" ] || [ ! -f $OUT/obj_$NAME/$f.o ] || [ $f.cu -nt $OUT/obj_$NAME/$f.o ]; then
    if [ "$f" = "dfk_sfm_tc" ]; then X="$EXTRA"; else X=""; fi
    nvcc $ARCH -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -I../../include -I. $X -c $f.cu -o $OUT/obj_$NAME/$f.o &
  fi
done
wait
nvcc $ARCH -shared -o $OUT/libdfk_$NAME.so $OUT/obj_$NAME/*.o
echo built $OUT/libdfk_$NAME.so
