#!/bin/bash
# tools/build_variant.sh NAME "EXTRA_NVCC_FLAGS"  -> tools/variants/libdfk_NAME.so (A/B kernel variants, loaded with DFK_LIB=...)
# Builds every source of deepfactors_b200/csrc/Makefile, with the extra flags, from a copy of the sources in
# tools/variants/src_NAME (so the in-tree objects stay as they are), from scratch every time.
set -e
NAME=$1; EXTRA=$2
ROOT=$(cd "$(dirname "$0")/.." && pwd)
OUT=$ROOT/tools/variants; SRC=$OUT/src_$NAME
rm -rf $SRC; mkdir -p $SRC
cp -p $ROOT/deepfactors_b200/csrc/Makefile $ROOT/deepfactors_b200/csrc/*.cu $ROOT/deepfactors_b200/csrc/*.cuh \
  $ROOT/deepfactors_b200/csrc/*.h $SRC/
make -C $SRC -j "$(nproc)" -s EXTRA="$EXTRA -I$ROOT/include" HDRS= OUT=$OUT/libdfk_$NAME.so
rm -rf $SRC
echo built $OUT/libdfk_$NAME.so
