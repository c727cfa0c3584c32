#!/bin/bash
# Build liborb_b200 variants for kernel-tunable experiments: tools/build_variants.sh "name:unit:-DFLAG=.. -DFLAG2=.." ...
# (unit = extractor | matcher | lba | pose_opt: the translation unit the flags apply to).  Output: build/liborb_<name>.so -- git-ignored,
# but shipped to the GPU box; select with ORB_B200_LIB=build/liborb_<name>.so.
set -e
cd "$(dirname "$0")/.."
FLAGS="-std=c++17 -O3 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC"
mkdir -p build/obj
for f in orb_slam3_modified_b200/csrc/*.cu; do
  b=$(basename $f .cu)
  if [ ! build/obj/$b.o -nt $f ] || [ -n "$(find orb_slam3_modified_b200/csrc include -newer build/obj/$b.o \( -name '*.h' -o -name '*.cuh' -o -name '*.inc' \) | head -1)" ]; then
    nvcc $FLAGS -c $f -o build/obj/$b.o &
  fi
done
wait
for spec in "$@"; do
  name=${spec%%:*}; rest=${spec#*:}; unit=${rest%%:*}; defs=${rest#*:}
  others=$(for f in orb_slam3_modified_b200/csrc/*.cu; do b=$(basename $f .cu); [ "$b" != "$unit" ] && echo build/obj/$b.o; done)
  ( nvcc $FLAGS $defs -c orb_slam3_modified_b200/csrc/$unit.cu -o build/obj/${unit}_$name.o
    nvcc -shared -o build/liborb_$name.so build/obj/${unit}_$name.o $others -lcudart ) &
done
wait
ls -la build/*.so
