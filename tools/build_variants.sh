#!/bin/bash
# Build field-product variants of the library next to the shipped one, here (no GPU needed), so the GPU box only has to run them:
#   proof_systems_b200/libzkb200_<tag>.so   for every "tag:flags" argument, e.g.  k5:-DZK_MUL_PLAIN_PER_ROW=5
# Select one at run time with ZKB200_LIB=<path> (proof_systems_b200/_lib.py).
set -e
cd "$(dirname "$0")/../proof_systems_b200/csrc"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
for spec in "$@"; do
  tag=${spec%%:*}; flags=${spec#*:}
  dir=/tmp/zkb_build_$tag; mkdir -p $dir
  for f in api msm ntt srs group_ntt decompress ipa open $EXTRA_SRCS; do
    [ -f $f.cu ] || continue
    $NVCC -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -Xcompiler -fPIC,-fvisibility=hidden -ccbin /usr/bin/g++ \
      --expt-relaxed-constexpr $flags -c -o $dir/$f.o $f.cu &
  done
  wait
  $NVCC -gencode arch=compute_90a,code=sm_90a -shared -o ../libzkb200_$tag.so $dir/*.o -Xcompiler -fPIC -lcudart
  echo "built libzkb200_$tag.so"
done
