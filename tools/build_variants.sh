#!/bin/bash
# Build experiment variants of libf3dgs_b200.so: tools/build_variants.sh name1 "flags1" name2 "flags2" ...
# -> feature-3dgs_b200/variants/<name>/libf3dgs_b200.so (git-ignored).
set -e
cd "$(dirname "$0")/.."
python feature-3dgs_b200/build.py > /dev/null 2>&1   # base objects up to date
B=feature-3dgs_b200/build; S=feature-3dgs_b200/csrc
FL="-std=c++17 -O3 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC -Xptxas -v --expt-relaxed-constexpr"
while [ $# -ge 2 ]; do
  n=$1; f=$2; shift 2
  d=feature-3dgs_b200/variants/$n; mkdir -p $d
  ( for u in composite_fwd composite_bwd feature_bwd; do nvcc -c $S/$u.cu -o $d/$u.o $FL $f > $d/$u.log 2>&1 & done; wait )
  nvcc -shared -o $d/libf3dgs_b200.so $B/api.cu.o $B/binning.cu.o $B/preprocess.cu.o $B/feature_head.cu.o $B/optimizer.cu.o $d/composite_fwd.o $d/composite_bwd.o $d/feature_bwd.o -gencode arch=compute_90a,code=sm_90a -cudart static
  echo "built $n ($f)"; grep -h "error" $d/*.log || true
done
