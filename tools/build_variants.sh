#!/bin/bash
# Development: A/B builds of libfqb200.so with different bulk-ring shapes (select one with FQB200_LIB=<path>).
#   tools/build_variants.sh "2 5 1 2" "4 6 1 1"      # each tuple = FQB_STAGE_VEC FQB_STAGES FQB_BULK_SPLIT FQB_BULK_CTAS
set -e
cd "$(dirname "$0")/.."
mkdir -p tools/_variants   # git-ignored
for v in "$@"; do
  set -- $v
  out=tools/_variants/libfqb200_v$1_k$2_s$3_c${4:-1}${5:+_$5}.so
  ${NVCC:-nvcc} -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -fmad=false -std=c++17 -shared -Xcompiler -fPIC \
    -DFQB_STAGE_VEC=$1 -DFQB_STAGES=$2 -DFQB_BULK_SPLIT=$3 -DFQB_BULK_CTAS=${4:-1} ${5:+-D$5} -o $out cnn-quantization_b200/csrc/fqb200.cu &
done
wait
ls -la tools/_variants
