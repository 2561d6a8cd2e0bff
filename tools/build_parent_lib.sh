#!/bin/bash
# Development: build libfqb200.so from another git revision with build.py's nvcc flags, for the A/B comparisons of the
# bench tools (tools/fly_bits_bench.py --parent-lib).  The output directory is git-ignored.
#   tools/build_parent_lib.sh [REVISION (default HEAD~1)] [OUTPUT (default tools/_variants/libfqb200_parent.so)]
set -e
cd "$(dirname "$0")/.."
rev=${1:-HEAD~1}
out=${2:-tools/_variants/libfqb200_parent.so}
flags=$(python -c 'import runpy; print(" ".join(runpy.run_path("cnn-quantization_b200/build.py")["NVCC_FLAGS"]))')
src=$(mktemp -d)
trap 'rm -rf "$src"' EXIT
git archive "$rev" cnn-quantization_b200/csrc include | tar -x -C "$src"
mkdir -p "$(dirname "$out")"
${NVCC:-nvcc} $flags -o "$out" "$src/cnn-quantization_b200/csrc/fqb200.cu"
echo "$out ($(git rev-parse --short "$rev"))"
