#!/bin/bash
# Build a kernel variant into tools/ab/lib_<name>.so without touching the product library:
#   tools/build_variant.sh v30 [extra nvcc flags]     (source: tools/ab/<name>.cuh, or the product header + flags)
set -e
cd "$(dirname "$0")/.."
name=$1; shift
tmp=$(mktemp -d /tmp/abXXXX)
mkdir -p $tmp/pkg/csrc
ln -s $PWD/include $tmp/include
cp bigclam_apachespark_b200/csrc/bigclam_capi.cu bigclam_apachespark_b200/csrc/initf_gpu.cu bigclam_apachespark_b200/csrc/edgelist.cpp bigclam_apachespark_b200/csrc/initf.cpp $tmp/pkg/csrc/
# kernel header: tools/ab/<name>.cuh when it exists, else the product one (variants made of -D flags only)
if test -f tools/ab/$name.cuh; then cp tools/ab/$name.cuh $tmp/pkg/csrc/bigclam_kernels.cuh; else cp bigclam_apachespark_b200/csrc/bigclam_kernels.cuh $tmp/pkg/csrc/; fi
cp bigclam_apachespark_b200/csrc/bigclam_sparse.cuh bigclam_apachespark_b200/csrc/bigclam_tile.cuh $tmp/pkg/csrc/
/usr/local/cuda/bin/nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -ccbin /usr/bin/g++ \
    -Xcompiler -fPIC,-O3 -Xptxas -v --expt-relaxed-constexpr "$@" -shared -o tools/ab/lib_$name.so \
    $tmp/pkg/csrc/bigclam_capi.cu $tmp/pkg/csrc/initf_gpu.cu $tmp/pkg/csrc/edgelist.cpp $tmp/pkg/csrc/initf.cpp 2> tools/ab/build_$name.log
grep -A3 "step_kernelILi4ELi[24]ELb0ELb0\|tile_step_kernelILb0ELb0" tools/ab/build_$name.log | grep -E "Used|spill" | head -8
rm -rf $tmp
