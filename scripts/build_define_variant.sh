#!/usr/bin/env bash
# Development aid: build the WORKING TREE's libkge_b200.so with extra nvcc flags into _variants/libkge_<name>.so
# (separate object directory, the product build is untouched), e.g. a profiling build without the gradient scatter:
#   scripts/build_define_variant.sh noscatter -DKGE_PROFILE_NOSCATTER
#   KGE_B200_LIB=$PWD/_variants/libkge_noscatter.so python scripts/kbench.py cfg2
set -euo pipefail
name=${1:?variant name}; shift
root=$(git rev-parse --show-toplevel)
wt=$(mktemp -d /tmp/kge_defvariant.XXXXXX)
trap 'rm -rf "$wt"' EXIT
mkdir -p "$wt/ampligraph_b200" "$root/_variants"
cp -r "$root/include" "$wt/include"
cp -r "$root/ampligraph_b200/csrc" "$wt/ampligraph_b200/csrc"
rm -rf "$wt/ampligraph_b200/csrc/_build"
make -C "$wt/ampligraph_b200/csrc" -j"$(nproc)" NVCCFLAGS="-O3 -std=c++17 -lineinfo -gencode arch=compute_90a,code=sm_90a -Xcompiler -fPIC -Xptxas -v --fmad=true $*" >/dev/null
cp "$wt/ampligraph_b200/libkge_b200.so" "$root/_variants/libkge_$name.so"
echo "built working tree with [$*] -> _variants/libkge_$name.so"
