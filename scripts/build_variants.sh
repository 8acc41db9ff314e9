#!/bin/bash
# experimental builds of the library with -D switches -> powdr_b200/_lib/variants/<name>.so (timed by scripts/p2_variants.py,
# scripts/leaf_variants.py on the GPU).  usage: build_variants.sh name1:"-DFOO -DBAR" name2:"" ...
cd "$(dirname "$0")/.."
mkdir -p powdr_b200/_lib/variants
for spec in "$@"; do
  name="${spec%%:*}"; flags="${spec#*:}"
  /usr/local/cuda/bin/nvcc -std=c++17 -O3 -ldl -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC -shared -ccbin /usr/bin/g++ $flags \
    -o powdr_b200/_lib/variants/$name.so powdr_b200/csrc/capi.cu &
done
wait
ls -la powdr_b200/_lib/variants/
