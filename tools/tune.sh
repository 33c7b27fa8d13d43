#!/bin/bash
# Build variants of libcpd_b200.so with other tunables into build/variants/ (git-ignored).
# usage: tools/tune.sh name "-DCPD_RI1=8 ..." [name flags]...
ROOT=$(cd "$(dirname "$0")/.." && pwd)
mkdir -p "$ROOT/build/variants"
while [ $# -ge 2 ]; do
  name=$1; flags=$2; shift 2
  nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -lineinfo -Xcompiler -fPIC -shared \
       -I"$ROOT/include" -I"$ROOT/probreg_b200/csrc" $flags -Xptxas -v \
       -o "$ROOT/build/variants/lib_$name.so" "$ROOT/probreg_b200/csrc/cpd_b200.cu" -ldl 2>&1 \
       | grep -A2 "pass[12]_kernel" | grep -E "registers" | tr '\n' ' '
  echo " <- $name ($flags)"
done
