#!/bin/bash
# Build libreagent_b200.so in-tree for sm_90a (H100).  Usage: build.sh [extra nvcc flags]
set -euo pipefail
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
OUT=../libreagent_b200.so
SRCS=$(ls rb200_*.cu)
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC"
mkdir -p build
objs=""
pids=""
for s in $SRCS; do
  o=build/${s%.cu}.o
  objs="$objs $o"
  if [ ! -f "$o" ] || [ "$s" -nt "$o" ] || [ -n "$(find . ../../include -maxdepth 1 \( -name '*.cuh' -o -name '*.h' \) -newer "$o" 2>/dev/null)" ]; then
    $NVCC $FLAGS "$@" -c "$s" -o "$o" &
    pids="$pids $!"
  fi
done
for p in $pids; do wait $p; done
cobjs=""
for s in $(ls rb200_*.c 2>/dev/null); do
  o=build/${s%.c}.o
  gcc -O3 -fPIC -std=c11 -c "$s" -o "$o"
  cobjs="$cobjs $o"
done
$NVCC -shared -o $OUT $objs $cobjs -lcudart
echo "built $(realpath $OUT)"
