#!/bin/bash
# Builds libt2v_b200.so for sm_90a (H100; cross-compiles without a GPU). Usage: csrc/build.sh [extra nvcc flags]
set -e
cd "$(dirname "$0")"
OUT=${T2V_BUILD_OUT:-../t2v_b200/libt2v_b200.so}      # variant builds: T2V_BUILD_OUT=<.so> T2V_BUILD_DIR=<obj dir> build.sh -D...
BUILD=${T2V_BUILD_DIR:-build}
mkdir -p ../t2v_b200 $BUILD
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -lineinfo -O3 -std=c++17 -Xcompiler -fPIC --expt-relaxed-constexpr $@"
objs=""
pids=""
for f in *.cu; do
  o=$BUILD/${f%.cu}.o
  objs="$objs $o"
  if [ ! -f "$o" ] || [ "$f" -nt "$o" ] || [ -n "$(find . -maxdepth 1 -name '*.cuh' -newer "$o")" ] || [ ../../include/t2v_b200.h -nt "$o" ]; then
    $NVCC $FLAGS -c "$f" -o "$o" &
    pids="$pids $!"
  fi
done
for p in $pids; do wait $p; done
$NVCC -shared -o $OUT $objs -gencode arch=compute_90a,code=sm_90a
echo "built $OUT"
