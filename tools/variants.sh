#!/bin/bash
# Developer aid: build librfid_b200 variants with extra -D flags and time each with tools/quick_bench.py (GPU box).
# usage: tools/variants.sh build "name1:-DX=1" "name2:-DY=2" ...   (here, cross-compiles)
#        tools/variants.sh run 148 1000                             (on the GPU box)
set -e
cd "$(dirname "$0")/.."
CS=gen2_uhf_rfid_reader_b200/csrc
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -fmad=false -Xcompiler -fPIC,-fvisibility=hidden -shared -diag-suppress 550,177"
mkdir -p gpurun_in
if [ "$1" = build ]; then
  shift
  rm -f gpurun_in/librfid_b200_*.so
  for v in "$@"; do
    name="${v%%:*}"; defs="${v#*:}"
    nvcc $FLAGS $defs -o gpurun_in/librfid_b200_$name.so $CS/rfid_b200.cu &
  done
  wait
  ls -la gpurun_in/
else
  shift
  for so in gpurun_in/librfid_b200_*.so; do
    echo "== $so"
    RFID_B200_LIB=$PWD/$so timeout 120 python tools/quick_bench.py "$@" 2>&1 | tail -n +1 | grep -v "^$"
  done
fi
