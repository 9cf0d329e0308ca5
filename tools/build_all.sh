#!/bin/bash
# Developer aid: build librfid_b200.so and the phase-profile variant; fails loudly.
set -e
cd "$(dirname "$0")/.."
python gen2_uhf_rfid_reader_b200/build.py | grep -A3 "rx_pack_kernel" | grep "Used" || true
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -fmad=false -Xcompiler -fPIC,-fvisibility=hidden -shared -diag-suppress 550 -DRFID_B200_PHASE_PROFILE -o gen2_uhf_rfid_reader_b200/librfid_b200_prof.so gen2_uhf_rfid_reader_b200/csrc/rfid_b200.cu
echo BUILD_OK
