#!/bin/bash
# Build a second copy of the library with extra -D flags for frontend_pow2.cu (A/B timing through B200A_LIB):
#   tools/build_alt.sh alt1 -DB200A_WIN_SMEM=0      -> audio_b200/build/libb200audio_alt1.so
set -e
name=$1; shift
cd "$(dirname "$0")/.."
B=audio_b200/build
nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -Xcompiler -fPIC -Xcompiler -fvisibility=hidden --expt-relaxed-constexpr "$@" -c audio_b200/csrc/frontend_pow2.cu -o $B/frontend_pow2_$name.o
nvcc -gencode arch=compute_90a,code=sm_90a -shared -o $B/libb200audio_$name.so $B/api.o $B/frontend_generic.o $B/frontend_pow2_$name.o $B/resample.o $B/standalone.o
ls -la $B/libb200audio_$name.so
