#!/bin/bash
# Builds the microbenchmarks of the latency / bandwidth floors the streaming kernel is built on (DESIGN.md section 5.4) (binaries are git-ignored).
cd "$(dirname "$0")"
for f in *_bench.cu; do
  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -lineinfo -o "${f%.cu}" "$f" || exit 1
done
