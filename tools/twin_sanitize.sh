#!/bin/bash
# The engine's two state machines (tests/host_twin: af_lane.cuh and af_core.cuh compiled for the host) under
# AddressSanitizer + UndefinedBehaviorSanitizer, driven by the fuzz campaign: the CPU-side counterpart of
# compute-sanitizer's memcheck for the code the kernels share with the twin (every table access of a replica goes
# through the same index arithmetic; the twin's "shared memory" and global tier are heap blocks of exactly the sizes
# make_cfg computes, so an index past a region's end is a heap-buffer-overflow here).
#   bash tools/twin_sanitize.sh [count]
cd "$(dirname "$0")/.." || exit 1
n=${1:-200}
so=/tmp/libaf_host_twin_asan.so
g++ -O1 -g -fsanitize=address,undefined -fno-omit-frame-pointer -ffp-contract=off -std=c++17 -fPIC -shared -x c++ \
    -o $so tests/host_twin/af_host_twin.cpp || exit 1
so2=/tmp/libaf_split_twin_asan.so
g++ -O1 -g -fsanitize=address,undefined -fno-omit-frame-pointer -ffp-contract=off -std=c++17 -fPIC -shared -x c++ \
    -o $so2 tests/host_twin/af_split_twin.cpp || exit 1
export LD_PRELOAD=$(gcc -print-file-name=libasan.so):$(gcc -print-file-name=libubsan.so)
export ASAN_OPTIONS=detect_leaks=0:halt_on_error=1 UBSAN_OPTIONS=print_stacktrace=1:halt_on_error=1 AF_TWIN_SO=$so AF_SPLIT_TWIN_SO=$so2
python tools/fuzz_campaign.py --first 1500000 --count $n --jobs 1 --layouts &&
python tools/fuzz_campaign.py --first 1510000 --count $((n / 10)) --jobs 1 --layouts --big &&
python tools/fuzz_campaign.py --first 1520000 --count $((n / 2)) --jobs 1 --engine warp &&
python tools/fuzz_campaign.py --first 1530000 --count $((n / 20)) --jobs 1 --engine warp --big
