#!/usr/bin/env bash
# TEST INFRASTRUCTURE: host sources of the product + the CPU oracle backend -> tests/hostsim/libwm_hostsim.so
set -euo pipefail
HERE=$(cd "$(dirname "$0")" && pwd); ROOT=$HERE/../..
CS=$ROOT/winnowmap_b200/csrc
/usr/bin/g++ -std=c++17 -O2 -g -fPIC -shared -fopenmp -ffp-contract=off -I${CUDA_HOME:-/usr/local/cuda}/include ${WMT_EXTRA:-} \
  $HERE/parts_backend.cpp $HERE/kernel_emul.cpp $CS/host_*.cpp \
  -x c $ROOT/oracle/wm_oracle.c -x c $ROOT/oracle/wm_oracle_occ.c -o $HERE/libwm_hostsim.so -lz -lm -lpthread
