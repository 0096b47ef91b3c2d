#!/usr/bin/env bash
# TEST INFRASTRUCTURE ONLY -- never linked, imported or executed by the product path.
#
# oracle/libwm_oracle_hpc.so: the CPU oracle (wm_oracle.c) plus its homopolymer-compressed sketch (wm_oracle_hpc.c).
# Where the reference's sources lie under $REF (default /root/reference) and build_ref.sh has built oracle/_ref/, also
# oracle/_ref/libref_harness_hpc.so: the wrappers of ref_harness.cpp plus the reference's HPC sketch and -H index.
set -euo pipefail
REF=${REF:-/root/reference}
HERE=$(cd "$(dirname "$0")" && pwd)
/usr/bin/gcc -O2 -g -fPIC -Wall -Wno-unused-function -ffp-contract=off -shared "$HERE/wm_oracle.c" "$HERE/wm_oracle_hpc.c" \
  -o "$HERE/libwm_oracle_hpc.so" -lm
if [ -d "$REF/src" ] && [ -f "$HERE/_ref/libwinnowmap.a" ]; then
  /usr/bin/g++ -O2 -fopenmp -std=c++11 -w -fPIC -shared -DHAVE_KALLOC -I"$REF/src" -I"$HERE" "$HERE/ref_harness_hpc.cpp" \
    "$HERE/_ref/libwinnowmap.a" -o "$HERE/_ref/libref_harness_hpc.so" -lm -lz -lpthread
fi
