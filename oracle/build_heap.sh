#!/usr/bin/env bash
# TEST INFRASTRUCTURE ONLY -- never linked, imported or executed by the product path.
#
# oracle/libwm_oracle_heap.so: the restatement of seed collection with --heap-sort=yes (wm_oracle_heap.c), with the oracle's
# sketch and flattened index (wm_oracle.c) beside it.  Where the reference's sources lie under $REF (default /root/reference) and
# build_ref.sh has built oracle/_ref/, also oracle/_ref/libref_harness_heap.so: the reference's own collect_seed_hits_heap and
# collect_seed_hits (ref_harness_heap.cpp).
set -euo pipefail
REF=${REF:-/root/reference}
HERE=$(cd "$(dirname "$0")" && pwd)
/usr/bin/gcc -O2 -g -fPIC -Wall -Wno-unused-function -ffp-contract=off -shared "$HERE/wm_oracle.c" "$HERE/wm_oracle_heap.c" \
  -o "$HERE/libwm_oracle_heap.so" -lm
if [ -d "$REF/src" ] && [ -f "$HERE/_ref/libwinnowmap.a" ] && [ -f "$HERE/_ref/build/map_patched.c" ]; then
  /usr/bin/g++ -O2 -fopenmp -std=c++11 -w -fPIC -shared -DHAVE_KALLOC -DOMP_PER_READ_THREADS=1 -I"$REF/src" -I"$HERE/_ref/build" "$HERE/ref_harness_heap.cpp" \
    "$HERE/_ref/libwinnowmap.a" -o "$HERE/_ref/libref_harness_heap.so" -lm -lz -lpthread
fi
