#!/usr/bin/env bash
# TEST INFRASTRUCTURE ONLY -- never linked, imported or executed by the product path.
#
# oracle/libwm_oracle_sdust.so: the SDUST restatement and the minimizer squeeze of -T (wm_oracle_sdust.c), with the oracle's
# sketch (wm_oracle.c) beside them.  Where the reference's sources lie under $REF (default /root/reference) and build_ref.sh
# has built oracle/_ref/, also oracle/_ref/libref_harness_sdust.so: the reference's own sdust() and mm_dust_minier
# (ref_harness_sdust.cpp).
set -euo pipefail
REF=${REF:-/root/reference}
HERE=$(cd "$(dirname "$0")" && pwd)
/usr/bin/gcc -O2 -g -fPIC -Wall -Wno-unused-function -ffp-contract=off -shared "$HERE/wm_oracle.c" "$HERE/wm_oracle_sdust.c" \
  -o "$HERE/libwm_oracle_sdust.so" -lm
if [ -d "$REF/src" ] && [ -f "$HERE/_ref/libwinnowmap.a" ] && [ -f "$HERE/_ref/build/map_patched.c" ]; then
  /usr/bin/g++ -O2 -fopenmp -std=c++11 -w -fPIC -shared -DHAVE_KALLOC -DOMP_PER_READ_THREADS=1 -I"$REF/src" -I"$HERE/_ref/build" "$HERE/ref_harness_sdust.cpp" \
    "$HERE/_ref/libwinnowmap.a" -o "$HERE/_ref/libref_harness_sdust.so" -lm -lz -lpthread
fi
