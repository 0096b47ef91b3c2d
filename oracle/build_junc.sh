#!/usr/bin/env bash
# TEST INFRASTRUCTURE ONLY -- never linked, imported or executed by the product path.
#
# oracle/libwm_oracle_junc.so: the junction annotation restated (wm_oracle_junc.c).
#
# Where the reference's sources lie under $REF (default /root/reference) and build_ref.sh has built oracle/_ref/, also the
# reference's own BED reader, which needs one more documented patch: mm_idx_read_bed (src/index.c:690) reads lines into a
# kstring_t of mmpriv.h's layout (unsigned l, m; src/mmpriv.h:39-44), but the line reader it calls, ks_getuntil2, is compiled
# in bseq.c with kseq.h's layout (size_t l, m; src/kseq.h:89-94).  The reader then takes the buffer's capacity for its
# pointer, and every run with --junc-bed crashes before the first line is parsed.  The patch gives that one local variable
# kseq.h's layout; nothing else changes.  Products (git-ignored, under oracle/_ref/):
#   build/index_junc.c        the patched copy (an output file: no reference source is committed)
#   winnowmap_junc            build_ref.sh's oracle with the patched index.o (the junction goldens come from it)
#   libref_harness_junc.so    mm_idx_bed_read / mm_idx_bed_junc of the patched index.o (ref_harness_junc.cpp)
set -euo pipefail
REF=${REF:-/root/reference}
HERE=$(cd "$(dirname "$0")" && pwd)
/usr/bin/gcc -O2 -g -fPIC -Wall -shared "$HERE/wm_oracle_junc.c" -o "$HERE/libwm_oracle_junc.so"
if [ -d "$REF/src" ] && [ -f "$HERE/_ref/libwinnowmap.a" ] && [ -f "$HERE/_ref/build/main.o" ]; then
  B=$HERE/_ref/build
  CXX=/usr/bin/g++
  FLAGS="-g -Wall -O2 -DOMP_PER_READ_THREADS=1 -DHAVE_KALLOC -fopenmp -std=c++11 -Wno-sign-compare -Wno-write-strings -Wno-unused-but-set-variable -fno-tree-vectorize -w -fPIC -I$REF/src"
  sed -e 's/^\tkstring_t str = {0,0,0};$/\tstruct { size_t l, m; char *s; } str = {0,0,0};/' \
      -e 's/ks_getuntil(ks, KS_SEP_LINE, &str, 0)/ks_getuntil(ks, KS_SEP_LINE, (kstring_t*)\&str, 0)/' "$REF/src/index.c" > "$B/index_junc.c"
  [ "$(grep -c 'struct { size_t l, m; char \*s; } str\|(kstring_t\*)&str' "$B/index_junc.c")" = 2 ] || { echo "[build_junc] patch did not apply" >&2; exit 1; }
  if [ ! -f "$B/index_junc.o" ] || [ "$B/index_junc.c" -nt "$B/index_junc.o" ]; then $CXX -c $FLAGS "$B/index_junc.c" -o "$B/index_junc.o"; fi
  rm -rf "$B/junc_ar" && mkdir -p "$B/junc_ar" && (cd "$B/junc_ar" && ar x "$HERE/_ref/libwinnowmap.a" && cp "$B/index_junc.o" index.o)
  rm -f "$HERE/_ref/libwinnowmap_junc.a" && ar -csr "$HERE/_ref/libwinnowmap_junc.a" "$B"/junc_ar/*.o
  $CXX -g -O2 -fopenmp "$B/main.o" "$HERE/_ref/libwinnowmap_junc.a" -o "$HERE/_ref/winnowmap_junc" -lm -lz -lpthread
  $CXX -O2 -fopenmp -std=c++11 -w -fPIC -shared -DHAVE_KALLOC -I"$REF/src" "$HERE/ref_harness_junc.cpp" \
    "$HERE/_ref/libwinnowmap_junc.a" -o "$HERE/_ref/libref_harness_junc.so" -lm -lz -lpthread
fi
