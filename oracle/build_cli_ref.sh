#!/usr/bin/env bash
# TEST INFRASTRUCTURE ONLY -- never linked, imported or executed by the product path.
#
# oracle/_ref/winnowmap_cli_dump: the reference's own main.o (built by build_ref.sh into oracle/_ref/build) linked with
# cli_ref_dump.c, whose wrappers record what main() would index and map with instead of doing it (see that file).
# tests/test_cli_options.py compares the product's command-line parser with it.  Skipped where the reference's sources
# or build_ref.sh's objects are absent.
set -euo pipefail
REF=${REF:-/root/reference}
HERE=$(cd "$(dirname "$0")" && pwd)
B=$HERE/_ref/build
OUT=$HERE/_ref/winnowmap_cli_dump
if [ ! -d "$REF/src" ] || [ ! -f "$B/main.o" ] || [ ! -f "$HERE/_ref/libwinnowmap.a" ]; then
  echo "[build_cli_ref] reference objects not present -- skipped" >&2
  exit 0
fi
if [ -f "$OUT" ] && [ "$OUT" -nt "$HERE/cli_ref_dump.c" ] && [ "$OUT" -nt "$HERE/cli_dump.h" ] && [ "$OUT" -nt "$B/main.o" ]; then exit 0; fi
WRAP=""
for f in sched_getaffinity mm_idx_reader_open mm_idx_reader_read mm_idx_reader_eof mm_idx_reader_close mm_idx_destroy mm_idx_stat \
         mm_idx_bed_read mm_mapopt_update mm_map_file mm_map_file_frag mm_split_merge mm_write_sam_hdr; do
  WRAP="$WRAP -Wl,--wrap=$f"
done
/usr/bin/g++ -O2 -w -x c++ -std=c++11 -c -I"$REF/src" -I"$HERE" "$HERE/cli_ref_dump.c" -o "$B/cli_ref_dump.o"
/usr/bin/g++ -fopenmp $WRAP "$B/main.o" "$B/cli_ref_dump.o" "$HERE/_ref/libwinnowmap.a" -o "$OUT" -lm -lz -lpthread
