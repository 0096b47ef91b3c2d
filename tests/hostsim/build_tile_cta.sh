#!/usr/bin/env bash
# TEST INFRASTRUCTURE: the giant-task chaining kernel's CTA body on an emulated CTA -> tests/hostsim/libwm_tilecta.so (needs
# libwm_hostsim.so from build.sh: the fiber runtime).  build_tile_cta.sh CSRC OUT builds it from the product headers in CSRC instead
# (a modified copy) into OUT.
set -euo pipefail
HERE=$(cd "$(dirname "$0")" && pwd)
CSRC=${1:-$HERE/../../winnowmap_b200/csrc}
OUT=${2:-$HERE/libwm_tilecta.so}
[ -f "$HERE/libwm_hostsim.so" ] || "$HERE/build.sh"
/usr/bin/g++ -std=c++17 -O2 -g -fPIC -shared -fvisibility=hidden -ffp-contract=off -I"$CSRC" -I${CUDA_HOME:-/usr/local/cuda}/include \
  "$HERE/tile_cta_emul.cpp" -o "$OUT" -L"$HERE" -l:libwm_hostsim.so -Wl,-rpath,"$HERE"
