// TEST INFRASTRUCTURE.  The giant-task chaining kernel's CTA body in its CDNA instantiation (the gap cost of spliced mapping) on the
// emulated CTA of tile_cta_emul.cpp, which is compiled unchanged into this file: its call of wm_chain_fill_tile_cta is redirected to
// wm_chain_fill_tile_cta<true>, and its entry points get a _cdna suffix.  Built like tile_cta_emul.cpp (tests/splice_lib.py).
#include "cuda_emul.h"
#include "wm_common.cuh"
#include "chain_tile.cuh"
#define wm_chain_fill_tile_cta wm_chain_fill_tile_cta<true>
#define wmt_tile_cta wmt_tile_cta_cdna
#define wmt_tile_scan_paths wmt_tile_scan_paths_plain // the scalar path census of the plain gap cost; not used for cDNA
#define wmt_tile_constants wmt_tile_constants_cdna
#include "tile_cta_emul.cpp"
