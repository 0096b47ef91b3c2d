#pragma once
#include "wm_common.cuh"
#include "sketch.cuh"

// Device-side index construction (index_dev.cu): sorts the n (minimizer, position) pairs of d_a (consumed) by minimizer hash,
// positions ascending, and builds keys / pos_off / pos on the device.
void wm_index_build_dev(wm128_dev *d_a, int64_t n, int k, uint64_t **d_keys_out, uint64_t **d_pos_off_out, uint64_t **d_pos_out, int64_t *n_keys_out, cudaStream_t st);
// The stable LSD radix sort of wm_index_build_dev on bare 64-bit keys (csrc/topfreq.cu): sorts the n keys of a by bits
// [bit_lo, bit_hi), 8 bits per pass, with b as the second buffer; returns a or b, whichever holds the result.
template <typename T> T *wm_lsd_sort(T *a, T *b, int64_t n, int bit_lo, int bit_hi, cudaStream_t st);
