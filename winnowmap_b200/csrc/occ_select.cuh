#pragma once
#include <stdint.h>
#include <cuda_runtime.h>

// The rank-th smallest (0-based) of the n occurrence counts pos_off[i+1] - pos_off[i] of a device CSR (n + 1 offsets);
// rank < n.  Exact for every count value and tie pattern; blocks until the value is known.
uint32_t wm_occ_select_dev(const uint64_t *d_pos_off, int64_t n, uint64_t rank, cudaStream_t st);
