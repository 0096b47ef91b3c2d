#pragma once
#include "host_backend.h"

namespace wmh {
// Uploads the flattened index (sorted unique minimizer hashes + CSR occurrence lists + packed reference +
// down-weight filter bits) to `device` and returns the CUDA backend.  Exits with a message if no device.
Backend *gpu_backend_create(const wm_host_idx *hidx, const uint64_t *keys, int64_t n_keys, const uint64_t *pos_off, const uint64_t *pos,
                            uint64_t bloom_bits, const uint8_t *bloom_table, int device);
// the same with the index arrays already on the device (ownership passes to the backend)
Backend *gpu_backend_create_dev(const wm_host_idx *hidx, uint64_t *d_keys, int64_t n_keys, uint64_t *d_poff, uint64_t *d_pos,
                                uint64_t bloom_bits, const uint8_t *bloom_table, int device);
// the index arrays the backend was created with (not those of the index gpu_backend_bind points it at)
void gpu_backend_index_arrays(Backend *be, const uint64_t **d_keys, const uint64_t **d_poff, const uint64_t **d_pos);
// map with the index another backend was created with (a part of the same multi-part index); streams and workspaces stay
void gpu_backend_bind(Backend *lane, const Backend *src);
// the junction intervals of hidx (read_bed_junc / set_junc) on the device, for the index `be` was created with
void gpu_backend_set_junc(Backend *be, const wm_host_idx *hidx);
void gpu_backend_destroy(Backend *be);
}

namespace wmh {
Backend *gpu_backend_clone(Backend *base, int n_lanes);
void gpu_backend_set_budget(Backend *be, size_t bytes);
size_t gpu_backend_get_budget(Backend *be);
void gpu_backend_trim_pool(int device);
}
