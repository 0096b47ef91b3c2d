// TEST INFRASTRUCTURE ONLY: the oracle-backed host pipeline of cpu_backend.cpp (tests/hostsim) with an index of
// homopolymer-compressed minimizers (-H).  cpu_backend.cpp is compiled unchanged inside this file:
//   wmo_sketch is redirected by the preprocessor to wmt_sketch_kind: the oracle's HPC sketch (oracle/wm_oracle_hpc.c) for
//              the reference and the reads;
//   batches are mapped by wmt_map_batch_hpc: the product's orchestration (host_map.cpp) on a copy of the index that carries
//              WM_I_HPC, through a backend wrapper that adds every minimizer's span to the seeding results (the GPU backend
//              reports them with an HPC index; the stage-1 divergence estimate averages them).
// tests/test_hpc_cpu.py builds it with the product's host sources into a library of its own.
#include "../../winnowmap_b200/csrc/host_backend.h"

extern "C" {
long wmt_sketch_kind(const char *str, int len, int w, int k, uint32_t rid, const void *bf, uint64_t *out_xy, long max_out);
long wmo_sketch_hpc(const char *str, int len, int w, int k, uint32_t rid, const void *bf, uint64_t *out_xy, long max_out);
}

#define wmo_sketch wmt_sketch_kind
#include "cpu_backend.cpp"
#undef wmo_sketch

extern "C" long wmt_sketch_kind(const char *str, int len, int w, int k, uint32_t rid, const void *bf, uint64_t *out_xy, long max_out)
{
	return wmo_sketch_hpc(str, len, w, k, rid, bf, out_xy, max_out);
}

#include "span_backend.h"

static void wmt_map_batch_hpc(wmh::Backend *be, const wm_host_idx *mi, const wm_mapopt_t *opt, const std::vector<const wm_read*> &reads,
                              std::vector<std::vector<wm_reg1_t>> &regs, std::vector<int> &rep_len, std::vector<int> &frag_gap, int n_threads,
                              wmh::MapStats *stats)
{
	wm_host_idx H = *mi;
	H.flag = WM_I_HPC;
	SpanBackend sb;
	sb.in = be, sb.mi = &H, sb.bloom = static_cast<CpuBackend*>(be)->bloom;
	wmh::map_batch(&sb, &H, opt, reads, regs, rep_len, frag_gap, n_threads, stats);
}
static const bool g_hpc_mapping = (g_map_batch = wmt_map_batch_hpc, true); // every run of this library maps through an HPC index
