// TEST INFRASTRUCTURE ONLY: the oracle-backed host pipeline of cpu_backend.cpp (tests/hostsim) with an index of
// homopolymer-compressed minimizers (-H).  cpu_backend.cpp is compiled unchanged inside this file, with two names
// redirected by the preprocessor:
//   wmo_sketch -> wmt_sketch_kind: the oracle's HPC sketch (oracle/wm_oracle_hpc.c) for the reference and the reads;
//   map_batch  -> wmt_map_batch_hpc: the product's orchestration (host_map.cpp) on a copy of the index that carries
//                 WM_I_HPC, through a backend wrapper that adds every minimizer's span to the seeding results (the
//                 GPU backend reports them with an HPC index; the stage-1 divergence estimate averages them).
// tests/test_hpc_cpu.py builds it with the product's host sources into a library of its own.
#include "../../winnowmap_b200/csrc/host_backend.h"

extern "C" {
long wmt_sketch_kind(const char *str, int len, int w, int k, uint32_t rid, const void *bf, uint64_t *out_xy, long max_out);
long wmo_sketch_hpc(const char *str, int len, int w, int k, uint32_t rid, const void *bf, uint64_t *out_xy, long max_out);
}
static void wmt_map_batch_hpc(wmh::Backend *be, const wm_host_idx *mi, const wm_mapopt_t *opt, const std::vector<const wm_read*> &reads,
                              std::vector<std::vector<wm_reg1_t>> &regs, std::vector<int> &rep_len, std::vector<int> &frag_gap, int n_threads,
                              wmh::MapStats *stats);

#define wmo_sketch wmt_sketch_kind
#define map_batch wmt_map_batch_hpc
#include "cpu_backend.cpp"
#undef map_batch
#undef wmo_sketch

extern "C" long wmt_sketch_kind(const char *str, int len, int w, int k, uint32_t rid, const void *bf, uint64_t *out_xy, long max_out)
{
	return wmo_sketch_hpc(str, len, w, k, rid, bf, out_xy, max_out);
}

namespace {
// forwards to the oracle backend and fills SeedOut::mz_span: the spans of the minimizers it sketched, in its order
class SpanBackend : public wmh::Backend {
public:
	wmh::Backend *in; const wm_host_idx *mi; void *bloom;
	std::vector<const wm_read*> reads;
	std::vector<std::vector<uint8_t>> spans;
	void begin_batch(const std::vector<const wm_read*> &r) override { reads = r; in->begin_batch(r); }
	void end_batch() override { in->end_batch(); }
	void seed_chain(const std::vector<wmh::SeedTask> &tasks, const int32_t *mask_pool, const wm_pair_t *pre_pool, const wmh::ChainParams cp[2],
	                int max_occ, std::vector<wmh::SeedOut> &out) override
	{
		in->seed_chain(tasks, mask_pool, pre_pool, cp, max_occ, out);
		const int n = (int)tasks.size();
		spans.assign(n, {});
		#pragma omp parallel for schedule(dynamic, 4)
		for (int i = 0; i < n; ++i) {
			const wmh::SeedTask &t = tasks[i];
			if (t.flags & wmh::SEED_NO_SKETCH) continue;
			std::string s(reads[t.win.read]->seq.data() + t.win.wb, t.win.wl); // the slice cpu_backend.cpp sketches
			if (t.flags & wmh::SEED_MASKED)
				for (int m = 0; m < t.n_mask; ++m)
					for (int p = mask_pool[2 * (t.mask_off + m)]; p < mask_pool[2 * (t.mask_off + m) + 1]; ++p) s[p] = 'N';
			std::vector<uint64_t> mv((size_t)2 * (s.size() / 2 + 64));
			const long nm = wmo_sketch_hpc(s.data(), (int)s.size(), mi->w, mi->k, 0, bloom, mv.data(), (long)mv.size() / 2);
			spans[i].resize(nm + 1);
			for (long m = 0; m < nm; ++m) spans[i][m] = (uint8_t)(mv[2 * m] & 0xff);
		}
		for (int i = 0; i < n; ++i)
			if (!spans[i].empty()) out[i].mz_span = spans[i].data();
	}
	void run_dp(const std::vector<wmh::DpJob> &jobs, const std::vector<wmh::MapWin> &wins, const wmh::DpScoring &sc, std::vector<wmh::DpRes> &res) override
	{ in->run_dp(jobs, wins, sc, res); }
	void run_ll(const std::vector<wmh::LlJob> &jobs, const std::vector<wmh::MapWin> &wins, const wmh::DpScoring &sc, std::vector<wmh::LlRes> &res) override
	{ in->run_ll(jobs, wins, sc, res); }
};
} // namespace

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
