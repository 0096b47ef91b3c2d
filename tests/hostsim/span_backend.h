// TEST INFRASTRUCTURE ONLY: a backend wrapper that forwards to the oracle backend and fills SeedOut::mz_span with the
// spans of the minimizers it sketched, in its order (the GPU backend reports them with an HPC index; the stage-1
// divergence estimate averages them).  Shared by hpc_backend.cpp and tee_backend.cpp.
#pragma once
#include <string>
#include <vector>
#include "../../winnowmap_b200/csrc/host_backend.h"

extern "C" long wmo_sketch_hpc(const char *str, int len, int w, int k, uint32_t rid, const void *bf, uint64_t *out_xy, long max_out);

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
