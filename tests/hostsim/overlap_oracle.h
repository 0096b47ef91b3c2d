// TEST INFRASTRUCTURE ONLY: the oracle backend of cpu_backend.cpp with the seed filter of self and all-vs-all mapping (-D,
// --dual=no, -X) and single-strand mapping (--for-only, --rev-only).  Included after cpu_backend.cpp (overlap_backend.cpp,
// overlap_tee.cpp).
//
// The filter is restated here from skip_seed (src/map.c:132-154) as the reference computes it: strcmp of the read's name
// against the index names, the window length as qlen.  It does not use the SKIP_* bits or the name ranks the orchestrator
// hands to the device, so that it checks the product's rank reduction as well.
#pragma once

extern "C" {
const uint64_t *wmo_idx_get(const void *ix, uint64_t minier, int *n);
}

class OverlapCpuBackend : public CpuBackend {
public:
	int64_t flag = 0; // the mapping flags

	// skip_seed (src/map.c:132-154): 1 = drop the occurrence r of a minimizer at q_pos; *is_self: MM_SEED_SELF
	int skip_seed(uint64_t r, uint32_t q_pos, const char *qname, int qlen, int *is_self) const
	{
		*is_self = 0;
		if (qname && (flag & (WM_F_NO_DIAG | WM_F_NO_DUAL))) {
			const uint32_t rid = (uint32_t)(r >> 32);
			const int cmp = strcmp(qname, hidx->name[rid].c_str());
			if ((flag & WM_F_NO_DIAG) && cmp == 0 && (int)hidx->len[rid] == qlen) {
				if ((uint32_t)r >> 1 == q_pos >> 1) return 1;
				if ((r & 1) == (q_pos & 1)) *is_self = 1;
			}
			if ((flag & WM_F_NO_DUAL) && cmp > 0) return 1;
		}
		if (flag & (WM_F_FOR_ONLY | WM_F_REV_ONLY)) {
			if ((r & 1) == (q_pos & 1)) { if (flag & WM_F_REV_ONLY) return 1; }
			else if (flag & WM_F_FOR_ONLY) return 1;
		}
		return 0;
	}

	// collect_matches + collect_seed_hits (src/map.c:97-130, :222-254) over the oracle's index, with the filter; mz_pos as
	// CpuBackend reports it
	void collect(const uint64_t *mv, long nm, int qlen, const char *qname, int max_occ, std::vector<wm_pair_t> &a, int *rep_len, std::vector<uint32_t> &mzp) const
	{
		int rep_st = 0, rep_en = 0, rl = 0;
		a.clear(); mzp.assign(nm, 0);
		for (long i = 0; i < nm; ++i) {
			const uint64_t px = mv[2 * i], py = mv[2 * i + 1];
			const uint32_t q_pos = (uint32_t)py, q_span = px & 0xff;
			int t;
			const uint64_t *cr = wmo_idx_get(idx, px >> 8, &t);
			mzp[i] = q_pos >> 1;
			if (t >= max_occ) {
				const int en = (int)(q_pos >> 1) + 1, st = en - (int)q_span;
				if (st > rep_en) { rl += rep_en - rep_st; rep_st = st, rep_en = en; }
				else rep_en = en;
				continue;
			}
			mzp[i] |= 0x80000000u;
			const bool tandem = (i > 0 && px >> 8 == mv[2 * (i - 1)] >> 8) || (i < nm - 1 && px >> 8 == mv[2 * (i + 1)] >> 8);
			for (int k = 0; k < t; ++k) {
				const uint64_t r = cr[k];
				int is_self;
				if (skip_seed(r, q_pos, qname, qlen, &is_self)) continue;
				wm_pair_t p;
				const int32_t rpos = (uint32_t)r >> 1;
				if ((r & 1) == (q_pos & 1)) {
					p.x = (r & 0xffffffff00000000ULL) | (uint32_t)rpos;
					p.y = (uint64_t)q_span << 32 | q_pos >> 1;
				} else {
					p.x = 1ULL << 63 | (r & 0xffffffff00000000ULL) | (uint32_t)rpos;
					p.y = (uint64_t)q_span << 32 | (uint32_t)(qlen - ((q_pos >> 1) + 1 - q_span) - 1);
				}
				p.y |= (uint64_t)(py >> 32) << 48;
				if (tandem) p.y |= WM_SEED_TANDEM;
				if (is_self) p.y |= WM_SEED_SELF;
				a.push_back(p);
			}
		}
		rl += rep_en - rep_st;
		*rep_len = rl;
		if (!a.empty()) wmo_radix_sort_128x(a.data(), (long)a.size());
	}

	void seed_chain(const std::vector<SeedTask> &tasks, const int32_t *mask_pool, const wm_pair_t *pre_pool, const ChainParams cp[2], int max_occ, std::vector<SeedOut> &out) override
	{
		const int n = (int)tasks.size();
		out.assign(n, SeedOut());
		mz_pos.assign(n, {}); us.assign(n, {}); bs.assign(n, {}); n_anchors.assign(n, 0);
		#pragma omp parallel for schedule(dynamic, 4)
		for (int i = 0; i < n; ++i) {
			const SeedTask &t = tasks[i];
			const wm_read *rd = reads[t.win.read];
			std::vector<wm_pair_t> a;
			int rep_len = 0;
			if (!(t.flags & SEED_NO_SKETCH)) {
				std::string s(rd->seq.data() + t.win.wb, t.win.wl);
				if (t.flags & SEED_MASKED)
					for (int m = 0; m < t.n_mask; ++m)
						for (int p = mask_pool[2 * (t.mask_off + m)]; p < mask_pool[2 * (t.mask_off + m) + 1]; ++p) s[p] = 'N';
				std::vector<uint64_t> mv((size_t)2 * (s.size() / 2 + 64));
				const long nm = wmo_sketch(s.data(), (int)s.size(), hidx->w, hidx->k, 0, bloom, mv.data(), (long)mv.size() / 2);
				collect(mv.data(), nm, t.win.wl, rd->has_name ? rd->name.c_str() : 0, max_occ, a, &rep_len, mz_pos[i]);
			}
			if (t.n_pre > 0) { // [pre ; seeds] then the unstable sort again (src/map.c:818-831)
				std::vector<wm_pair_t> w(pre_pool + t.pre_off, pre_pool + t.pre_off + t.n_pre);
				w.insert(w.end(), a.begin(), a.end());
				if (!a.empty()) wmo_radix_sort_128x(w.data(), (long)w.size());
				a.swap(w);
			}
			n_anchors[i] = (int64_t)a.size();
			const ChainParams &c = cp[t.chain_set];
			us[i].resize(a.size() + 1); bs[i].resize(a.size() + 1);
			long nb = 0;
			const int nu = wmo_chain_dp(c.max_dist_x, c.min_dist_x, c.max_dist_y, c.bw, c.max_skip, c.max_iter, c.min_cnt, c.min_sc, c.gap_scale, (long)a.size(),
			                            (uint64_t*)a.data(), us[i].data(), (uint64_t*)bs[i].data(), &nb);
			SeedOut &o = out[i];
			o.rep_len = (t.flags & SEED_NO_SKETCH) ? 0 : rep_len;
			o.n_mz = (int32_t)mz_pos[i].size(); o.mz_pos = mz_pos[i].data();
			o.n_u = nu; o.u = us[i].data(); o.n_b = nb; o.b = bs[i].data();
		}
	}
};

