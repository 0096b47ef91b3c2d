// TEST INFRASTRUCTURE ONLY: crafted seed_chain calls with the seed filter of -D / --dual=no / -X / --for-only / --rev-only
// through the tee of tee_backend.cpp (compiled unchanged into this file).  The served side is the CUDA backend, which gets
// the SKIP_* bits and name ranks the orchestrator derives from the flags (skip_bits); the expected side is the filtering
// oracle backend of overlap_oracle.h, which works from strcmp of the names, the mapping flags and the window length.  Every
// field of every task is compared, the anchors of the chains with their MM_SEED_SELF bits included.
//
// Built by tests/test_gpu_overlap_tee.py against libwinnowmap_b200.so, like tee_backend.cpp.
#include "tee_backend.cpp"
#include "overlap_oracle.h"

// One stage-1-shaped seed_chain call over query windows (rows: read, wb, wl) of named reads (names[i] == NULL: a read
// without a name) on chain set 0, under the mapping flags `flag`.  dev_kind 0: the CUDA backend serves; 1: a second
// filtering oracle backend (the crafted batch checked without a device).  The report adds the counters overlap.self_anchors
// (chained anchors with MM_SEED_SELF), overlap.empty_tasks (windows left without an anchor) and overlap.tasks_filtered.
extern "C" int wmt_tee_overlap_seed_chain(const char *ref_fn, int k, int w, int dev_kind, int64_t flag, int n_reads, const char *const *names,
                                          const char *seq, const int64_t *read_off, int n1, const int32_t *rows1, const int32_t *cp_i,
                                          const float *cp_f, int max_occ, const char *report_fn)
{
	TeeRun R;
	int rc = R.init(ref_fn, 0, k, w, 0, dev_kind == 0 ? 0 : 1, 0, 0);
	if (rc < 0) return rc;
	OverlapCpuBackend ora, ora2;
	for (OverlapCpuBackend *o : {&ora, &ora2}) o->flag = flag, o->hidx = &R.X.H, o->bloom = R.X.bloom, o->idx = R.cpu_e.idx;
	R.tee.ora = &ora, R.tee.fetcher = &ora;
	if (dev_kind != 0) R.tee.dev = &ora2;
	std::vector<wm_read> rs(n_reads);
	std::vector<const wm_read*> rp(n_reads);
	for (int i = 0; i < n_reads; ++i) {
		rs[i].has_name = names[i] != 0, rs[i].name = names[i] ? names[i] : "";
		rs[i].seq.assign(seq + read_off[i], read_off[i + 1] - read_off[i]), rp[i] = &rs[i];
	}
	ChainParams cp[2];
	for (int s = 0; s < 2; ++s) {
		const int32_t *c = cp_i + 8 * s;
		cp[s].max_dist_x = c[0], cp[s].min_dist_x = c[1], cp[s].max_dist_y = c[2], cp[s].bw = c[3];
		cp[s].max_skip = c[4], cp[s].max_iter = c[5], cp[s].min_cnt = c[6], cp[s].min_sc = c[7], cp[s].gap_scale = cp_f[s];
	}
	R.tee.begin_batch(rp);
	std::vector<SeedTask> t1(n1);
	int64_t n_filtered = 0;
	for (int i = 0; i < n1; ++i) {
		const int32_t *r = rows1 + 3 * i;
		SeedTask &t = t1[i];
		t.win = MapWin{ r[0], r[1], r[2] }, t.flags = 0, t.chain_set = 0, t.n_mask = 0, t.mask_off = 0, t.n_pre = 0, t.pre_off = 0;
		t.skip = skip_bits(&R.X.H, flag, &rs[r[0]], &t.name_lt);
		n_filtered += t.skip != 0;
	}
	std::vector<SeedOut> o1;
	int32_t no_mask[2] = {0, 0};
	R.tee.seed_chain(t1, no_mask, 0, cp, max_occ, o1);
	int64_t n_self = 0, n_empty = 0;
	for (int i = 0; i < n1; ++i) {
		for (int64_t j = 0; j < o1[i].n_b; ++j) n_self += (o1[i].b[j].y & WM_SEED_SELF) != 0;
		n_empty += ora.n_anchors[i] == 0;
	}
	R.tee.add("overlap.self_anchors", n_self); R.tee.add("overlap.empty_tasks", n_empty); R.tee.add("overlap.tasks_filtered", n_filtered);
	R.tee.end_batch();
	return R.finish(report_fn);
}
