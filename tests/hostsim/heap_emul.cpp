// TEST INFRASTRUCTURE.  The device code of --heap-sort=yes (csrc/seed_heap.cuh: wm_heap_replay_task, one warp per task, and
// wm_seed_anchor) compiled for the host on top of cuda_emul.h and run on the software warp of kernel_emul.cpp, so that
// tests/test_heap_cpu.py can check it against the oracle (oracle/wm_oracle_heap.c) without a GPU.
#include <vector>
#include "cuda_emul.h"
#include "../../winnowmap_b200/csrc/seed_heap.cuh"

// One task: query minimizers mz_xy[0 .. n_mz) (x, y pairs) with, per minimizer, cnt (occurrences kept, 0 at or above max_occ),
// list_off (start in pos) and tandem; the index's pos, seq_len and name_rank; skip = (WM_SKIP_* bits, names below the read's), the
// filter running when filter != 0.  a_xy[0 .. n) holds the task's kept anchors in ascending x (any order among equal x) and gets
// the heap's order.  stage != 0 stages the occurrence lists as shared memory would.  Returns what lane 0 returns.
extern "C" long wmt_heap_replay_dev(const uint64_t *mz_xy, int n_mz, const int32_t *cnt, const uint64_t *list_off, const uint8_t *tandem,
                                    const uint64_t *pos, const uint32_t *seq_len, const uint32_t *name_rank, int qlen, uint32_t skip_bits,
                                    uint32_t name_lt, int filter, int stage, uint64_t *a_xy, long n)
{
	std::vector<int64_t> raw_off(n_mz + 1, 0);
	for (int m = 0; m < n_mz; ++m) raw_off[m + 1] = raw_off[m] + cnt[m];
	std::vector<wm128_dev> H(n_mz + 1);
	std::vector<wm_heap_list> L(n_mz + 1);
	std::vector<uint64_t> S(raw_off[n_mz] + 1);
	struct Args {
		wm_idx_dev ix; const wm128_dev *mz; int n_mz; const int32_t *cnt; const uint64_t *list_off; const uint8_t *tandem; const int64_t *raw_off;
		int qlen; uint2 sk; int filter; wm128_dev *H; wm_heap_list *L; uint64_t *stage; wm128_dev *a; int64_t n, ret;
	} A;
	memset(&A.ix, 0, sizeof(A.ix));
	A.ix.pos = pos, A.ix.seq_len = seq_len, A.ix.name_rank = name_rank;
	A.mz = (const wm128_dev*)mz_xy, A.n_mz = n_mz, A.cnt = cnt, A.list_off = list_off, A.tandem = tandem, A.raw_off = raw_off.data();
	A.qlen = qlen, A.sk.x = skip_bits, A.sk.y = name_lt, A.filter = filter;
	A.H = H.data(), A.L = L.data(), A.stage = stage ? S.data() : 0, A.a = (wm128_dev*)a_xy, A.n = n, A.ret = 0;
	wm_emul::run_warp([](int l, void *p) {
		Args &a = *(Args*)p;
		const int64_t r = a.filter ? wm_heap_replay_task<true>(a.ix, a.mz, 0, a.n_mz, a.cnt, a.list_off, a.tandem, a.raw_off, a.qlen, a.sk, a.H, a.L, a.stage, a.a, a.n, l)
		                           : wm_heap_replay_task<false>(a.ix, a.mz, 0, a.n_mz, a.cnt, a.list_off, a.tandem, a.raw_off, a.qlen, a.sk, a.H, a.L, a.stage, a.a, a.n, l);
		if (l == 0) a.ret = r;
	}, &A);
	return (long)A.ret;
}
