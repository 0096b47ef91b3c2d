// TEST INFRASTRUCTURE ONLY. The wrappers of ref_harness.cpp plus the reference's homopolymer-compressed paths:
// mm_sketch with is_hpc = 1 (src/sketch.c:146-157) and an index read with an index flag (-H sets MM_I_HPC,
// src/main.c:166).  Built into oracle/_ref/libref_harness_hpc.so by oracle/build_hpc.sh; nothing in the product path
// links or loads it.
#include "ref_harness.cpp"

extern "C" {

long ref_sketch_hpc(void *ctx, const char *seq, int len, int w, int k, uint32_t rid, uint64_t *out_xy, long max_out)
{
	ref_sk *c = (ref_sk*)ctx;
	mm128_v v = {0, 0, 0};
	mm_sketch(0, seq, len, w, k, rid, 1, &v, &c->mi);
	long n = (long)v.n < max_out ? (long)v.n : max_out;
	memcpy(out_xy, v.a, n * 16);
	long tot = v.n;
	kfree(0, v.a);
	return tot;
}

// ref_idx_build_flat with the index flag of mm_idxopt_t (the bucket walk is the same)
void *ref_idx_build_flat_flag(const char *fn, const char *kmer_fn, int w, int k, int flag, int n_threads)
{
	mm_idxopt_t io; mm_mapopt_t mo;
	mm_set_opt(0, &io, &mo);
	io.k = k, io.w = w, io.flag = flag;
	mm_idx_reader_t *r = mm_idx_reader_open(fn, &io, 0);
	if (!r) return 0;
	mm_idx_t *mi = mm_idx_reader_read(r, n_threads, kmer_fn ? kmer_fn : "");
	mm_idx_reader_close(r);
	if (!mi) return 0;
	ref_flat *f = new ref_flat(); f->mi = mi;
	std::vector<std::pair<uint64_t, std::pair<const uint64_t*, int> > > all;
	const ref_bucket_t *B = (const ref_bucket_t*)mi->B;
	for (uint32_t b = 0; b < 1U << mi->b; ++b) {
		khash_t(refidx) *h = (khash_t(refidx)*)B[b].h;
		if (h == 0) continue;
		for (khint_t x = 0; x < kh_end(h); ++x) {
			if (!kh_exist(h, x)) continue;
			const uint64_t minier = (kh_key(h, x) >> 1) << mi->b | b;
			if (kh_key(h, x) & 1) all.push_back(std::make_pair(minier, std::make_pair((const uint64_t*)&kh_val(h, x), 1)));
			else all.push_back(std::make_pair(minier, std::make_pair((const uint64_t*)&B[b].p[kh_val(h, x) >> 32], (int)(uint32_t)kh_val(h, x))));
		}
	}
	std::sort(all.begin(), all.end());
	for (size_t i = 0; i < all.size(); ++i) {
		f->keys.push_back(all[i].first); f->pos_off.push_back(f->pos.size());
		f->pos.insert(f->pos.end(), all[i].second.first, all[i].second.first + all[i].second.second);
	}
	f->pos_off.push_back(f->pos.size());
	for (uint32_t i = 0; i < mi->n_seq; ++i) { f->names.push_back(mi->seq[i].name); f->seq_len.push_back(mi->seq[i].len); f->seq_off.push_back(mi->seq[i].offset); }
	return f;
}
int ref_idx_flat_flag(void *p) { return ((ref_flat*)p)->mi->flag; }

} // extern "C"
