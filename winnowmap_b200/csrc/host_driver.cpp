// The file-level mapping driver (host_driver.h): mini-batches, length sort, rank dealing, the output step and the in-memory
// merge of --split-prefix.
#include <errno.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <condition_variable>
#include <mutex>
#include <thread>
#include "host_driver.h"
#include "host_glue.h"
#include "host_io.h"

namespace wmh {

void format_read(std::string &dst, const wm_host_idx *mi, int64_t opt_flag, const wm_read *t, int n_reg, const wm_reg1_t *regs, int rep_len,
                 const char *prefix, const char *rg_id)
{
	std::string line;
	const bool sam = (opt_flag & WM_F_OUT_SAM) != 0;
	auto emit = [&](int j) { // hit j of the read, or the empty record (j < 0)
		if (sam) write_sam(line, mi, t, j, n_reg, regs, opt_flag, rep_len, rg_id ? rg_id : "");
		else write_paf(line, mi, t, j >= 0 ? &regs[j] : 0, opt_flag, rep_len);
		if (prefix) dst += prefix;
		dst += line; dst += '\n';
	};
	if (n_reg > 0) {
		for (int j = 0; j < n_reg; ++j) {
			if ((opt_flag & WM_F_NO_PRINT_2ND) && regs[j].id != regs[j].parent) continue;
			emit(j);
		}
	} else if ((opt_flag & WM_F_PAF_NO_HIT) || (sam && !(opt_flag & WM_F_SAM_HIT_ONLY))) emit(-1);
}

// merge_hits in memory: the regs of the parts concatenated in part order, rid shifted by the sequences of the earlier parts,
// then mm_hit_sort, mm_set_parent, mm_select_sub and mm_set_sam_pri (not under MM_F_ALL_CHAINS) and mm_set_mapq with the
// largest rep_len of the parts.
bool map_merged(IndexParts &ix, const wm_mapopt_t *opt, const std::vector<const wm_read*> &reads, std::vector<std::vector<wm_reg1_t>> &regs,
                int n_threads)
{
	const int n = (int)reads.size();
	regs.assign(n, std::vector<wm_reg1_t>());
	std::vector<int> rep_len(n, 0);
	int32_t rid_shift = 0;
	for (int p = 0; p < ix.n_parts(); ++p) {
		wm_mapopt_t o;
		if (!ix.part_opt(p, opt, &o)) return false;
		std::vector<std::vector<wm_reg1_t>> r; std::vector<int> rl;
		ix.map(p, &o, reads, r, rl, n_threads);
		for (int i = 0; i < n; ++i) {
			for (auto &x : r[i]) { x.rid += rid_shift; regs[i].push_back(x); }
			rep_len[i] = std::max(rep_len[i], rl[i]);
		}
		rid_shift += (int32_t)ix.part(p)->name.size();
	}
	const int k = ix.all()->k;
	#pragma omp parallel for schedule(dynamic, 16) num_threads(n_threads > 0 ? n_threads : 1)
	for (int i = 0; i < n; ++i) {
		std::vector<wm_reg1_t> &v = regs[i];
		hit_sort(v, opt->alt_drop);
		set_parent(opt->mask_level, opt->mask_len, (int)v.size(), v.data(), opt->a * 2 + opt->b, (int)(opt->flag & WM_F_HARD_MLEVEL), opt->alt_drop);
		if (!(opt->flag & WM_F_ALL_CHAINS)) {
			select_sub(opt->pri_ratio, k * 2, opt->best_n, v);
			set_sam_pri((int)v.size(), v.data());
		}
		set_mapq(v, opt->min_chain_score, opt->a, rep_len[i], 0);
	}
	return true;
}

// One pass over the read file: part `part` of ix (mapped and written as mm_map_file does), or, with part < 0, every part
// mapped and merged per read (map_merged), written with the sequence table of all parts.  Reads are taken in the reference's
// mini-batches (src/bseq.c:80-119), sorted by length descending inside a batch (src/map.c:1124-1143) and printed in that
// order (:1173-1208).  -2 when the read file cannot be opened.
static int map_file_pass(IndexParts &ix, int part, const wm_mapopt_t *opt_in, const char *reads_fn, FILE *out, const char *rg_id, int n_threads, int rank,
                         int world, int tag_order, int64_t max_batch_bases)
{
	SeqReader rd;
	if (!rd.open(reads_fn)) { fprintf(stderr, "ERROR: failed to open file '%s': %s\n", reads_fn, strerror(errno)); return -2; }
	const bool merged = part < 0;
	wm_mapopt_t opt_part;
	if (!merged && !ix.part_opt(part, opt_in, &opt_part)) return -1;
	const wm_mapopt_t *opt = merged ? opt_in : &opt_part;
	const wm_host_idx *mi = merged ? ix.all() : ix.part(part);
	const int64_t chunk = opt->mini_batch_size;
	bool failed = false;
	// The three steps of the reference's pipeline (src/map.c:1107-1224: read, map, write) run on three threads with
	// one mini-batch of slack between them: the next batch is parsed and the previous one formatted while the GPU maps.
	struct FileBatch {
		int64_t no;
		std::vector<wm_read> reads;
		std::vector<const wm_read*> mine; std::vector<int> mine_pos;          // this rank's reads, in output order
		std::vector<std::vector<wm_reg1_t>> regs; std::vector<int> rl;        // aligned with `mine`
	};
	struct Slot { // a one-element hand-over queue
		std::mutex mu; std::condition_variable cv; FileBatch *item = 0; bool closed = false;
		void put(FileBatch *b) { std::unique_lock<std::mutex> lk(mu); cv.wait(lk, [&] { return item == 0; }); item = b; cv.notify_all(); }
		void close() { std::unique_lock<std::mutex> lk(mu); cv.wait(lk, [&] { return item == 0; }); closed = true; cv.notify_all(); }
		FileBatch *get() { std::unique_lock<std::mutex> lk(mu); cv.wait(lk, [&] { return item != 0 || closed; }); FileBatch *b = item; item = 0; cv.notify_all(); return b; }
	} q_in, q_out;
	std::thread reader([&]() {
		int64_t batch_no = 0;
		for (;;) {
			FileBatch *b = new FileBatch();
			int64_t size = 0;
			wm_read r;
			const bool with_qual = (opt->flag & WM_F_OUT_SAM) && !(opt->flag & WM_F_NO_QUAL); // src/map.c:1112
			while (rd.next(r)) {
				size += (int64_t)r.seq.size();
				if (!with_qual) r.qual.clear();
				b->reads.push_back(r);
				if (size >= chunk) break;
			}
			if (b->reads.empty()) { delete b; break; }
			b->no = batch_no++;
			q_in.put(b);
		}
		q_in.close();
	});
	std::thread writer([&]() {
		std::vector<std::string> lines;
		for (;;) {
			FileBatch *b = q_out.get();
			if (!b) break;
			const int n = (int)b->mine.size();
			lines.assign(n, std::string());
			#pragma omp parallel for schedule(dynamic, 16) num_threads(n_threads > 8 ? 8 : (n_threads > 0 ? n_threads : 1))
			for (int i = 0; i < n; ++i) {
				char tag[64];
				if (tag_order) snprintf(tag, sizeof(tag), "%lld\t%d\t", (long long)b->no, b->mine_pos[i]);
				format_read(lines[i], mi, opt->flag, b->mine[i], (int)b->regs[i].size(), b->regs[i].data(), b->rl[i], tag_order ? tag : 0, rg_id);
				for (auto &rr : b->regs[i]) free(rr.p);
			}
			for (int i = 0; i < n; ++i) fwrite(lines[i].data(), 1, lines[i].size(), out);
			delete b;
		}
	});
	for (;;) {
		FileBatch *b = q_in.get();
		if (!b) break;
		// longer reads first; ties by larger input index first (std::greater on (len, index), src/map.c:1129)
		std::vector<std::pair<int, int>> ord;
		for (size_t i = 0; i < b->reads.size(); ++i) ord.emplace_back((int)b->reads[i].seq.size(), (int)i);
		std::sort(ord.begin(), ord.end(), std::greater<std::pair<int, int>>());
		for (size_t p = 0; p < ord.size(); ++p)
			if ((int)(p % (size_t)world) == rank) { b->mine.push_back(&b->reads[ord[p].second]); b->mine_pos.push_back((int)p); }
		b->regs.resize(b->mine.size()); b->rl.assign(b->mine.size(), 0);
		// internal sub-batches bound device memory; results do not depend on how reads are grouped
		size_t s0 = 0;
		while (s0 < b->mine.size()) {
			size_t s1 = s0; int64_t nb = 0;
			while (s1 < b->mine.size() && (s1 == s0 || nb + (int64_t)b->mine[s1]->seq.size() <= max_batch_bases)) nb += (int64_t)b->mine[s1]->seq.size(), ++s1;
			std::vector<const wm_read*> sub(b->mine.begin() + s0, b->mine.begin() + s1);
			std::vector<std::vector<wm_reg1_t>> regs; std::vector<int> rl;
			if (merged) { // the merge pass leaves rep_len 0 in what it prints (src/map.c:1050-1105 does not set it)
				if (!failed && !map_merged(ix, opt, sub, regs, n_threads)) failed = true;
				if (failed) regs.assign(sub.size(), std::vector<wm_reg1_t>());
				rl.assign(sub.size(), 0);
			} else ix.map(part, opt, sub, regs, rl, n_threads);
			for (size_t i = 0; i < sub.size(); ++i) { b->regs[s0 + i].swap(regs[i]); b->rl[s0 + i] = rl[i]; }
			s0 = s1;
		}
		q_out.put(b);
	}
	q_out.close();
	reader.join(); writer.join();
	return failed ? -1 : 0;
}

// Without split_prefix a multi-part index is mapped part by part and written part-major, as the reference's loop over the
// parts does (src/main.c:384-424); the SAM header then has no @SQ line (mm_write_sam_hdr(0, ...), :391-398).  With
// split_prefix the parts' hits are merged per read in one pass (mm_split_merge, src/map.c:1278-1321), also for a single
// index: its @SQ lines then come twice, the normal header's and the merge's, as the reference prints them.  The reference
// goes through temporary files <prefix>.NNNN.tmp; here the merge runs in memory and no file is written.
int map_files(IndexParts &ix, const wm_mapopt_t *opt, const std::vector<const char*> &reads_fns, const char *out_fn, const char *sam_cl, const char *rg,
              int n_threads, int rank, int world, int tag_order, int64_t max_batch_bases)
{
	const bool merged = opt->split_prefix != 0;
	if (ix.n_parts() > 1 && !merged && world > 1) {
		fprintf(stderr, "[ERROR] wm_map_file: a multi-part index without split_prefix is written part-major, which does not shard over ranks\n");
		return -1;
	}
	FILE *out = out_fn && strcmp(out_fn, "-") ? fopen(out_fn, "wb") : stdout;
	if (!out) return -1;
	std::string rg_line, rg_id;
	if ((opt->flag & WM_F_OUT_SAM) && rg && sam_rg_line(rg, rg_line, rg_id) < 0) rg_line.clear(), rg_id.clear(); // reported; mapping goes on
	if ((opt->flag & WM_F_OUT_SAM) && rank == 0 && !tag_order) { // mm_write_sam_hdr (src/main.c:391-398); the merge's @SQ lines follow (src/map.c:1304-1306)
		std::string h;
		wm_host_idx none;
		const wm_host_idx *all = ix.all();
		write_sam_hdr(h, ix.n_parts() > 1 ? &none : all, "2.03", sam_cl, rg_line.empty() ? 0 : rg_line.c_str());
		if (merged)
			for (size_t i = 0; i < all->name.size(); ++i) { h += "@SQ\tSN:"; h += all->name[i]; h += "\tLN:"; h += std::to_string(all->len[i]); h += '\n'; }
		fwrite(h.data(), 1, h.size(), out);
	}
	int rc = 0;
	auto pass = [&](int p, const char *fn) {
		const int r = map_file_pass(ix, p, opt, fn, out, rg_id.c_str(), n_threads, rank, world, tag_order, max_batch_bases);
		if (r == -1) rc = -1;
	};
	if (merged) for (size_t f = 0; f < reads_fns.size() && rc == 0; ++f) pass(-1, reads_fns[f]);
	else for (int p = 0; p < ix.n_parts() && rc == 0; ++p) for (size_t f = 0; f < reads_fns.size() && rc == 0; ++f) pass(p, reads_fns[f]);
	if (out != stdout) fclose(out); else fflush(out);
	return rc;
}

int map_file(IndexParts &ix, const wm_mapopt_t *opt, const char *reads_fn, const char *out_fn, const char *sam_cl, int n_threads, int rank, int world,
             int tag_order, int64_t max_batch_bases)
{
	{ // the read file is checked before the output is created
		SeqReader rd;
		if (!rd.open(reads_fn)) { fprintf(stderr, "ERROR: failed to open file '%s': %s\n", reads_fn, strerror(errno)); return -1; }
	}
	return map_files(ix, opt, std::vector<const char*>(1, reads_fn), out_fn, sam_cl, 0, n_threads, rank, world, tag_order, max_batch_bases);
}

} // namespace wmh
