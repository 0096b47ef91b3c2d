// Junction intervals from a BED file (mm_idx_read_bed / mm_idx_bed_read, reference src/index.c:690-778, with read_junc = 1 as
// src/main.c:416 calls it): what spliced alignment annotates its DP targets with (mm_idx_bed_junc, src/index.c:780; on the
// device: bed_junc.cuh).
#include <ctype.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include <string>
#include <unordered_map>
#include <vector>
#include "host_io.h"

namespace wmh {

// One line, split on tabs as the reference splits it: column 0 names the sequence (an unknown name drops the line: "track" and
// "#" lines, among others), 1 and 2 are start and end (a negative value stops the parse), 4 the score, 5 the strand, 9 the block
// count (a non-digit there stops the parse), 10 and 11 the block sizes and starts.  A line that reaches column 11 gives the gaps
// between its consecutive blocks, the others [start, end) itself; a line with start >= end gives nothing.
static void bed_line(std::string &line, const std::unordered_map<std::string, int> &ids, std::vector<std::vector<wm_idx_intv1_t>> &out)
{
	wm_idx_intv1_t t;
	t.st = t.en = t.max = -1, t.score = -1, t.strand = 0;
	int id = -1, col = 0;
	int32_t n_blk = 0;
	char *s = &line[0], *lend = s + line.size(), *q = s, *bl = 0, *bs = 0;
	for (char *p = s;; ++p) {
		if (*p != 0 && *p != '\t') continue;
		const char c = *p;
		*p = 0;
		if (col == 0) {
			auto it = ids.find(q);
			if (it == ids.end()) break;
			id = it->second;
		} else if (col == 1) {
			t.st = (int32_t)atol(q);
			if (t.st < 0) break;
		} else if (col == 2) {
			t.en = (int32_t)atol(q);
			if (t.en < 0) break;
		} else if (col == 4) {
			t.score = (int32_t)atol(q);
		} else if (col == 5) {
			t.strand = *q == '+' ? 1 : *q == '-' ? -1 : 0;
		} else if (col == 9) {
			if (!isdigit((unsigned char)*q)) break;
			n_blk = (int32_t)atol(q);
		} else if (col == 10) {
			bl = q;
		} else if (col == 11) {
			bs = q;
			break;
		}
		if (c == 0) break;
		++col, q = p + 1;
	}
	if (id < 0 || t.st < 0 || t.st >= t.en) return;
	std::vector<wm_idx_intv1_t> &r = out[id];
	if (col < 11) { r.push_back(t); return; }
	// BED12: block b spans [t.st + start_b, t.st + start_b + size_b); each list is read as strtol reads it, one separator skipped
	// after every number (past the end of a short list, the text of the next column, as in the reference; never past the line)
	auto next = [lend](char *&p) { const int32_t v = (int32_t)strtol(p, &p, 10); if (p < lend) ++p; return v; };
	int32_t bst = next(bs), bsz = next(bl), en = t.st + bst + bsz;
	for (int32_t b = 1; b < n_blk; ++b) {
		bst = next(bs), bsz = next(bl);
		wm_idx_intv1_t g = t;
		g.st = en, g.en = t.st + bst;
		en = t.st + bst + bsz;
		if (g.en > g.st) r.push_back(g);
		if (bs >= lend && bl >= lend && en == t.st) break; // both lists used up: every further gap is [t.st, t.st)
	}
}

static void put_junc(wm_host_idx *mi, std::vector<std::vector<wm_idx_intv1_t>> &per)
{
	mi->junc_iv.clear();
	mi->junc_off.assign(1, 0);
	for (auto &v : per) {
		// the reference radix-sorts on st; the order of equal starts does not change any annotation
		std::stable_sort(v.begin(), v.end(), [](const wm_idx_intv1_t &a, const wm_idx_intv1_t &b) { return a.st < b.st; });
		mi->junc_iv.insert(mi->junc_iv.end(), v.begin(), v.end());
		mi->junc_off.push_back((int64_t)mi->junc_iv.size());
	}
}

int read_bed_junc(wm_host_idx *mi, const char *fn)
{
	SeqReader rd;
	if (!rd.open(fn)) return -1;
	std::unordered_map<std::string, int> ids; // mm_idx_name2id (src/index.c:133-159): with repeated names, the first sequence of the name
	for (size_t i = 0; i < mi->name.size(); ++i) ids.emplace(mi->name[i], (int)i);
	std::vector<std::vector<wm_idx_intv1_t>> per(mi->name.size());
	std::string line;
	while (rd.next_line(line)) bed_line(line, ids, per);
	put_junc(mi, per);
	return 0;
}

void set_junc(wm_host_idx *mi, const wm_idx_intv_t *I)
{
	std::vector<std::vector<wm_idx_intv1_t>> per(mi->name.size());
	for (size_t i = 0; i < per.size(); ++i)
		if (I[i].n > 0) per[i].assign(I[i].a, I[i].a + I[i].n);
	put_junc(mi, per);
}

} // namespace wmh
