// See host_align.h.  Reference: src/align.c (line numbers cited per function).
#include <assert.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <algorithm>
#include "host_align.h"
#include "host_timers.h"
#include "host_glue.h"

namespace wmh {

#define EZ_RIGHT      0x02
#define EZ_APPROX_MAX 0x08
#define EZ_SCAN_ZDROP 0x10000 // not a ksw2 flag: asks the backend for the mm_test_zdrop score walk over the result (DpRes::has_zd)
#define EZ_EXTZ_ONLY  0x40
#define EZ_REV_CIGAR  0x80
#define EZ_SPLICE_FOR 0x100
#define EZ_SPLICE_REV 0x200
#define EZ_SPLICE_FLANK 0x400

// seq_nt4_table (src/sketch.c:19-36): bytes 0..3 and ACGT/acgt (U/u as T) are bases, everything else 4
struct Nt4Table {
	uint8_t t[256];
	Nt4Table() {
		for (int i = 0; i < 256; ++i) t[i] = 4;
		t[0] = t['A'] = t['a'] = 0; t[1] = t['C'] = t['c'] = 1; t[2] = t['G'] = t['g'] = 2; t[3] = t['T'] = t['t'] = t['U'] = t['u'] = 3;
	}
};
static const Nt4Table g_nt4;
static inline uint8_t nt4(unsigned char c) { return g_nt4.t[c]; }

void gen_simple_mat(int8_t *mat, int8_t a, int8_t b, int8_t sc_ambi)
{ // ksw_gen_simple_mat, src/align.c:9-22 with m = 5
	a = a < 0 ? -a : a;
	b = b > 0 ? -b : b;
	sc_ambi = sc_ambi > 0 ? -sc_ambi : sc_ambi;
	for (int i = 0; i < 4; ++i) {
		for (int j = 0; j < 4; ++j) mat[i * 5 + j] = i == j ? a : b;
		mat[i * 5 + 4] = sc_ambi;
	}
	for (int j = 0; j < 5; ++j) mat[20 + j] = sc_ambi;
}

static inline uint32_t round_up_pow2(uint32_t x)
{ // kroundup32
	--x; x |= x >> 1; x |= x >> 2; x |= x >> 4; x |= x >> 8; x |= x >> 16; return ++x;
}

void append_cigar(wm_reg1_t *r, uint32_t n_cigar, const uint32_t *cigar)
{ // mm_append_cigar, src/align.c:288-311 (libc allocation: the caller frees r->p)
	if (n_cigar == 0) return;
	if (r->p == 0) {
		uint32_t capacity = round_up_pow2(n_cigar + (uint32_t)(sizeof(wm_extra_t) / 4));
		r->p = (wm_extra_t*)calloc(capacity, 4);
		r->p->capacity = capacity;
	} else if (r->p->n_cigar + n_cigar + sizeof(wm_extra_t) / 4 > r->p->capacity) {
		r->p->capacity = round_up_pow2(r->p->n_cigar + n_cigar + (uint32_t)(sizeof(wm_extra_t) / 4));
		r->p = (wm_extra_t*)realloc(r->p, (size_t)r->p->capacity * 4);
	}
	wm_extra_t *p = r->p;
	if (p->n_cigar > 0 && (p->cigar[p->n_cigar - 1] & 0xf) == (cigar[0] & 0xf)) {
		p->cigar[p->n_cigar - 1] += cigar[0] >> 4 << 4;
		if (n_cigar > 1) memcpy(p->cigar + p->n_cigar, cigar + 1, (n_cigar - 1) * 4);
		p->n_cigar += n_cigar - 1;
	} else {
		memcpy(p->cigar + p->n_cigar, cigar, n_cigar * 4);
		p->n_cigar += n_cigar;
	}
}

static void fix_cigar(wm_reg1_t *r, const uint8_t *qseq, const uint8_t *tseq, int *qshift, int *tshift)
{ // mm_fix_cigar, src/align.c:91-167: left-align indels, merge xIyDzI runs, drop leading I/D
	wm_extra_t *p = r->p;
	int32_t toff = 0, qoff = 0, to_shrink = 0;
	*qshift = *tshift = 0;
	if (p->n_cigar <= 1) return;
	for (uint32_t k = 0; k < p->n_cigar; ++k) {
		const uint32_t op = p->cigar[k] & 0xf, len = p->cigar[k] >> 4;
		if (len == 0) to_shrink = 1;
		if (op == 0) toff += len, qoff += len;
		else if (op == 1 || op == 2) {
			if (k > 0 && k < p->n_cigar - 1 && (p->cigar[k - 1] & 0xf) == 0 && (p->cigar[k + 1] & 0xf) == 0) {
				int l, prev_len = p->cigar[k - 1] >> 4;
				if (op == 1) { for (l = 0; l < prev_len; ++l) if (qseq[qoff - 1 - l] != qseq[qoff + len - 1 - l]) break; }
				else { for (l = 0; l < prev_len; ++l) if (tseq[toff - 1 - l] != tseq[toff + len - 1 - l]) break; }
				if (l > 0) p->cigar[k - 1] -= l << 4, p->cigar[k + 1] += l << 4, qoff -= l, toff -= l;
				if (l == prev_len) to_shrink = 1;
			}
			if (op == 1) qoff += len; else toff += len;
		} else if (op == 3) toff += len;
	}
	for (uint32_t k = 0; k + 2 < p->n_cigar; ++k) {
		if ((p->cigar[k] & 0xf) > 0 && (p->cigar[k] & 0xf) + (p->cigar[k + 1] & 0xf) == 3) {
			uint32_t l, s[3] = {0, 0, 0};
			for (l = k; l < p->n_cigar; ++l) {
				uint32_t op = p->cigar[l] & 0xf;
				if (op == 1 || op == 2 || p->cigar[l] >> 4 == 0) s[op] += p->cigar[l] >> 4;
				else break;
			}
			if (s[1] > 0 && s[2] > 0 && l - k > 2) {
				p->cigar[k] = s[1] << 4 | 1;
				p->cigar[k + 1] = s[2] << 4 | 2;
				for (k += 2; k < l; ++k) p->cigar[k] &= 0xf;
				to_shrink = 1;
			}
			k = l;
		}
	}
	if (to_shrink) {
		int32_t l = 0;
		for (uint32_t k = 0; k < p->n_cigar; ++k) if (p->cigar[k] >> 4 != 0) p->cigar[l++] = p->cigar[k];
		p->n_cigar = l;
		l = 0;
		for (uint32_t k = 0; k < p->n_cigar; ++k)
			if (k == p->n_cigar - 1 || (p->cigar[k] & 0xf) != (p->cigar[k + 1] & 0xf)) p->cigar[l++] = p->cigar[k];
			else p->cigar[k + 1] += p->cigar[k] >> 4 << 4;
		p->n_cigar = l;
	}
	if ((p->cigar[0] & 0xf) == 1 || (p->cigar[0] & 0xf) == 2) {
		int32_t l = p->cigar[0] >> 4;
		if ((p->cigar[0] & 0xf) == 1) {
			if (r->rev) r->qe -= l; else r->qs += l;
			*qshift = l;
		} else r->rs += l, *tshift = l;
		--p->n_cigar;
		memmove(p->cigar, p->cigar + 1, p->n_cigar * 4);
	}
}

static void cigar_to_eqx(wm_reg1_t *r, const uint8_t *qseq, const uint8_t *tseq)
{ // mm_update_cigar_eqx, src/align.c:169-238
	uint32_t n_EQX = 0, k, l, m, cap, toff = 0, qoff = 0, n_M = 0;
	if (r->p == 0) return;
	for (k = 0; k < r->p->n_cigar; ++k) {
		uint32_t op = r->p->cigar[k] & 0xf, len = r->p->cigar[k] >> 4;
		if (op == 0) {
			while (len > 0) {
				for (l = 0; l < len && qseq[qoff + l] == tseq[toff + l]; ++l) {}
				if (l > 0) { ++n_EQX; len -= l; toff += l; qoff += l; }
				for (l = 0; l < len && qseq[qoff + l] != tseq[toff + l]; ++l) {}
				if (l > 0) { ++n_EQX; len -= l; toff += l; qoff += l; }
			}
			++n_M;
		} else if (op == 1) qoff += len;
		else if (op == 2 || op == 3) toff += len;
	}
	if (n_EQX == n_M) {
		for (k = 0; k < r->p->n_cigar; ++k) {
			uint32_t op = r->p->cigar[k] & 0xf, len = r->p->cigar[k] >> 4;
			if (op == 0) r->p->cigar[k] = len << 4 | 7;
		}
		return;
	}
	cap = round_up_pow2(r->p->n_cigar + (n_EQX - n_M) + (uint32_t)sizeof(wm_extra_t));
	wm_extra_t *p = (wm_extra_t*)calloc(cap, 4);
	memcpy(p, r->p, sizeof(wm_extra_t));
	p->capacity = cap;
	toff = qoff = m = 0;
	for (k = 0; k < r->p->n_cigar; ++k) {
		uint32_t op = r->p->cigar[k] & 0xf, len = r->p->cigar[k] >> 4;
		if (op == 0) {
			while (len > 0) {
				for (l = 0; l < len && qseq[qoff + l] == tseq[toff + l]; ++l) {}
				if (l > 0) p->cigar[m++] = l << 4 | 7;
				len -= l; toff += l, qoff += l;
				for (l = 0; l < len && qseq[qoff + l] != tseq[toff + l]; ++l) {}
				if (l > 0) p->cigar[m++] = l << 4 | 8;
				len -= l; toff += l, qoff += l;
			}
			continue;
		} else if (op == 1) qoff += len;
		else if (op == 2 || op == 3) toff += len;
		p->cigar[m++] = r->p->cigar[k];
	}
	p->n_cigar = m;
	free(r->p);
	r->p = p;
}

void update_extra(wm_reg1_t *r, const uint8_t *qseq, const uint8_t *tseq, const int8_t *mat, int8_t q, int8_t e, int is_eqx)
{ // mm_update_extra, src/align.c:240-286
	int32_t s = 0, max = 0, qshift, tshift, toff = 0, qoff = 0;
	wm_extra_t *p = r->p;
	if (p == 0) return;
	fix_cigar(r, qseq, tseq, &qshift, &tshift);
	qseq += qshift, tseq += tshift;
	r->blen = r->mlen = 0;
	// the four match scores are equal and positive for every matrix ksw_gen_simple_mat builds (src/align.c:9-22)
	const int32_t match_sc = mat[0];
	const bool uniform_match = match_sc > 0 && mat[6] == match_sc && mat[12] == match_sc && mat[18] == match_sc;
	for (uint32_t k = 0; k < p->n_cigar; ++k) {
		const uint32_t op = p->cigar[k] & 0xf, len = p->cigar[k] >> 4;
		if (op == 0) {
			int n_ambi = 0, n_diff = 0;
			const uint8_t *qp = qseq + qoff, *tp = tseq + toff;
			uint32_t l = 0;
			while (l < len) {
				if (uniform_match) { // a run of identical unambiguous bases adds a match score per base: s only grows, max follows
					uint32_t run = 0;
					while (l + run + 8 <= len) {
						uint64_t wq, wt;
						memcpy(&wq, qp + l + run, 8); memcpy(&wt, tp + l + run, 8);
						const uint64_t x = (wq ^ wt) | (wq & 0xfcfcfcfcfcfcfcfcULL); // a non-zero byte: mismatch or ambiguous base
						if (x == 0) { run += 8; continue; }
						run += (uint32_t)(__builtin_ctzll(x) >> 3);
						goto run_done;
					}
					while (l + run < len && qp[l + run] == tp[l + run] && qp[l + run] <= 3) ++run;
				run_done:
					if (run > 0) {
						s += match_sc * (int32_t)run; // s >= 0 on entry (every other step clamps it), so no clamp can trigger inside the run
						max = max > s ? max : s;
						l += run;
						continue;
					}
				}
				const int cq = qp[l], ct = tp[l];
				if (ct > 3 || cq > 3) ++n_ambi;
				else if (ct != cq) ++n_diff;
				s += mat[ct * 5 + cq];
				if (s < 0) s = 0; else max = max > s ? max : s;
				++l;
			}
			r->blen += len - n_ambi, r->mlen += len - (n_ambi + n_diff), p->n_ambi += n_ambi;
			toff += len, qoff += len;
		} else if (op == 1) {
			int n_ambi = 0;
			for (uint32_t l = 0; l < len; ++l) if (qseq[qoff + l] > 3) ++n_ambi;
			r->blen += len - n_ambi, p->n_ambi += n_ambi;
			s -= q + e * len;
			if (s < 0) s = 0;
			qoff += len;
		} else if (op == 2) {
			int n_ambi = 0;
			for (uint32_t l = 0; l < len; ++l) if (tseq[toff + l] > 3) ++n_ambi;
			r->blen += len - n_ambi, p->n_ambi += n_ambi;
			s -= q + e * len;
			if (s < 0) s = 0;
			toff += len;
		} else if (op == 3) toff += len;
	}
	p->dp_max = max;
	if (is_eqx) cigar_to_eqx(r, qseq, tseq);
}

// ---- seed clean-up ahead of the DP (src/align.c:365-495) ----
static std::vector<int> long_gaps(int as1, int cnt1, const wm_pair_t *a, int min_gap)
{ // collect_long_gaps :365-384; empty result when there are fewer than two
	std::vector<int> K;
	for (int i = 1; i < cnt1; ++i) {
		int gap = ((int32_t)a[as1 + i].y - a[as1 + i - 1].y) - ((int32_t)a[as1 + i].x - a[as1 + i - 1].x);
		if (gap < -min_gap || gap > min_gap) K.push_back(i);
	}
	if (K.size() <= 1) K.clear();
	return K;
}

static void filter_bad_seeds(int as1, int cnt1, wm_pair_t *a, int min_gap, int diff_thres, int max_ext_len, int max_ext_cnt)
{ // mm_filter_bad_seeds :386-421
	std::vector<int> K = long_gaps(as1, cnt1, a, min_gap);
	const int n = (int)K.size();
	if (n == 0) return;
	int max = 0, max_st = -1, max_en = -1;
	for (int k = 0;; ++k) {
		int gap, l, n_ins = 0, n_del = 0, qs, rs, max_diff = 0, max_diff_l = -1;
		if (k == n || k >= max_en) {
			if (max_en > 0)
				for (int i = K[max_st]; i < K[max_en]; ++i) a[as1 + i].y |= WM_SEED_IGNORE;
			max = 0, max_st = max_en = -1;
			if (k == n) break;
		}
		const int i = K[k];
		gap = ((int32_t)a[as1 + i].y - (int32_t)a[as1 + i - 1].y) - (int32_t)(a[as1 + i].x - a[as1 + i - 1].x);
		if (gap > 0) n_ins += gap; else n_del += -gap;
		qs = (int32_t)a[as1 + i - 1].y;
		rs = (int32_t)a[as1 + i - 1].x;
		for (l = k + 1; l < n && l <= k + max_ext_cnt; ++l) {
			const int j = K[l];
			if ((int32_t)a[as1 + j].y - qs > max_ext_len || (int32_t)a[as1 + j].x - rs > max_ext_len) break;
			gap = ((int32_t)a[as1 + j].y - (int32_t)a[as1 + j - 1].y) - (int32_t)(a[as1 + j].x - a[as1 + j - 1].x);
			if (gap > 0) n_ins += gap; else n_del += -gap;
			const int diff = n_ins + n_del - abs(n_ins - n_del);
			if (max_diff < diff) max_diff = diff, max_diff_l = l;
		}
		if (max_diff > diff_thres && max_diff > max) max = max_diff, max_st = k, max_en = max_diff_l;
	}
}

static void filter_bad_seeds_alt(int as1, int cnt1, wm_pair_t *a, int min_gap, int max_ext)
{ // mm_filter_bad_seeds_alt :423-457
	std::vector<int> K = long_gaps(as1, cnt1, a, min_gap);
	const int n = (int)K.size();
	for (int k = 0; k < n;) {
		const int i = K[k];
		int l;
		int gap1 = ((int32_t)a[as1 + i].y - (int32_t)a[as1 + i - 1].y) - ((int32_t)a[as1 + i].x - (int32_t)a[as1 + i - 1].x);
		int re1 = (int32_t)a[as1 + i].x, qe1 = (int32_t)a[as1 + i].y;
		gap1 = gap1 > 0 ? gap1 : -gap1;
		for (l = k + 1; l < n; ++l) {
			const int j = K[l];
			if ((int32_t)a[as1 + j].y - qe1 > max_ext || (int32_t)a[as1 + j].x - re1 > max_ext) break;
			int gap2 = ((int32_t)a[as1 + j].y - (int32_t)a[as1 + j - 1].y) - (int32_t)(a[as1 + j].x - a[as1 + j - 1].x);
			const int q_span_pre = a[as1 + j - 1].y >> 32 & 0xff;
			const int rs2 = (int32_t)a[as1 + j - 1].x + q_span_pre, qs2 = (int32_t)a[as1 + j - 1].y + q_span_pre;
			const int m = rs2 - re1 < qs2 - qe1 ? rs2 - re1 : qs2 - qe1;
			gap2 = gap2 > 0 ? gap2 : -gap2;
			if (m > gap1 + gap2) break;
			re1 = (int32_t)a[as1 + j].x, qe1 = (int32_t)a[as1 + j].y;
			gap1 = gap2;
		}
		if (l > k + 1) {
			const int end = K[l - 1];
			for (int j = K[k]; j < end; ++j) a[as1 + j].y |= WM_SEED_IGNORE;
			a[as1 + end].y |= WM_SEED_LONG_JOIN;
		}
		k = l;
	}
}

static void fix_bad_ends(const wm_reg1_t *r, const wm_pair_t *a, int bw, int min_match, int32_t *as, int32_t *cnt)
{ // mm_fix_bad_ends :459-495
	int32_t i, l, m;
	*as = r->as, *cnt = r->cnt;
	if (r->cnt < 3) return;
	m = l = a[r->as].y >> 32 & 0xff;
	for (i = r->as + 1; i < r->as + r->cnt - 1; ++i) {
		const int32_t q_span = a[i].y >> 32 & 0xff;
		if (a[i].y & WM_SEED_LONG_JOIN) break;
		const int32_t lr = (int32_t)a[i].x - (int32_t)a[i - 1].x, lq = (int32_t)a[i].y - (int32_t)a[i - 1].y;
		const int32_t min = lr < lq ? lr : lq, max = lr > lq ? lr : lq;
		if (max - min > l >> 1) *as = i;
		l += min;
		m += min < q_span ? min : q_span;
		if (l >= bw << 1 || (m >= min_match && m >= bw) || m >= r->mlen >> 1) break;
	}
	*cnt = r->as + r->cnt - *as;
	m = l = a[r->as + r->cnt - 1].y >> 32 & 0xff;
	for (i = r->as + r->cnt - 2; i > *as; --i) {
		const int32_t q_span = a[i + 1].y >> 32 & 0xff;
		if (a[i + 1].y & WM_SEED_LONG_JOIN) break;
		const int32_t lr = (int32_t)a[i + 1].x - (int32_t)a[i].x, lq = (int32_t)a[i + 1].y - (int32_t)a[i].y;
		const int32_t min = lr < lq ? lr : lq, max = lr > lq ? lr : lq;
		if (max - min > l >> 1) *cnt = i + 1 - *as;
		l += min;
		m += min < q_span ? min : q_span;
		if (l >= bw << 1 || (m >= min_match && m >= bw) || m >= r->mlen >> 1) break;
	}
}

// ---- AlignTask ----
void encode_strands(const char *seq, int len, uint8_t *fwd, uint8_t *rev)
{ // src/align.c:871-877
	for (int i = 0; i < len; ++i) {
		const uint8_t c = nt4((unsigned char)seq[i]);
		fwd[i] = c;
		rev[len - 1 - i] = c < 4 ? 3 - c : 4;
	}
}

void AlignTask::init(const wm_mapopt_t *opt_, const wm_host_idx *mi_, int task_id_, int qlen_, const char *qstr, std::vector<wm_reg1_t> &regs_in, wm_pair_t *a_,
                     const uint8_t *q0, const uint8_t *q1)
{
	opt = opt_, mi = mi_, task_id = task_id_, qlen = qlen_, a = a_;
	regs.clear(); // the task object is reused across waves
	regs.swap(regs_in);
	firsts.clear(); out.clear(); from_first.clear();
	if (q0 && q1) q_strand[0] = q0, q_strand[1] = q1;
	else {
		qcodes.resize((size_t)qlen * 2);
		encode_strands(qstr, qlen, qcodes.data(), qcodes.data() + qlen);
		q_strand[0] = qcodes.data(), q_strand[1] = qcodes.data() + qlen;
	}
	gen_simple_mat(mat, (int8_t)opt->a, (int8_t)opt->b, (int8_t)opt->sc_ambi);
	n_a = squeeze_a(regs, a); // :880
	phase = 0; cur = 0; sub = 0; inv_job = -1;
	const int64_t both = WM_F_SPLICE | WM_F_SPLICE_FOR | WM_F_SPLICE_REV;
	n_round = (opt->flag & both) == both ? 2 : 1; // :884
}

// The mm_align1 instances of one hit (one, or one per strand flag), and the ll jobs of mm_fix_bad_ends_splice (:545-563):
// mm_seed_ext_score (:523-543) of the first and of the last anchor, where the anchor is short for the gap that follows it.
// The filter reads the anchors' positions and spans only, so its result is the same in both rounds.
void AlignTask::start_rounds(const wm_reg1_t &r, Align1 *A, JobSink &sink)
{
	for (int k = 0; k < n_round; ++k) {
		A[k] = Align1(); A[k].r = r; A[k].state = 0;
		A[k].splice_flag = n_round == 2 ? (k == 0 ? WM_F_SPLICE_FOR : WM_F_SPLICE_REV) : (int32_t)(opt->flag & (WM_F_SPLICE_FOR | WM_F_SPLICE_REV));
	}
	if (!(opt->flag & WM_F_SPLICE) || (opt->flag & WM_F_NO_END_FLT) || r.cnt < 3) return;
	const int ext_len = opt->anchor_ext_len;
	for (int e = 0; e < 2; ++e) {
		const wm_pair_t *p = &a[e == 0 ? r.as : r.as + r.cnt - 1], *nb = e == 0 ? p + 1 : p - 1;
		const double log_gap = e == 0 ? log((int32_t)nb->x - (int32_t)p->x) : log((int32_t)p->x - (int32_t)nb->x);
		if ((p->y >> 32 & 0xff) >= log_gap + opt->anchor_ext_shift) continue;
		const int q_span = p->y >> 32 & 0xff, rid = (int)(p->x << 1 >> 33), ref_len = (int)mi->len[rid];
		int re = (int)((uint32_t)p->x + 1), rs = re - q_span, qe = (int)((uint32_t)p->y + 1), qs = qe - q_span;
		rs = rs - ext_len > 0 ? rs - ext_len : 0;
		qs = qs - ext_len > 0 ? qs - ext_len : 0;
		re = re + ext_len < ref_len ? re + ext_len : ref_len;
		qe = qe + ext_len < qlen ? qe + ext_len : qlen;
		LlJob j;
		j.task = task_id;
		j.q = SeqRef{ (int32_t)(p->x >> 63) ? SEQ_Q1 : SEQ_Q0, 0, qs, qe - qs, 0 };
		j.t = SeqRef{ SEQ_REF, rid, rs, re - rs, 0 };
		A[0].end_ll[e] = (int)sink.ll.size();
		sink.ll.push_back(j);
	}
}

// as1 / cnt1 of mm_fix_bad_ends_splice from the ll scores, then everything mm_align1 does before its first DP, per round
void AlignTask::plan_rounds(Align1 *A, const LlRes *ll, JobSink &sink)
{
	if ((opt->flag & WM_F_SPLICE) && !(opt->flag & WM_F_NO_END_FLT)) {
		const wm_reg1_t *r = &A[0].r;
		int32_t as1 = r->as, cnt1 = r->cnt;
		for (int e = 0; e < 2; ++e) {
			if (A[0].end_ll[e] < 0) continue;
			const wm_pair_t *p = &a[e == 0 ? r->as : r->as + r->cnt - 1], *nb = e == 0 ? p + 1 : p - 1;
			const double log_gap = e == 0 ? log((int32_t)nb->x - (int32_t)p->x) : log((int32_t)p->x - (int32_t)nb->x);
			if ((double)ll[A[0].end_ll[e]].score / mat[0] < log_gap + opt->anchor_ext_shift) { // "score < log_4(gap) + shift"
				if (e == 0) ++as1;
				--cnt1;
			}
		}
		for (int k = 0; k < n_round; ++k) A[k].end_as1 = as1, A[k].end_cnt1 = cnt1, A[k].end_ll[0] = A[k].end_ll[1] = -1;
	}
	for (int k = 0; k < n_round; ++k) plan1(A[k], sink);
}

// The round a hit keeps (:890-904): the higher dp_score; on a tie trans_strand 3 and a choice by parity.  One round: the
// strand flag says it, so `-u n` gives trans_strand 2.
void AlignTask::pick_round(Align1 *A, wm_reg1_t *r, wm_reg1_t *r2) const
{
	auto extra = [](wm_reg1_t *x) { // (the reference dereferences p here; a hit without any DP has none)
		if (x->p) return;
		uint32_t capacity = round_up_pow2((uint32_t)(sizeof(wm_extra_t) / 4));
		x->p = (wm_extra_t*)calloc(capacity, 4);
		x->p->capacity = capacity;
	};
	if (n_round == 2) {
		extra(&A[0].r), extra(&A[1].r);
		int which, trans_strand;
		if (A[0].r.p->dp_score > A[1].r.p->dp_score) which = 0, trans_strand = 1;
		else if (A[0].r.p->dp_score < A[1].r.p->dp_score) which = 1, trans_strand = 2;
		else trans_strand = 3, which = (qlen + A[0].r.p->dp_score) & 1;
		*r = A[which].r, *r2 = A[which].r2;
		free(A[!which].r.p);
		r->p->trans_strand = trans_strand;
		return;
	}
	*r = A[0].r, *r2 = A[0].r2;
	if (opt->flag & WM_F_SPLICE) { extra(r); r->p->trans_strand = (opt->flag & WM_F_SPLICE_FOR) ? 1 : 2; }
}

// extra_flag of mm_align1 (:602-606): the splice signals of the round's strand flag, as seen from the hit's strand
static int32_t ez_splice_flag(const wm_mapopt_t *opt, const Align1 &A)
{
	int32_t f = 0;
	if (!(opt->flag & WM_F_SPLICE)) return 0;
	if (A.splice_flag & WM_F_SPLICE_FOR) f |= A.rev ? EZ_SPLICE_REV : EZ_SPLICE_FOR;
	if (A.splice_flag & WM_F_SPLICE_REV) f |= A.rev ? EZ_SPLICE_FOR : EZ_SPLICE_REV;
	if (opt->flag & WM_F_SPLICE_FLANK) f |= EZ_SPLICE_FLANK;
	return f;
}

static inline void adjust_minier(const wm_host_idx *mi, const uint8_t *const qseq0[2], const wm_pair_t *p, int32_t *r, int32_t *q)
{ // mm_adjust_minier :350-365
	if (mi->flag & WM_I_HPC) {
		// the query walks back to the start of its homopolymer; as in the reference the loop never tests base 0
		const uint8_t *qseq = qseq0[p->x >> 63];
		int32_t i, c;
		*q = (int32_t)p->y;
		for (i = *q - 1, c = qseq[*q]; i > 0; --i)
			if (qseq[i] != c) break;
		*q = i + 1;
		// mm_get_hplen_back (:341-348): the reference's run down to the contig's first base inclusive
		const uint32_t rid = (uint32_t)(p->x << 1 >> 33);
		const int64_t off0 = (int64_t)mi->offset[rid], off = off0 + (uint32_t)p->x;
		const int cr = mi->base((uint64_t)off);
		int64_t j;
		for (j = off - 1; j >= off0; --j)
			if (mi->base((uint64_t)j) != cr) break;
		*r = (int32_t)p->x + 1 - (int32_t)(off - j);
	} else {
		*r = (int32_t)p->x - (mi->k >> 1);
		*q = (int32_t)p->y - (mi->k >> 1);
	}
}

// everything mm_align1 decides before its first DP (:565-688), plus the speculative job list
void AlignTask::plan1(Align1 &A, JobSink &sink)
{
	static const bool sub_t = getenv("WM_SUBTIMING") != 0;
	struct PlanTimer { bool on; double t0; PlanTimer(bool o) : on(o), t0(o ? Timers::now() : 0) {} ~PlanTimer() { if (on) g_timers.add("adv.plan1", Timers::now() - t0); } } plan_timer(sub_t);
	wm_reg1_t *r = &A.r;
	A.left_job = A.right_job = -1; A.gaps.clear(); A.gap_cur = 0; A.left_done = false; A.dropped = false; A.pending_job = -1; A.captured = false;
	A.r2.cnt = 0;
	if (r->cnt == 0) { A.state = 9; return; }
	const int32_t rid = A.rid = (int32_t)(a[r->as].x << 1 >> 33), rev = A.rev = (int32_t)(a[r->as].x >> 63);
	const int bw = A.bw = (int)(opt->bw * 1.5 + 1.);
	int32_t as1, cnt1, rs, qs, re, qe, rs0, qs0, re0, qe0, rs1, qs1, re1, qe1, i, l;
	const int32_t ref_len = (int32_t)mi->len[rid];
	if (!(opt->flag & WM_F_NO_END_FLT)) {
		if (opt->flag & WM_F_SPLICE) as1 = A.end_as1, cnt1 = A.end_cnt1; // mm_fix_bad_ends_splice (plan_rounds)
		else fix_bad_ends(r, a, opt->bw, opt->min_chain_score * 2, &as1, &cnt1);
	} else as1 = r->as, cnt1 = r->cnt;
	const int32_t extra_flag = ez_splice_flag(opt, A);
	filter_bad_seeds(as1, cnt1, a, 10, 40, opt->max_gap >> 1, 10);
	filter_bad_seeds_alt(as1, cnt1, a, 30, opt->max_gap >> 1);
	adjust_minier(mi, q_strand, &a[as1], &rs, &qs);
	adjust_minier(mi, q_strand, &a[as1 + cnt1 - 1], &re, &qe);
	A.as1 = as1, A.cnt1 = cnt1;
	// DP region (:613-684)
	rs0 = (int32_t)a[r->as].x + 1 - (int32_t)(a[r->as].y >> 32 & 0xff);
	qs0 = (int32_t)a[r->as].y + 1 - (int32_t)(a[r->as].y >> 32 & 0xff);
	if (rs0 < 0) rs0 = 0;
	rs1 = qs1 = 0;
	for (i = r->as - 1, l = 0; i >= 0 && a[i].x >> 32 == a[r->as].x >> 32; --i) {
		int32_t x = (int32_t)a[i].x + 1 - (int32_t)(a[i].y >> 32 & 0xff);
		int32_t y = (int32_t)a[i].y + 1 - (int32_t)(a[i].y >> 32 & 0xff);
		if (x < rs0 && y < qs0) {
			if (++l > opt->min_cnt) {
				l = rs0 - x > qs0 - y ? rs0 - x : qs0 - y;
				rs1 = rs0 - l, qs1 = qs0 - l;
				if (rs1 < 0) rs1 = 0;
				break;
			}
		}
	}
	if (qs > 0 && rs > 0) {
		l = qs < opt->max_gap ? qs : opt->max_gap;
		qs1 = qs1 > qs - l ? qs1 : qs - l;
		qs0 = qs0 < qs1 ? qs0 : qs1;
		l += l * opt->a > opt->q ? (l * opt->a - opt->q) / opt->e : 0;
		l = l < opt->max_gap ? l : opt->max_gap;
		l = l < rs ? l : rs;
		rs1 = rs1 > rs - l ? rs1 : rs - l;
		rs0 = rs0 < rs1 ? rs0 : rs1;
		rs0 = rs0 < rs ? rs0 : rs;
	} else rs0 = rs, qs0 = qs;
	re0 = (int32_t)a[r->as + r->cnt - 1].x + 1;
	qe0 = (int32_t)a[r->as + r->cnt - 1].y + 1;
	re1 = ref_len, qe1 = qlen;
	for (i = r->as + r->cnt, l = 0; i < n_a && a[i].x >> 32 == a[r->as].x >> 32; ++i) {
		int32_t x = (int32_t)a[i].x + 1, y = (int32_t)a[i].y + 1;
		if (x > re0 && y > qe0) {
			if (++l > opt->min_cnt) {
				l = x - re0 > y - qe0 ? x - re0 : y - qe0;
				re1 = re0 + l, qe1 = qe0 + l;
				break;
			}
		}
	}
	if (qe < qlen && re < ref_len) {
		l = qlen - qe < opt->max_gap ? qlen - qe : opt->max_gap;
		qe1 = qe1 < qe + l ? qe1 : qe + l;
		qe0 = qe0 > qe1 ? qe0 : qe1;
		l += l * opt->a > opt->q ? (l * opt->a - opt->q) / opt->e : 0;
		l = l < opt->max_gap ? l : opt->max_gap;
		l = l < ref_len - re ? l : ref_len - re;
		re1 = re1 < re + l ? re1 : re + l;
		re0 = re0 > re1 ? re0 : re1;
	} else re0 = re, qe0 = qe;
	if (a[r->as].y & WM_SEED_SELF) {
		int max_ext = r->qs > r->rs ? r->qs - r->rs : r->rs - r->qs;
		if (r->rs - rs0 > max_ext) rs0 = r->rs - max_ext;
		if (r->qs - qs0 > max_ext) qs0 = r->qs - max_ext;
		max_ext = r->qe > r->re ? r->qe - r->re : r->re - r->qe;
		if (re0 - r->re > max_ext) re0 = r->re + max_ext;
		if (qe0 - r->qe > max_ext) qe0 = r->qe + max_ext;
	}
	A.rs0 = rs0, A.qs0 = qs0, A.re0 = re0, A.qe0 = qe0;
	A.rs_init = rs, A.qs_init = qs;
	// left extension (:690-705): both sequences reversed
	if (qs > 0 && rs > 0) {
		DpJob j;
		j.task = task_id;
		j.q = SeqRef{ rev ? SEQ_Q1 : SEQ_Q0, 0, qs0, qs - qs0, 1 };
		j.t = SeqRef{ SEQ_REF, rid, rs0, rs - rs0, 1 };
		j.w = bw, j.end_bonus = opt->end_bonus, j.zdrop = r->split_inv ? opt->zdrop_inv : opt->zdrop;
		j.flag = extra_flag | EZ_EXTZ_ONLY | EZ_RIGHT | EZ_REV_CIGAR;
		A.left_job = (int)sink.dp.size();
		sink.dp.push_back(j);
	}
	// gap filling windows (:709-730); they depend on the anchors only
	for (i = 1; i < cnt1; ++i) {
		if ((a[as1 + i].y & (WM_SEED_IGNORE | WM_SEED_TANDEM)) && i != cnt1 - 1) continue;
		adjust_minier(mi, q_strand, &a[as1 + i], &re, &qe);
		if (i == cnt1 - 1 || (a[as1 + i].y & WM_SEED_LONG_JOIN) || (qe - qs >= opt->min_ksw_len && re - rs >= opt->min_ksw_len)) {
			Align1::Gap g;
			g.i = i, g.rs = rs, g.qs = qs, g.re = re, g.qe = qe, g.bw1 = bw;
			if (a[as1 + i].y & WM_SEED_LONG_JOIN) g.bw1 = qe - qs > re - rs ? qe - qs : re - rs;
			DpJob j;
			j.task = task_id;
			j.q = SeqRef{ rev ? SEQ_Q1 : SEQ_Q0, 0, qs, qe - qs, 0 };
			j.t = SeqRef{ SEQ_REF, rid, rs, re - rs, 0 };
			j.w = g.bw1, j.end_bonus = -1, j.zdrop = opt->zdrop, j.flag = extra_flag | EZ_APPROX_MAX | EZ_SCAN_ZDROP; // first pass (:733)
			g.job = (int)sink.dp.size();
			sink.dp.push_back(j);
			A.gaps.push_back(g);
			rs = re, qs = qe;
		}
	}
	A.rs = rs, A.qs = qs, A.re = re, A.qe = qe;
	// right extension (:767-778), used only if no gap fill is Z-dropped
	if (qe < qe0 && re < re0) {
		DpJob j;
		j.task = task_id;
		j.q = SeqRef{ rev ? SEQ_Q1 : SEQ_Q0, 0, qe, qe0 - qe, 0 };
		j.t = SeqRef{ SEQ_REF, rid, re, re0 - re, 0 };
		j.w = bw, j.end_bonus = opt->end_bonus, j.zdrop = opt->zdrop, j.flag = extra_flag | EZ_EXTZ_ONLY;
		A.right_job = (int)sink.dp.size();
		sink.dp.push_back(j);
	}
	A.state = 1;
}

// the score walk of mm_test_zdrop (:47-70); returns max_zdrop and the most-dropped region
static int zdrop_scan(const wm_mapopt_t *opt, const uint8_t *qseq, const uint8_t *tseq, uint32_t n_cigar, const uint32_t *cigar, const int8_t *mat, int pos[2][2])
{
	int32_t score = 0, max = INT32_MIN, max_i = -1, max_j = -1, i = 0, j = 0, max_zdrop = 0;
	pos[0][0] = pos[0][1] = pos[1][0] = pos[1][1] = -1;
	auto upd = [&](int32_t sc, int ii, int jj) { // update_max_zdrop :32-45
		if (sc < max) {
			int li = ii - max_i, lj = jj - max_j;
			int diff = li > lj ? li - lj : lj - li;
			int z = max - sc - diff * opt->e;
			if (z > max_zdrop) { max_zdrop = z; pos[0][0] = max_i, pos[0][1] = ii; pos[1][0] = max_j, pos[1][1] = jj; }
		} else max = sc, max_i = ii, max_j = jj;
	};
	for (uint32_t k = 0; k < n_cigar; ++k) {
		const uint32_t op = cigar[k] & 0xf, len = cigar[k] >> 4;
		if (op == 0) {
			for (uint32_t l = 0; l < len; ++l) {
				score += mat[tseq[i + l] * 5 + qseq[j + l]];
				upd(score, i + l, j + l);
			}
			i += len, j += len;
		} else if (op == 1 || op == 2 || op == 3) {
			score -= opt->q + opt->e * len;
			if (op == 1) j += len; else i += len;
			upd(score, i, j);
		}
	}
	return max_zdrop;
}

// Walk the results of one mm_align1 in reference order.  Returns true when finished.
bool AlignTask::walk1(Align1 &A, const DpRes *dp, const LlRes *ll, JobSink &sink)
{
	wm_reg1_t *r = &A.r;
	if (A.state == 9) return true;
	const int rev = A.rev, rid = A.rid;
	static const bool sub_w = getenv("WM_SUBTIMING") != 0;
	const double w0 = sub_w ? Timers::now() : 0;
	if (!A.captured) { // keep the pass-1 results: later rounds reuse the result buffers
		size_t tot = 0;
		if (A.left_job >= 0) tot += dp[A.left_job].n_cigar > 0 ? dp[A.left_job].n_cigar : 0;
		if (A.right_job >= 0) tot += dp[A.right_job].n_cigar > 0 ? dp[A.right_job].n_cigar : 0;
		for (auto &g : A.gaps) tot += dp[g.job].n_cigar > 0 ? dp[g.job].n_cigar : 0;
		A.cig_pool.clear(); A.cig_pool.reserve(tot);
		auto grab = [&](int job, DpRes &res, size_t &off) {
			res = dp[job];
			off = A.cig_pool.size();
			if (res.n_cigar > 0) A.cig_pool.insert(A.cig_pool.end(), res.cigar, res.cigar + res.n_cigar);
			res.cigar = 0;
		};
		if (A.left_job >= 0) grab(A.left_job, A.left_res, A.left_cig);
		if (A.right_job >= 0) grab(A.right_job, A.right_res, A.right_cig);
		for (auto &g : A.gaps) grab(g.job, g.res, g.cig_off);
		A.captured = true;
	}
	if (sub_w) g_timers.add("walk.capture", Timers::now() - w0);
	if (!A.left_done) { // :690-708
		if (A.left_job >= 0) {
			DpRes ez = A.left_res; ez.cigar = A.cig_pool.data() + A.left_cig;
			if (ez.n_cigar > 0) { append_cigar(r, ez.n_cigar, ez.cigar); r->p->dp_score += ez.max; }
			A.rs1 = A.rs_init - (ez.reach_end ? ez.mqe_t + 1 : ez.max_t + 1);
			A.qs1 = A.qs_init - (ez.reach_end ? A.qs_init - A.qs0 : ez.max_q + 1);
		} else A.rs1 = A.rs_init, A.qs1 = A.qs_init;
		A.re1 = A.rs_init, A.qe1 = A.qs_init;
		A.left_done = true;
	}
	std::vector<uint8_t> tbuf;
	while (A.gap_cur < A.gaps.size()) {
		const Align1::Gap &g = A.gaps[A.gap_cur];
		const uint8_t *qs_ptr = qseq(rev) + g.qs;
		DpRes ez;
		int zdrop_code = 0;
		if (A.state == 1) { // first-pass result just arrived: test Z-drop (:736)
			static const bool sub_t = getenv("WM_SUBTIMING") != 0;
			const double q0 = sub_t ? Timers::now() : 0;
			int pos[2][2], max_zdrop;
			if (g.res.has_zd) { // the device walked the CIGAR right after the traceback
				max_zdrop = g.res.zd_max;
				pos[0][0] = g.res.zd_pos[0], pos[0][1] = g.res.zd_pos[1], pos[1][0] = g.res.zd_pos[2], pos[1][1] = g.res.zd_pos[3];
			} else {
				tbuf.resize(g.re - g.rs);
				mi->getseq(rid, g.rs, g.re, tbuf.data());
				max_zdrop = zdrop_scan(opt, qs_ptr, tbuf.data(), g.res.n_cigar, A.cig_pool.data() + g.cig_off, mat, pos);
			}
			if (sub_t) g_timers.add("adv.zdrop_scan", Timers::now() - q0);
			const int q_len = pos[1][1] - pos[1][0], t_len = pos[0][1] - pos[0][0];
			A.zd_max_zdrop = max_zdrop;
			if (!(opt->flag & (WM_F_SPLICE | WM_F_SR | WM_F_FOR_ONLY | WM_F_REV_ONLY)) && max_zdrop > opt->zdrop_inv && q_len < opt->max_gap && t_len < opt->max_gap) {
				if (q_len > 0 && t_len > 0) { // inversion test on the most-dropped region (:72-87)
					LlJob j;
					j.task = task_id;
					// revcomp(qseq[pos10, pos11)) of strand `rev` is a forward slice of the other strand
					j.q = SeqRef{ rev ? SEQ_Q0 : SEQ_Q1, 0, (int64_t)qlen - g.qs - pos[1][1], q_len, 0 };
					j.t = SeqRef{ SEQ_REF, rid, (int64_t)g.rs + pos[0][0], t_len, 0 };
					A.pending_job = (int)sink.ll.size();
					sink.ll.push_back(j);
					A.state = 2;
					return false;
				}
				// an empty query or target scores 0 in ksw_ll_i16
				zdrop_code = (0 >= opt->min_chain_score * opt->a && 0 >= opt->min_dp_max) ? 2 : (max_zdrop > opt->zdrop ? 1 : 0);
			} else zdrop_code = max_zdrop > opt->zdrop ? 1 : 0;
		} else if (A.state == 2) { // ll score arrived
			const int score = ll[A.pending_job].score;
			zdrop_code = (score >= opt->min_chain_score * opt->a && score >= opt->min_dp_max) ? 2 : (A.zd_max_zdrop > opt->zdrop ? 1 : 0);
			A.state = 1;
		}
		if (A.state == 3) { // second pass arrived (:737)
			ez = dp[A.pending_job];
			zdrop_code = A.zd_max_zdrop; // stashed code
			A.state = 1;
		} else if (zdrop_code != 0) {
			DpJob j;
			j.task = task_id;
			j.q = SeqRef{ rev ? SEQ_Q1 : SEQ_Q0, 0, g.qs, g.qe - g.qs, 0 };
			j.t = SeqRef{ SEQ_REF, rid, g.rs, g.re - g.rs, 0 };
			j.w = g.bw1, j.end_bonus = -1, j.zdrop = zdrop_code == 2 ? opt->zdrop_inv : opt->zdrop, j.flag = ez_splice_flag(opt, A);
			A.pending_job = (int)sink.dp.size();
			sink.dp.push_back(j);
			A.zd_max_zdrop = zdrop_code;
			A.state = 3;
			return false;
		} else { ez = g.res; ez.cigar = A.cig_pool.data() + g.cig_off; }
		// :739-765
		const double w1 = sub_w ? Timers::now() : 0;
		if (ez.n_cigar > 0) append_cigar(r, ez.n_cigar, ez.cigar);
		if (sub_w) g_timers.add("walk.append", Timers::now() - w1);
		if (ez.zdropped) {
			if (!r->p) {
				uint32_t capacity = round_up_pow2((uint32_t)(sizeof(wm_extra_t) / 4));
				r->p = (wm_extra_t*)calloc(capacity, 4);
				r->p->capacity = capacity;
			}
			int j;
			for (j = g.i - 1; j >= 0; --j)
				if ((int32_t)a[A.as1 + j].x <= g.rs + ez.max_t) break;
			A.dropped = true;
			if (j < 0) j = 0;
			r->p->dp_score += ez.max;
			A.re1 = g.rs + (ez.max_t + 1);
			A.qe1 = g.qs + (ez.max_q + 1);
			if (A.cnt1 - (j + 1) >= opt->min_cnt) {
				split_reg(r, &A.r2, A.as1 + j + 1 - r->as, qlen, a);
				if (zdrop_code == 2) A.r2.split_inv = 1;
			}
			break;
		} else r->p->dp_score += ez.score;
		++A.gap_cur;
	}
	if (!A.dropped) {
		A.re1 = A.re, A.qe1 = A.qe; // :715 re1/qe1 follow the last seed
		if (A.right_job >= 0) { // :767-778
			DpRes ez = A.right_res; ez.cigar = A.cig_pool.data() + A.right_cig;
			if (ez.n_cigar > 0) { append_cigar(r, ez.n_cigar, ez.cigar); r->p->dp_score += ez.max; }
			A.re1 = A.re + (ez.reach_end ? ez.mqe_t + 1 : ez.max_t + 1);
			A.qe1 = A.qe + (ez.reach_end ? A.qe0 - A.qe : ez.max_q + 1);
		}
	}
	// :781-793
	r->rs = A.rs1, r->re = A.re1;
	if (rev) r->qs = qlen - A.qe1, r->qe = qlen - A.qs1;
	else r->qs = A.qs1, r->qe = A.qe1;
	if (r->p) {
		static const bool sub_t2 = getenv("WM_SUBTIMING") != 0;
		const double q0 = sub_t2 ? Timers::now() : 0;
		tbuf.resize(A.re1 > A.rs1 ? A.re1 - A.rs1 : 0);
		if (A.re1 > A.rs1) mi->getseq(rid, A.rs1, A.re1, tbuf.data());
		update_extra(r, qseq(r->rev) + A.qs1, tbuf.data(), mat, (int8_t)opt->q, (int8_t)opt->e, (int)(opt->flag & WM_F_EQX));
		if (rev && r->p->trans_strand) r->p->trans_strand ^= 3; // :789-790, before mm_align_skeleton sets it
		if (sub_t2) g_timers.add("adv.update_extra", Timers::now() - q0);
	}
	A.state = 9;
	return true;
}

// Phase 2: the loop of mm_align_skeleton (:882-911) replayed over `out`; hits aligned in phase 1 are taken
// as they are, split children are aligned here one at a time, inversions are tested in the same order.
bool AlignTask::step_phase2(const DpRes *dp, const LlRes *ll, JobSink &sink)
{
	for (;;) {
		if (cur >= out.size()) return true;
		if (sub == 0) {
			if (from_first[cur]) { sub = 4; }
			else {
				start_rounds(out[cur], child, sink);
				sub = 5;
				if (ends_pending(child[0])) return false;
			}
		}
		if (sub == 5) {
			plan_rounds(child, ll, sink);
			sub = 1;
			bool planned = true;
			for (int k = 0; k < n_round; ++k) if (child[k].state != 9) planned = false;
			if (!planned) return false;
		}
		if (sub == 1) {
			bool done = true;
			for (int k = 0; k < n_round; ++k) if (!walk1(child[k], dp, ll, sink)) done = false;
			if (!done) return false;
			wm_reg1_t r2;
			pick_round(child, &out[cur], &r2);
			if (r2.cnt > 0) { out.insert(out.begin() + cur + 1, r2); from_first.insert(from_first.begin() + cur + 1, 0); }
			sub = 4;
		}
		if (sub == 4) { // inversion test against the element just before (:907-912)
			sub = 0;
			if (cur > 0 && out[cur].split_inv) {
				const wm_reg1_t *r1 = &out[cur - 1], *r2 = &out[cur];
				bool ok = (r1->split & 1) && (r2->split & 2);
				if (ok && r1->id != r1->parent && r1->parent != WM_PARENT_TMP_PRI) ok = false;
				if (ok && r2->id != r2->parent && r2->parent != WM_PARENT_TMP_PRI) ok = false;
				if (ok && (r1->rid != r2->rid || r1->rev != r2->rev)) ok = false;
				int ql = 0, tl = 0;
				if (ok) {
					ql = r1->rev ? r1->qs - r2->qe : r2->qs - r1->qe;
					tl = r2->rs - r1->re;
					if (ql < opt->min_chain_score || ql > opt->max_gap) ok = false;
					if (tl < opt->min_chain_score || tl > opt->max_gap) ok = false;
				}
				if (ok) { // :814-823: local SW of the reversed gap sequences
					inv_ql = ql, inv_tl = tl;
					LlJob j;
					j.task = task_id;
					j.q = r1->rev ? SeqRef{ SEQ_Q0, 0, r2->qe, ql, 1 } : SeqRef{ SEQ_Q1, 0, (int64_t)qlen - r2->qs, ql, 1 };
					j.t = SeqRef{ SEQ_REF, r1->rid, r1->re, tl, 1 };
					inv_job = (int)sink.ll.size();
					sink.ll.push_back(j);
					sub = 2;
					return false;
				}
			}
			++cur;
			continue;
		}
		if (sub == 2) {
			const LlRes &lr = ll[inv_job];
			const wm_reg1_t *r1 = &out[cur - 1], *r2 = &out[cur];
			if (lr.score < opt->min_dp_max) { sub = 0; ++cur; continue; }
			inv_qoff = inv_ql - (lr.qe + 1), inv_toff = inv_tl - (lr.te + 1);
			DpJob j;
			j.task = task_id;
			const int64_t qbase = r1->rev ? r2->qe : (int64_t)qlen - r2->qs;
			j.q = SeqRef{ r1->rev ? SEQ_Q0 : SEQ_Q1, 0, qbase + inv_qoff, inv_ql - inv_qoff, 0 };
			j.t = SeqRef{ SEQ_REF, r1->rid, (int64_t)r1->re + inv_toff, inv_tl - inv_toff, 0 };
			j.w = (int)(opt->bw * 1.5), j.end_bonus = -1, j.zdrop = opt->zdrop, j.flag = EZ_EXTZ_ONLY;
			inv_job = (int)sink.dp.size();
			sink.dp.push_back(j);
			sub = 3;
			return false;
		}
		if (sub == 3) { // :829-849
			const DpRes &ez = dp[inv_job];
			const wm_reg1_t r1 = out[cur - 1], r2 = out[cur];
			sub = 0;
			if (ez.n_cigar == 0) { ++cur; continue; }
			wm_reg1_t r_inv;
			memset(&r_inv, 0, sizeof(r_inv));
			append_cigar(&r_inv, ez.n_cigar, ez.cigar);
			r_inv.p->dp_score = ez.max;
			r_inv.id = -1;
			r_inv.parent = WM_PARENT_UNSET;
			r_inv.inv = 1;
			r_inv.rev = !r1.rev;
			r_inv.rid = r1.rid;
			r_inv.div = -1.0f;
			if (r_inv.rev == 0) {
				r_inv.qs = r2.qe + inv_qoff;
				r_inv.qe = r_inv.qs + ez.max_q + 1;
			} else {
				r_inv.qe = r2.qs - inv_qoff;
				r_inv.qs = r_inv.qe - (ez.max_q + 1);
			}
			r_inv.rs = r1.re + inv_toff;
			r_inv.re = r_inv.rs + ez.max_t + 1;
			{
				const int64_t qbase = r1.rev ? r2.qe : (int64_t)qlen - r2.qs;
				const uint8_t *qp = qseq(r1.rev ? 0 : 1) + qbase + inv_qoff;
				std::vector<uint8_t> tbuf(inv_tl - inv_toff);
				mi->getseq(r1.rid, r1.re + inv_toff, r1.re + inv_tl, tbuf.data());
				update_extra(&r_inv, qp, tbuf.data(), mat, (int8_t)opt->q, (int8_t)opt->e, (int)(opt->flag & WM_F_EQX));
			}
			out.insert(out.begin() + cur + 1, r_inv);
			from_first.insert(from_first.begin() + cur + 1, 1);
			cur += 2; // skip the inserted INV alignment
			continue;
		}
	}
}

bool AlignTask::advance(const DpRes *dp, const LlRes *ll, JobSink &sink)
{
	static const bool sub_t = getenv("WM_SUBTIMING") != 0;
	if (phase == 0) {
		const double q0 = sub_t ? Timers::now() : 0;
		firsts.resize(regs.size() * n_round);
		bool wait = false;
		for (size_t i = 0; i < regs.size(); ++i) {
			start_rounds(regs[i], &firsts[i * n_round], sink);
			wait = wait || ends_pending(firsts[i * n_round]);
		}
		phase = 4;
		if (sub_t) g_timers.add("adv.phase0", Timers::now() - q0);
		if (wait) return false;
	}
	if (phase == 4) {
		const double q0 = sub_t ? Timers::now() : 0;
		for (size_t i = 0; i < regs.size(); ++i) plan_rounds(&firsts[i * n_round], ll, sink);
		phase = 1;
		bool all = true;
		for (auto &A : firsts) if (A.state != 9) all = false;
		if (sub_t) g_timers.add("adv.phase0", Timers::now() - q0);
		if (!all) return false;
	}
	if (phase == 1) {
		const double q0 = sub_t ? Timers::now() : 0;
		bool all = true;
		for (auto &A : firsts) if (!walk1(A, dp, ll, sink)) all = false;
		if (sub_t) g_timers.add("adv.walk1", Timers::now() - q0);
		if (!all) return false;
		out.clear(); from_first.clear();
		for (size_t i = 0; i < firsts.size(); i += n_round) {
			wm_reg1_t r, r2;
			pick_round(&firsts[i], &r, &r2);
			out.push_back(r); from_first.push_back(1);
			if (r2.cnt > 0) { out.push_back(r2); from_first.push_back(0); }
		}
		firsts.clear();
		phase = 2; cur = 0; sub = 0;
	}
	if (phase == 2) {
		const double q0 = sub_t ? Timers::now() : 0;
		const bool fin = step_phase2(dp, ll, sink);
		if (sub_t) g_timers.add("adv.phase2", Timers::now() - q0);
		if (!fin) return false;
		regs.swap(out);
		filter_regs(opt, qlen, regs); // :916-917
		hit_sort(regs, opt->alt_drop);
		phase = 3;
	}
	return true;
}

} // namespace wmh
