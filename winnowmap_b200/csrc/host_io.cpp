// Host side of the drop-in: option presets (reference src/options.c), FASTA/FASTQ reading with the
// reference's batching rule (src/bseq.c:80-119), index construction (src/index.c:378-449, with the reference
// sketch computed by the same CUDA sketch kernel the mapper uses), PAF output (src/format.c:266-334) and the
// batch loop of mm_map_file (src/map.c:1107-1224) with kt_for(worker_for) replaced by GPU batch dispatch.
#include <errno.h>
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <zlib.h>
#include <algorithm>
#include <chrono>
#include <fstream>
#include <functional>
#include <limits.h>
#include <sstream>
#include "host_io.h"

namespace wmh {

static double now_s() { return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count(); }

// ---------------- options (src/options.c) ----------------
void idxopt_init(wm_idxopt_t *o)
{ // mm_idxopt_init :5-12
	memset(o, 0, sizeof(*o));
	o->k = 15, o->w = 50, o->flag = 0, o->bucket_bits = 14;
	o->mini_batch_size = 50000000;
	o->batch_size = 4000000000ULL;
}

void mapopt_init(wm_mapopt_t *o)
{ // mm_mapopt_init :14-69
	memset(o, 0, sizeof(*o));
	o->seed = 11;
	o->mid_occ_frac = -1.0f;
	o->mid_occ = 5000;
	o->sdust_thres = 0;
	o->min_cnt = 3, o->min_chain_score = 40, o->bw = 500, o->max_gap = 5000, o->min_gap_ref = 1000, o->max_gap_ref = -1;
	o->max_chain_skip = 25, o->max_chain_iter = 5000, o->chain_gap_scale = 1.0f;
	o->mask_level = 0.5f, o->mask_len = INT_MAX, o->pri_ratio = 0.8f, o->best_n = 5;
	o->max_join_long = 20000, o->max_join_short = 2000, o->min_join_flank_sc = 1000, o->min_join_flank_ratio = 0.5f;
	o->a = 2, o->b = 4, o->q = 4, o->e = 2, o->q2 = 24, o->e2 = 1;
	o->sc_ambi = 1;
	o->zdrop = 400, o->zdrop_inv = 200;
	o->end_bonus = -1;
	o->min_dp_max = o->min_chain_score * o->a;
	o->min_ksw_len = 200;
	o->anchor_ext_len = 20, o->anchor_ext_shift = 6;
	o->max_clip_ratio = 1.0f;
	o->mini_batch_size = 1000000000;
	o->pe_ori = 0, o->pe_bonus = 33;
	o->maxPrefixLength = 16000;
	o->minPrefixLength = o->suffixSampleOffset = 2000;
	o->prefixIncrementFactor = std::pow((o->maxPrefixLength - 1) * 1.0 / o->minPrefixLength, 0.5);
	o->min_mapq = 5;
	o->min_qcov = 0.5;
	o->SVaware = true;
	o->SVawareMinReadLength = 10000;
	o->stage2_zdrop_inv = 25, o->stage2_bw = 2000, o->stage2_max_gap = o->maxPrefixLength, o->stage2_extension_inc = 1;
}

int set_opt(const char *preset, wm_idxopt_t *io, wm_mapopt_t *mo)
{ // mm_set_opt :89-131 (the splice presets map without base alignment: check_opt refuses them with MM_F_CIGAR)
	if (preset == 0) { idxopt_init(io); mapopt_init(mo); }
	else if (strcmp(preset, "map-ont") == 0) { io->flag = 0, io->k = 15; }
	else if (strcmp(preset, "map-pb") == 0) {
		io->flag = 0, io->k = 15;
		mo->maxPrefixLength = mo->stage2_max_gap = 8000;
		mo->suffixSampleOffset = mo->minPrefixLength = 1000;
		mo->stage2_bw = 1000;
		mo->prefixIncrementFactor = std::pow((mo->maxPrefixLength - 1) * 1.0 / mo->minPrefixLength, 0.33);
	} else if (strcmp(preset, "map-pb-clr") == 0) mo->SVaware = false;
	else if (strcmp(preset, "asm5") == 0) {
		io->flag = 0, io->k = 19;
		mo->a = 1, mo->b = 19, mo->q = 39, mo->q2 = 81, mo->e = 3, mo->e2 = 1, mo->zdrop = mo->zdrop_inv = 200;
		mo->min_dp_max = 200;
	} else if (strcmp(preset, "asm10") == 0) {
		io->flag = 0, io->k = 19;
		mo->a = 1, mo->b = 9, mo->q = 16, mo->q2 = 41, mo->e = 2, mo->e2 = 1, mo->zdrop = mo->zdrop_inv = 200;
		mo->min_dp_max = 200;
	} else if (strcmp(preset, "asm20") == 0) {
		io->flag = 0, io->k = 19;
		mo->a = 1, mo->b = 4, mo->q = 6, mo->q2 = 26, mo->e = 2, mo->e2 = 1, mo->zdrop = mo->zdrop_inv = 200;
		mo->min_dp_max = 200;
	} else if (strncmp(preset, "splice", 6) == 0 || strcmp(preset, "cdna") == 0) { // "splice:<anything>" is "splice"
		mo->SVaware = false;
		io->w = 25;
		io->flag = 0, io->k = 15;
		mo->flag |= WM_F_SPLICE | WM_F_SPLICE_FOR | WM_F_SPLICE_REV | WM_F_SPLICE_FLANK;
		mo->max_gap = 2000, mo->max_gap_ref = mo->bw = 200000;
		mo->a = 1, mo->b = 2, mo->q = 2, mo->e = 1, mo->q2 = 32, mo->e2 = 0;
		mo->noncan = 9;
		mo->junc_bonus = 9;
		mo->zdrop = 200, mo->zdrop_inv = 100;
		if (strcmp(preset, "splice:hq") == 0) mo->junc_bonus = 5, mo->b = 4, mo->q = 6, mo->q2 = 24;
	} else return -1;
	return 0;
}

void mapopt_max_intron_len(wm_mapopt_t *opt, int max_intron_len)
{ // mm_mapopt_max_intron_len :83-87 (-G): only once MM_F_SPLICE is set
	if ((opt->flag & WM_F_SPLICE) && max_intron_len > 0) opt->max_gap_ref = opt->bw = max_intron_len;
}

int check_opt(const wm_idxopt_t *io, const wm_mapopt_t *mo)
{ // mm_check_opt :133-188 (same return codes)
	if (mo->split_prefix && (mo->flag & (WM_F_OUT_CS | WM_F_OUT_MD))) return -6;
	if (io->k <= 0 || io->w <= 0) return -5;
	if (io->k > 28 || io->w >= 256) return -5; // the sketch asserts 0 < w < 256 && 0 < k <= 28 (src/sketch.c:140); refused here instead of aborting later
	if (mo->best_n < 0) return -4;
	if (mo->pri_ratio < 0.0f || mo->pri_ratio > 1.0f) return -4;
	if ((mo->flag & WM_F_FOR_ONLY) && (mo->flag & WM_F_REV_ONLY)) return -3;
	if (mo->e <= 0 || mo->q <= 0) return -1;
	if ((mo->q != mo->q2 || mo->e != mo->e2) && !(mo->e > mo->e2 && mo->q + mo->e < mo->q2 + mo->e2)) return -2;
	if ((mo->q + mo->e) + (mo->q2 + mo->e2) > 127) return -1;
	// Not in the reference.  With two gap pairs (q + e < q2 + e2 by the check above), ksw_extd2_sse's int8 lanes wrap once
	// a - z + q can fall below -128 (src/ksw2_extd2_sse.c:52-58, with x, v >= -(q + e) and the score difference z <= -A),
	// i.e. when -A + q + 2e > 128.  The device fill keeps these values in 16 bits and does not wrap, so it would silently
	// differ from the reference: such scorings are refused.  (ksw_extz2, one gap pair, wraps as the reference does.)
	if ((mo->q != mo->q2 || mo->e != mo->e2) && mo->a + mo->q + 2 * mo->e > 128) return -7;
	if (mo->zdrop < mo->zdrop_inv) return -5;
	if ((mo->flag & WM_F_NO_PRINT_2ND) && (mo->flag & WM_F_ALL_CHAINS)) return -5;
	// Not in the reference: spliced base alignment (splice with -c / -a) is a library / boundary path (wm_gpu_map_batch,
	// wm_map_file, Mapper(spliced_alignment=True)); the command line refuses it until its refusal tests are retired.
	if ((mo->flag & WM_F_SPLICE) && (mo->flag & WM_F_CIGAR)) return -8;
	return 0;
}

// ---------------- FASTA / FASTQ (plain or gzip) ----------------
struct SeqReader::Impl {
	gzFile fp;
	std::vector<char> buf; size_t beg, end; bool eof;
	int last_char; // header character already consumed for the next record (0 if none)
	Impl() : fp(0), beg(0), end(0), eof(false), last_char(0) { buf.resize(1 << 20); }
	int getc_() {
		if (beg >= end) {
			if (eof) return -1;
			int n = gzread(fp, buf.data(), (unsigned)buf.size());
			if (n <= 0) { eof = true; return -1; }
			beg = 0, end = (size_t)n;
		}
		return (unsigned char)buf[beg++];
	}
	// read up to (not including) newline; returns false at EOF with nothing read
	bool getline_(std::string &s, bool append) {
		if (!append) s.clear();
		bool any = false;
		for (;;) {
			if (beg >= end) { int c = getc_(); if (c < 0) return any; --beg; }
			any = true;
			char *p = buf.data() + beg, *e = buf.data() + end;
			char *nl = (char*)memchr(p, '\n', e - p);
			if (nl) { s.append(p, nl - p); beg = (nl - buf.data()) + 1; break; }
			s.append(p, e - p); beg = end;
		}
		if (!s.empty() && s.back() == '\r') s.pop_back();
		return true;
	}
};

SeqReader::SeqReader() : p(new Impl()) {}
SeqReader::~SeqReader() { if (p->fp) gzclose(p->fp); delete p; }
bool SeqReader::open(const char *fn)
{
	p->fp = (fn == 0 || strcmp(fn, "-") == 0) ? gzdopen(0, "r") : gzopen(fn, "r");
	if (p->fp) gzbuffer(p->fp, 1 << 18);
	return p->fp != 0;
}

bool SeqReader::next_line(std::string &s) { return p->getline_(s, false); }

// one record with kseq semantics (src/kseq.h): name up to the first white space, rest of the header line is the
// comment; sequence lines are concatenated; '+' starts the quality of a FASTQ record
bool SeqReader::next(wm_read &r)
{
	Impl &I = *p;
	int c;
	if (I.last_char == 0) {
		while ((c = I.getc_()) >= 0 && c != '>' && c != '@') {}
		if (c < 0) return false;
	}
	I.last_char = 0;
	std::string hdr;
	I.getline_(hdr, false);
	size_t sp = 0;
	while (sp < hdr.size() && !isspace((unsigned char)hdr[sp])) ++sp;
	r.name.assign(hdr, 0, sp);
	size_t cs = sp;
	while (cs < hdr.size() && isspace((unsigned char)hdr[cs])) ++cs;
	r.comment.assign(hdr, cs, std::string::npos);
	r.seq.clear(); r.qual.clear();
	std::string line;
	for (;;) {
		c = I.getc_();
		if (c < 0) break;
		if (c == '>' || c == '@') { I.last_char = c; break; }
		if (c == '+') { // FASTQ: skip the rest of the '+' line, then read as many quality characters as bases
			I.getline_(line, false);
			while (r.qual.size() < r.seq.size()) { if (!I.getline_(line, false)) break; r.qual += line; }
			break;
		}
		if (c == '\n') continue;
		--I.beg; // put back
		I.getline_(r.seq, true);
	}
	for (char &ch : r.seq) if (ch == 'u' || ch == 'U') --ch; // src/bseq.c:73-75
	return true;
}

// ---------------- index construction ----------------
static uint64_t encode_kmer(const std::string &s)
{ // encodeKmer, src/index.c:362-376
	uint64_t kmer[2] = {0, 0};
	const int k = (int)s.size();
	const uint64_t shift1 = 2 * (k - 1);
	for (int i = 0; i < k; ++i) {
		int c;
		switch (s[i]) { case 'A': case 'a': c = 0; break; case 'C': case 'c': c = 1; break; case 'G': case 'g': c = 2; break;
			case 'T': case 't': case 'U': case 'u': c = 3; break; default: c = 4; }
		kmer[0] = kmer[0] << 2 | (uint64_t)c;
		kmer[1] = (kmer[1] >> 2) | (3ULL ^ (uint64_t)c) << shift1;
	}
	return kmer[0] < kmer[1] ? kmer[0] : kmer[1];
}

int read_kmer_list(const char *fn, int k, std::vector<uint64_t> &out)
{ // src/index.c:390-432: "kmer count" pairs; an unreadable / absent file yields an empty list
	out.clear();
	if (fn == 0) return 0;
	std::ifstream idt(fn);
	std::string kmer; uint64_t freq;
	while (idt >> kmer >> freq) out.push_back(encode_kmer(kmer));
	// like the reference (:399-406), only the LAST k-mer read is checked against k; entries of another length are
	// encoded over their own length, as encodeKmer does
	if (!out.empty() && (int)kmer.size() != k) {
		fprintf(stderr, "ERROR: input list of k-mers and winnowmap parameter k are inconsistent\n");
		return -1;
	}
	return 0;
}

} // namespace wmh
