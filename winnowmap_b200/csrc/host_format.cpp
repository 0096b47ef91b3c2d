// PAF and SAM output, byte-identical to the reference writers (src/format.c:266-334 and :341-548; tags :280-306).
#include <stdio.h>
#include <string.h>
#include <vector>
#include "host_io.h"

namespace wmh {

static inline void put_int(std::string &s, int c)
{ // the %d of mm_sprintf_lite (src/format.c:36-44)
	char buf[16]; int l = 0;
	unsigned x = c >= 0 ? c : -c;
	do { buf[l++] = x % 10 + '0'; x /= 10; } while (x > 0);
	if (c < 0) buf[l++] = '-';
	while (l > 0) s.push_back(buf[--l]);
}

static double event_identity(const wm_reg1_t *r)
{ // mm_event_identity (src/format.c:267-278)
	int32_t n_gapo = 0, n_gap = 0;
	if (r->p == 0) return -1.0f;
	for (uint32_t i = 0; i < r->p->n_cigar; ++i) {
		int32_t op = r->p->cigar[i] & 0xf, len = r->p->cigar[i] >> 4;
		if (op == 1 || op == 2) ++n_gapo, n_gap += len;
	}
	return (double)r->mlen / (r->blen + r->p->n_ambi - n_gap + n_gapo);
}

static void write_tags(std::string &s, const wm_reg1_t *r)
{ // src/format.c:280-306
	int type;
	if (r->id == r->parent) type = r->inv ? 'I' : 'P';
	else type = r->inv ? 'i' : 'S';
	if (r->p) {
		s += "\tNM:i:"; put_int(s, r->blen - r->mlen + r->p->n_ambi);
		s += "\tms:i:"; put_int(s, r->p->dp_max);
		s += "\tAS:i:"; put_int(s, r->p->dp_score);
		s += "\tnn:i:"; put_int(s, r->p->n_ambi);
		if (r->p->trans_strand == 1 || r->p->trans_strand == 2) { s += "\tts:A:"; s.push_back("?+-?"[r->p->trans_strand]); }
	}
	s += "\ttp:A:"; s.push_back((char)type);
	s += "\tcm:i:"; put_int(s, r->cnt);
	s += "\ts1:i:"; put_int(s, r->score);
	if (r->parent == r->id) { s += "\ts2:i:"; put_int(s, r->subsc); }
	if (r->p) {
		char buf[16];
		double div = 1.0 - event_identity(r);
		if (div == 0.0) buf[0] = '0', buf[1] = 0;
		else snprintf(buf, 16, "%.4f", 1.0 - event_identity(r));
		s += "\tde:f:"; s += buf;
	} else if (r->div >= 0.0f && r->div <= 1.0f) {
		char buf[16];
		if (r->div == 0.0f) buf[0] = '0', buf[1] = 0;
		else snprintf(buf, 16, "%.4f", r->div);
		s += "\tdv:f:"; s += buf;
	}
	if (r->split) { s += "\tzd:i:"; put_int(s, r->split); }
}

// cs:Z: / MD:Z: difference strings (src/format.c:141-243); qseq/tseq are 0..4 codes in alignment orientation
static void write_cs_core(std::string &s, const uint8_t *tseq, const uint8_t *qseq, const wm_reg1_t *r, int no_iden, int write_tag)
{
	if (write_tag) s += "\tcs:Z:";
	int q_off = 0, t_off = 0;
	std::string tmp;
	for (uint32_t i = 0; i < r->p->n_cigar; ++i) {
		const int op = r->p->cigar[i] & 0xf, len = r->p->cigar[i] >> 4;
		if (op == 0 || op == 7 || op == 8) {
			tmp.clear();
			auto flush = [&]() {
				if (tmp.empty()) return;
				if (!no_iden) { s.push_back('='); s += tmp; } else { s.push_back(':'); put_int(s, (int)tmp.size()); }
				tmp.clear();
			};
			for (int j = 0; j < len; ++j) {
				if (qseq[q_off + j] != tseq[t_off + j]) {
					flush();
					s.push_back('*'); s.push_back("acgtn"[tseq[t_off + j]]); s.push_back("acgtn"[qseq[q_off + j]]);
				} else tmp.push_back("ACGTN"[qseq[q_off + j]]);
			}
			flush();
			q_off += len, t_off += len;
		} else if (op == 1) {
			s.push_back('+');
			for (int j = 0; j < len; ++j) s.push_back("acgtn"[qseq[q_off + j]]);
			q_off += len;
		} else if (op == 2) {
			s.push_back('-');
			for (int j = 0; j < len; ++j) s.push_back("acgtn"[tseq[t_off + j]]);
			t_off += len;
		} else { // intron
			s.push_back('~'); s.push_back("acgtn"[tseq[t_off]]); s.push_back("acgtn"[tseq[t_off + 1]]); put_int(s, len);
			s.push_back("acgtn"[tseq[t_off + len - 2]]); s.push_back("acgtn"[tseq[t_off + len - 1]]);
			t_off += len;
		}
	}
}

static void write_MD_core(std::string &s, const uint8_t *tseq, const uint8_t *qseq, const wm_reg1_t *r, int write_tag)
{
	if (write_tag) s += "\tMD:Z:";
	int q_off = 0, t_off = 0, l_MD = 0;
	for (uint32_t i = 0; i < r->p->n_cigar; ++i) {
		const int op = r->p->cigar[i] & 0xf, len = r->p->cigar[i] >> 4;
		if (op == 0 || op == 7 || op == 8) {
			for (int j = 0; j < len; ++j) {
				if (qseq[q_off + j] != tseq[t_off + j]) { put_int(s, l_MD); s.push_back("ACGTN"[tseq[t_off + j]]); l_MD = 0; }
				else ++l_MD;
			}
			q_off += len, t_off += len;
		} else if (op == 1) q_off += len;
		else if (op == 2) {
			put_int(s, l_MD); s.push_back('^');
			for (int j = 0; j < len; ++j) s.push_back("ACGTN"[tseq[t_off + j]]);
			l_MD = 0;
			t_off += len;
		} else if (op == 3) t_off += len;
	}
	if (l_MD > 0) put_int(s, l_MD);
}

static void write_cs_or_MD(std::string &s, const wm_host_idx *mi, const char *seq, const wm_reg1_t *r, int no_iden, int is_MD, int write_tag)
{ // src/format.c:220-243
	if (r->p == 0) return;
	static const struct Nt4 { uint8_t t[256]; Nt4() { for (int i = 0; i < 256; ++i) t[i] = 4; t[0] = t['A'] = t['a'] = 0; t[1] = t['C'] = t['c'] = 1;
		t[2] = t['G'] = t['g'] = 2; t[3] = t['T'] = t['t'] = t['U'] = t['u'] = 3; } } nt4;
	std::vector<uint8_t> qseq(r->qe - r->qs), tseq(r->re - r->rs);
	mi->getseq(r->rid, r->rs, r->re, tseq.data());
	if (!r->rev) for (int i = r->qs; i < r->qe; ++i) qseq[i - r->qs] = nt4.t[(uint8_t)seq[i]];
	else for (int i = r->qs; i < r->qe; ++i) { const uint8_t c = nt4.t[(uint8_t)seq[i]]; qseq[r->qe - i - 1] = c >= 4 ? 4 : 3 - c; }
	if (is_MD) write_MD_core(s, tseq.data(), qseq.data(), r, write_tag);
	else write_cs_core(s, tseq.data(), qseq.data(), r, no_iden, write_tag);
}

void write_paf(std::string &s, const wm_host_idx *mi, const wm_read *t, const wm_reg1_t *r, int64_t opt_flag, int rep_len)
{
	s.clear();
	if (r == 0) {
		s += t->name; s.push_back('\t'); put_int(s, (int)t->seq.size());
		s += "\t0\t0\t*\t*\t0\t0\t0\t0\t0\t0";
		if (rep_len >= 0) { s += "\trl:i:"; put_int(s, rep_len); }
		return;
	}
	s += t->name; s.push_back('\t'); put_int(s, (int)t->seq.size()); s.push_back('\t'); put_int(s, r->qs); s.push_back('\t'); put_int(s, r->qe);
	s.push_back('\t'); s.push_back("+-"[r->rev]); s.push_back('\t');
	s += mi->name[r->rid];
	s.push_back('\t'); put_int(s, (int)mi->len[r->rid]); s.push_back('\t'); put_int(s, r->rs); s.push_back('\t'); put_int(s, r->re);
	s.push_back('\t'); put_int(s, r->mlen); s.push_back('\t'); put_int(s, r->blen);
	s.push_back('\t'); put_int(s, (int)r->mapq);
	write_tags(s, r);
	if (rep_len >= 0) { s += "\trl:i:"; put_int(s, rep_len); }
	if (r->p && (opt_flag & WM_F_OUT_CG)) {
		s += "\tcg:Z:";
		for (uint32_t k = 0; k < r->p->n_cigar; ++k) { put_int(s, (int)(r->p->cigar[k] >> 4)); s.push_back("MIDNSHP=XB"[r->p->cigar[k] & 0xf]); }
	}
	if (r->p && (opt_flag & (WM_F_OUT_CS | WM_F_OUT_MD))) write_cs_or_MD(s, mi, t->seq.data(), r, !(opt_flag & WM_F_OUT_CS_LONG), (opt_flag & WM_F_OUT_MD) != 0, 1);
	if ((opt_flag & WM_F_COPY_COMMENT) && !t->comment.empty()) { s.push_back('\t'); s += t->comment; }
}

// seq_comp_table (src/bseq.c): IUPAC complement, case preserved; bytes without a complement map to themselves
static const struct CompTable {
	unsigned char t[256];
	CompTable() {
		for (int i = 0; i < 256; ++i) t[i] = (unsigned char)i;
		const char *a = "ACGTUMRWSYKVHDBN", *b = "TGCAAKYWSRMBDHVN";
		for (int i = 0; a[i]; ++i) { t[(unsigned char)a[i]] = (unsigned char)b[i]; t[(unsigned char)(a[i] + 32)] = (unsigned char)(b[i] + 32); }
	}
} g_comp;

static void sam_write_sq(std::string &s, const char *seq, int l, int rev, int comp)
{ // src/format.c:341-353
	if (rev) {
		for (int i = 0; i < l; ++i) {
			const int c = (unsigned char)seq[l - 1 - i];
			s.push_back((char)(c < 128 && comp ? g_comp.t[c] : c));
		}
	} else s.append(seq, seq + l);
}

static void write_sam_cigar(std::string &s, int sam_flag, int in_tag, int qlen, const wm_reg1_t *r, int64_t opt_flag)
{ // src/format.c:365-389
	if (r->p == 0) { s.push_back('*'); return; }
	uint32_t clip_len[2];
	clip_len[0] = r->rev ? qlen - r->qe : r->qs;
	clip_len[1] = r->rev ? r->qs : qlen - r->qe;
	if (in_tag) {
		const int clip_char = (sam_flag & 0x800) && !(opt_flag & WM_F_SOFTCLIP) ? 5 : 4;
		s += "\tCG:B:I";
		if (clip_len[0]) { s.push_back(','); put_int(s, (int)(clip_len[0] << 4 | clip_char)); }
		for (uint32_t k = 0; k < r->p->n_cigar; ++k) { s.push_back(','); put_int(s, (int)r->p->cigar[k]); }
		if (clip_len[1]) { s.push_back(','); put_int(s, (int)(clip_len[1] << 4 | clip_char)); }
	} else {
		const char clip_char = (sam_flag & 0x800) && !(opt_flag & WM_F_SOFTCLIP) ? 'H' : 'S';
		if (clip_len[0]) { put_int(s, (int)clip_len[0]); s.push_back(clip_char); }
		for (uint32_t k = 0; k < r->p->n_cigar; ++k) { put_int(s, (int)(r->p->cigar[k] >> 4)); s.push_back("MIDNSHP=XB"[r->p->cigar[k] & 0xf]); }
		if (clip_len[1]) { put_int(s, (int)clip_len[1]); s.push_back(clip_char); }
	}
}

// mm_write_sam3 (src/format.c:391-548) for a single-segment read (n_seg == 1); reg_idx < 0 writes the unmapped record.
// rg_id is the @RG ID ("" = none).
void write_sam(std::string &s, const wm_host_idx *mi, const wm_read *t, int reg_idx, int n_regs, const wm_reg1_t *regs, int64_t opt_flag, int rep_len,
               const char *rg_id)
{
	const int max_bam_cigar_op = 65535;
	const int l_seq = (int)t->seq.size();
	const wm_reg1_t *r = n_regs > 0 && reg_idx < n_regs && reg_idx >= 0 ? &regs[reg_idx] : 0;
	int flag = 0, cigar_in_tag = 0;
	s.clear();
	s += t->name;
	if (r == 0) flag |= 0x4;
	else {
		if (r->rev) flag |= 0x10;
		if (r->parent != r->id) flag |= 0x100;
		else if (!r->sam_pri) flag |= 0x800;
	}
	s.push_back('\t'); put_int(s, flag);
	if (r == 0) s += "\t*\t0\t0\t*";
	else {
		s.push_back('\t'); s += mi->name[r->rid]; s.push_back('\t'); put_int(s, r->rs + 1); s.push_back('\t'); put_int(s, (int)r->mapq); s.push_back('\t');
		if ((opt_flag & WM_F_LONG_CIGAR) && r->p && (int)r->p->n_cigar > max_bam_cigar_op - 2) {
			int n_cigar = (int)r->p->n_cigar;
			if (r->qs != 0) ++n_cigar;
			if (r->qe != l_seq) ++n_cigar;
			if (n_cigar > max_bam_cigar_op) cigar_in_tag = 1;
		}
		if (cigar_in_tag) {
			int slen;
			if ((flag & 0x900) == 0 || (opt_flag & WM_F_SOFTCLIP)) slen = l_seq;
			else if (flag & 0x100) slen = 0;
			else slen = r->qe - r->qs;
			put_int(s, slen); s.push_back('S'); put_int(s, r->re - r->rs); s.push_back('N');
		} else write_sam_cigar(s, flag, 0, l_seq, r, opt_flag);
	}
	s += "\t*\t0\t0\t";
	const char *seq = t->seq.data(), *qual = t->qual.empty() ? 0 : t->qual.data();
	if (r == 0) {
		sam_write_sq(s, seq, l_seq, 0, 0);
		s.push_back('\t');
		if (qual) sam_write_sq(s, qual, l_seq, 0, 0); else s.push_back('*');
	} else if ((flag & 0x900) == 0 || (opt_flag & WM_F_SOFTCLIP)) {
		sam_write_sq(s, seq, l_seq, r->rev, r->rev);
		s.push_back('\t');
		if (qual) sam_write_sq(s, qual, l_seq, r->rev, 0); else s.push_back('*');
	} else if (flag & 0x100) {
		s += "*\t*";
	} else {
		sam_write_sq(s, seq + r->qs, r->qe - r->qs, r->rev, r->rev);
		s.push_back('\t');
		if (qual) sam_write_sq(s, qual + r->qs, r->qe - r->qs, r->rev, 0); else s.push_back('*');
	}
	if (rg_id && rg_id[0]) { s += "\tRG:Z:"; s += rg_id; }
	if (r) {
		write_tags(s, r);
		if (r->parent == r->id && r->p && n_regs > 1) { // supplementary alignments may exist
			int n_sa = 0;
			for (int i = 0; i < n_regs; ++i)
				if (i != reg_idx && regs[i].parent == regs[i].id && regs[i].p) ++n_sa;
			if (n_sa > 0) {
				s += "\tSA:Z:";
				for (int i = 0; i < n_regs; ++i) {
					const wm_reg1_t *q = &regs[i];
					int l_M, l_I = 0, l_D = 0, clip5, clip3;
					if (r == q || q->parent != q->id || q->p == 0) continue;
					if (q->qe - q->qs < q->re - q->rs) l_M = q->qe - q->qs, l_D = (q->re - q->rs) - l_M;
					else l_M = q->re - q->rs, l_I = (q->qe - q->qs) - l_M;
					clip5 = q->rev ? l_seq - q->qe : q->qs;
					clip3 = q->rev ? q->qs : l_seq - q->qe;
					s += mi->name[q->rid]; s.push_back(','); put_int(s, q->rs + 1); s.push_back(','); s.push_back("+-"[q->rev]); s.push_back(',');
					if (clip5) { put_int(s, clip5); s.push_back('S'); }
					if (l_M) { put_int(s, l_M); s.push_back('M'); }
					if (l_I) { put_int(s, l_I); s.push_back('I'); }
					if (l_D) { put_int(s, l_D); s.push_back('D'); }
					if (clip3) { put_int(s, clip3); s.push_back('S'); }
					s.push_back(','); put_int(s, (int)q->mapq); s.push_back(','); put_int(s, q->blen - q->mlen + q->p->n_ambi); s.push_back(';');
				}
			}
		}
		if (r->p && (opt_flag & (WM_F_OUT_CS | WM_F_OUT_MD))) write_cs_or_MD(s, mi, t->seq.data(), r, !(opt_flag & WM_F_OUT_CS_LONG), (opt_flag & WM_F_OUT_MD) != 0, 1);
		if (cigar_in_tag) write_sam_cigar(s, flag, 1, l_seq, r, opt_flag);
	}
	if (rep_len >= 0) { s += "\trl:i:"; put_int(s, rep_len); }
	if ((opt_flag & WM_F_COPY_COMMENT) && !t->comment.empty()) { s.push_back('\t'); s += t->comment; }
}

int sam_rg_line(const char *s, std::string &line, std::string &id)
{
	line.clear(), id.clear();
	if (strncmp(s, "@RG", 3) != 0) { fprintf(stderr, "[ERROR] the read group line is not started with @RG\n"); return -1; }
	if (strchr(s, '\t')) { fprintf(stderr, "[ERROR] the read group line contained literal <tab> characters -- replace with escaped tabs: \\t\n"); return -1; }
	for (const char *p = s; *p; ++p) { // mm_escape (src/format.c:68-80): \t and \\ resolved, any other escape dropped
		if (*p != '\\') { line.push_back(*p); continue; }
		if (!*++p) break;
		if (*p == 't') line.push_back('\t');
		else if (*p == '\\') line.push_back('\\');
	}
	const size_t at = line.find("\tID:");
	if (at == std::string::npos) { fprintf(stderr, "[ERROR] no ID within the read group line\n"); line.clear(); return -1; }
	const size_t b = at + 4, e = line.find_first_of("\t\n", b);
	id = line.substr(b, e == std::string::npos ? std::string::npos : e - b);
	if (id.size() + 1 > 256) { fprintf(stderr, "[ERROR] @RG:ID is longer than 255 characters\n"); line.clear(), id.clear(); return -1; }
	return 0;
}

// mm_write_sam_hdr (src/format.c:118-139): @SQ lines, the read group line and the @PG line; `cl` is the command line the
// caller wants recorded (the reference prints its own argv), may be null
void write_sam_hdr(std::string &s, const wm_host_idx *mi, const char *version, const char *cl, const char *rg_line)
{
	s.clear();
	for (size_t i = 0; i < mi->name.size(); ++i) {
		s += "@SQ\tSN:"; s += mi->name[i]; s += "\tLN:"; put_int(s, (int)mi->len[i]); s.push_back('\n');
	}
	if (rg_line) { s += rg_line; s.push_back('\n'); }
	s += "@PG\tID:Winnowmap\tPN:Winnowmap";
	if (version) { s += "\tVN:"; s += version; }
	if (cl && cl[0]) { s += "\tCL:"; s += cl; }
	s.push_back('\n');
}

// mm_gen_cs / mm_gen_MD (src/format.c:245-266): the difference string of one hit, without the tag prefix
void gen_cs_or_MD(std::string &s, const wm_host_idx *mi, const wm_reg1_t *r, const char *seq, int is_MD, int no_iden)
{
	s.clear();
	write_cs_or_MD(s, mi, seq, r, no_iden, is_MD, 0);
}

} // namespace wmh
