#pragma once
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <vector>
#include "host_types.h"
#include "host_backend.h"

namespace wmh {

void idxopt_init(wm_idxopt_t *o);
void mapopt_init(wm_mapopt_t *o);
int set_opt(const char *preset, wm_idxopt_t *io, wm_mapopt_t *mo);
int check_opt(const wm_idxopt_t *io, const wm_mapopt_t *mo);
void mapopt_max_intron_len(wm_mapopt_t *opt, int max_intron_len);

class SeqReader { // FASTA/FASTQ, plain or gzip (kseq semantics, src/kseq.h)
public:
	SeqReader(); ~SeqReader();
	bool open(const char *fn);
	bool next(wm_read &r);
	bool next_line(std::string &s); // one line without its \n (and a \r before it, as kseq's KS_SEP_LINE); false at the end
private:
	struct Impl; Impl *p;
};

int read_kmer_list(const char *fn, int k, std::vector<uint64_t> &canon_kmers);
// mm_idx_bed_read(mi, fn, 1) (src/index.c:690-778): the junction intervals of a BED file (plain or gzip, "-" for stdin) for
// the sequences of mi, replacing any it had; 0, or -1 when the file cannot be opened (mi is then left as it was)
int read_bed_junc(wm_host_idx *mi, const char *fn);
// the same from the reference's mm_idx_t::I (one record per sequence of mi, each sorted by st)
void set_junc(wm_host_idx *mi, const wm_idx_intv_t *I);

// PAF line of one hit / of an unmapped read (mm_write_paf3, src/format.c:308-334)
void write_paf(std::string &s, const wm_host_idx *mi, const wm_read *t, const wm_reg1_t *r, int64_t opt_flag, int rep_len);
// SAM record of hit reg_idx of a single-segment read (reg_idx < 0: the unmapped record), mm_write_sam3 (src/format.c:391-548)
void write_sam(std::string &s, const wm_host_idx *mi, const wm_read *t, int reg_idx, int n_regs, const wm_reg1_t *regs, int64_t opt_flag, int rep_len,
               const char *rg_id);
// cs / MD difference string of one hit without the tag prefix (mm_gen_cs / mm_gen_MD, src/format.c:245-266); seq = the read, ASCII
void gen_cs_or_MD(std::string &s, const wm_host_idx *mi, const wm_reg1_t *r, const char *seq, int is_MD, int no_iden);
// @SQ, @RG and @PG header lines (mm_write_sam_hdr, src/format.c:118-139); rg_line is what sam_rg_line made of -R, or null
void write_sam_hdr(std::string &s, const wm_host_idx *mi, const char *version, const char *cl, const char *rg_line = 0);
// The read group of -R (sam_write_rg_line, src/format.c:82-116): the line with its \t and \\ escapes resolved, and its ID.
// -1, with a message, when the line does not start with @RG, holds a literal tab, has no ID or an ID over 255 characters.
int sam_rg_line(const char *s, std::string &line, std::string &id);

} // namespace wmh
