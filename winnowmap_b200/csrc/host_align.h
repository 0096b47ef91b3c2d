// Alignment driver of one mini-mapping, host side: the control flow of mm_align_skeleton / mm_align1 /
// mm_align1_inv (reference src/align.c:565-920) re-organised as resumable state machines so that every
// extension DP (ksw_extd2) and every local SW (ksw_ll) is shipped to the GPU in batches.  All DP windows
// of a hit are functions of its anchors only, so they are issued speculatively in one batch; the walk
// over the results then follows the reference's order and early exits (Z-drop split, second pass).
#pragma once
#include <stdint.h>
#include <vector>
#include "host_types.h"

namespace wmh {

enum { SEQ_Q0 = 0, SEQ_Q1 = 1, SEQ_REF = 2 };

struct SeqRef { // a slice of the query window (strand 0/1) or of a reference sequence
	int32_t kind, rid;
	int64_t off;
	int32_t len;
	int32_t reversed; // deliver the slice in reverse order (mm_seq_rev)
};

struct DpJob { // one ksw_extd2 call (mm_align_pair, src/align.c:313-339)
	int32_t task;
	SeqRef q, t;
	int32_t w, zdrop, end_bonus, flag;
};

struct DpRes { // ksw_extz_t (src/ksw2.h:23-32)
	int32_t max, zdropped, max_q, max_t, mqe, mqe_t, mte, mte_q, score, reach_end, n_cigar;
	const uint32_t *cigar;
	// optional: the backend already did the score walk of mm_test_zdrop over the CIGAR (jobs flagged EZ_SCAN_ZDROP)
	int32_t has_zd, zd_max, zd_pos[4]; // pos = {t0, t1, q0, q1}
};

struct LlJob { // one ksw_ll_qinit + ksw_ll_i16 (src/ksw2_ll_sse.c:32,80)
	int32_t task;
	SeqRef q, t;
};
struct LlRes { int32_t score, qe, te; };

struct JobSink {
	std::vector<DpJob> dp;
	std::vector<LlJob> ll;
};

// one mm_align1 instance
struct Align1 {
	wm_reg1_t r, r2;
	int state; // 0 = not planned, 1 = waiting for pass 1, 2 = waiting for ll, 3 = waiting for pass 2, 9 = done
	int32_t rid, rev, as1, cnt1, bw;
	int32_t rs, qs, re, qe, rs0, qs0, re0, qe0, rs1, qs1, re1, qe1;
	int32_t rs_init, qs_init;
	int left_job, right_job; // indices into the round's job list, -1 if none
	struct Gap { int32_t i, rs, qs, re, qe, bw1; int job; DpRes res; size_t cig_off; };
	bool captured;          // pass-1 results copied out of the round buffers
	DpRes left_res, right_res;
	size_t left_cig, right_cig;       // offsets into cig_pool
	std::vector<uint32_t> cig_pool;    // one pool for all captured pass-1 CIGARs of this hit
	std::vector<Gap> gaps;
	size_t gap_cur;
	bool left_done, dropped;
	int pending_job;        // job index of the outstanding ll / pass-2 request
	int32_t zd_max_zdrop;   // carried across the ll round
	// spliced alignment: the KSW_EZ_SPLICE_* bits of every DP of this instance (extra_flag, src/align.c:602-606), and the
	// boundary-exon filter of mm_fix_bad_ends_splice (:545-563), planned once per hit and shared by its two strand rounds
	int32_t splice_flag = 0;
	int end_ll[2] = {-1, -1};   // ll job of the first / last anchor (mm_seed_ext_score), -1 if not needed
	int32_t end_as1 = 0, end_cnt1 = 0;
};

struct AlignTask {
	const wm_mapopt_t *opt;
	const wm_host_idx *mi;
	int task_id, qlen;
	std::vector<uint8_t> qcodes; // 2*qlen: strand 0 then strand 1 of the window (src/align.c:871-877), when the caller has no codes
	const uint8_t *q_strand[2];  // 0..4 codes of the window, strand 0 / strand 1
	wm_pair_t *a;
	int n_a;
	std::vector<wm_reg1_t> regs; // in/out
	int8_t mat[25];

	// state
	std::vector<Align1> firsts;  // phase 1: n_round per original hit, all in flight together
	int n_round;                 // 2: spliced alignment with both strand flags (src/align.c:884-900), two mm_align1 per hit
	int phase;                   // 0 = init, 4 = splice end filter planned, 1 = phase 1 running, 2 = sequential follow-ups, 3 = finished
	// phase 2 (exact loop order of mm_align_skeleton for split children and inversions)
	std::vector<wm_reg1_t> out;
	size_t cur;                  // index into `out` of the element being processed
	int sub;                     // 0 = need align1 (or reuse phase-1 result), 5 = splice end filter wait, 1 = align1 running, 2 = inv ll wait, 3 = inv dp wait
	Align1 child[2];
	std::vector<char> from_first; // out[i] was aligned in phase 1
	int inv_job; int32_t inv_ql, inv_tl, inv_qoff, inv_toff;

	// q0 / q1: codes of the window's two strands if the caller already has them (slices of the read's code arrays), else null
	void init(const wm_mapopt_t *opt_, const wm_host_idx *mi_, int task_id_, int qlen_, const char *qstr, std::vector<wm_reg1_t> &regs_in, wm_pair_t *a_,
	          const uint8_t *q0 = 0, const uint8_t *q1 = 0);
	// Advance as far as possible. `dp`/`ll` are the results of the jobs this task pushed in the previous call
	// (indexed by the job numbers it was given: base_dp/base_ll + local index).  New jobs are appended to `sink`.
	// Returns true when the task is complete (regs holds the result of mm_align_skeleton).
	bool advance(const DpRes *dp, const LlRes *ll, JobSink &sink);

	const uint8_t *qseq(int strand) const { return q_strand[strand]; }
private:
	void start_rounds(const wm_reg1_t &r, Align1 *A, JobSink &sink);
	bool ends_pending(const Align1 &A) const { return A.end_ll[0] >= 0 || A.end_ll[1] >= 0; }
	void plan_rounds(Align1 *A, const LlRes *ll, JobSink &sink);
	void pick_round(Align1 *A, wm_reg1_t *r, wm_reg1_t *r2) const;
	void plan1(Align1 &A, JobSink &sink);
	bool walk1(Align1 &A, const DpRes *dp, const LlRes *ll, JobSink &sink);
	bool step_phase2(const DpRes *dp, const LlRes *ll, JobSink &sink);
};

void gen_simple_mat(int8_t *mat, int8_t a, int8_t b, int8_t sc_ambi);
// 0..4 codes of a sequence and of its reverse complement (src/align.c:871-877)
void encode_strands(const char *seq, int len, uint8_t *fwd, uint8_t *rev);
void update_extra(wm_reg1_t *r, const uint8_t *qseq, const uint8_t *tseq, const int8_t *mat, int8_t q, int8_t e, int is_eqx);
void append_cigar(wm_reg1_t *r, uint32_t n_cigar, const uint32_t *cigar);

} // namespace wmh
