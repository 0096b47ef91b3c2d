// Host-side types of the mapping path.  Layouts that cross the C ABI mirror the reference's
// public structs field for field (src/minimap.h) so that a reference-side caller can pass its own
// objects by pointer: wm_mapopt_t <-> mm_mapopt_t (:112-176), wm_reg1_t <-> mm_reg1_t (:88-103),
// wm_extra_t <-> mm_extra_t (:80-86), wm_idxopt_t <-> mm_idxopt_t (:106-110).
#pragma once
#include <stdint.h>
#include <string>
#include <vector>

// mapping flags, same values as src/minimap.h:9-40
#define WM_F_NO_DIAG       0x001
#define WM_F_NO_DUAL       0x002
#define WM_F_CIGAR         0x004
#define WM_F_OUT_SAM       0x008
#define WM_F_NO_QUAL       0x010
#define WM_F_OUT_CG        0x020
#define WM_F_OUT_CS        0x040
#define WM_F_SPLICE        0x080
#define WM_F_SPLICE_FOR    0x100
#define WM_F_SPLICE_REV    0x200
#define WM_F_NO_LJOIN      0x400
#define WM_F_OUT_CS_LONG   0x800
#define WM_F_SR            0x1000
#define WM_F_FRAG_MODE     0x2000
#define WM_F_NO_PRINT_2ND  0x4000
#define WM_F_2_IO_THREADS  0x8000
#define WM_F_LONG_CIGAR    0x10000
#define WM_F_INDEPEND_SEG  0x20000
#define WM_F_SPLICE_FLANK  0x40000
#define WM_F_SOFTCLIP      0x80000
#define WM_F_FOR_ONLY      0x100000
#define WM_F_REV_ONLY      0x200000
#define WM_F_HEAP_SORT     0x400000
#define WM_F_ALL_CHAINS    0x800000
#define WM_F_OUT_MD        0x1000000
#define WM_F_COPY_COMMENT  0x2000000
#define WM_F_EQX           0x4000000
#define WM_F_PAF_NO_HIT    0x8000000
#define WM_F_NO_END_FLT    0x10000000
#define WM_F_HARD_MLEVEL   0x20000000
#define WM_F_SAM_HIT_ONLY  0x40000000

#define WM_I_HPC 0x1
#define WM_I_JUNC WM_IDX_JUNC // not an mm_idx_t flag: the index carries junction intervals (mm_idx_t::I, --junc-bed)

// anchor flag bits in mm128_t.y (src/mmpriv.h:17-23)
#define WM_SEED_LONG_JOIN (1ULL << 40)
#define WM_SEED_IGNORE    (1ULL << 41)
#define WM_SEED_TANDEM    (1ULL << 42)
#define WM_SEED_SELF      (1ULL << 43)

#define WM_PARENT_UNSET   (-1)
#define WM_PARENT_TMP_PRI (-2)

#include "../../include/winnowmap_b200.h"
typedef wm128_t wm_pair_t; // mm128_t



// Host copy of what the path needs from the index (mm_idx_t / mm_idx_seq_t, src/minimap.h:59-77)
struct wm_host_idx {
	int k, w;
	int flag = 0;            // mm_idx_t::flag: WM_I_HPC when the index holds homopolymer-compressed minimizers
	bool junc = false;       // uploaded with WM_IDX_JUNC: the caller's index has junction intervals (map_batch refuses spliced alignment until they are set)
	// junction intervals (mm_idx_t::I after mm_idx_bed_read, src/index.c:769-778): those of sequence rid at
	// junc_iv[junc_off[rid] .. junc_off[rid + 1]), sorted by st; junc_off is empty until a BED was read or intervals were set
	std::vector<wm_idx_intv1_t> junc_iv; std::vector<int64_t> junc_off;
	bool has_junc() const { return !junc_off.empty(); }
	std::vector<std::string> name;
	std::vector<uint32_t> len;
	std::vector<uint64_t> offset;
	std::vector<uint32_t> S; // 4-bit packed, mm_seq4_set layout (src/mmpriv.h:29-30)
	// strcmp order of the names (set_name_order): the name tests of -D / --dual=no become integer comparisons.
	// name_rank[rid] = number of names strictly less than name[rid]; name_sorted: the rids in that order
	std::vector<uint32_t> name_rank, name_sorted;
	inline int base(uint64_t i) const { return S[i >> 3] >> ((i & 7) << 2) & 0xf; }
	// mm_idx_getseq (src/index.c:161-171)
	int getseq(uint32_t rid, uint32_t st, uint32_t en, uint8_t *seq) const {
		if (rid >= len.size() || st >= len[rid]) return -1;
		if (en > len[rid]) en = len[rid];
		uint64_t st1 = offset[rid] + st, en1 = offset[rid] + en, i = st1;
		for (; i < en1 && (i & 7); ++i) seq[i - st1] = (uint8_t)base(i);
		for (; i + 8 <= en1; i += 8) { // one 32-bit word = eight bases
			uint32_t w = S[i >> 3];
			uint8_t *o = seq + (i - st1);
			o[0] = w & 0xf, o[1] = w >> 4 & 0xf, o[2] = w >> 8 & 0xf, o[3] = w >> 12 & 0xf;
			o[4] = w >> 16 & 0xf, o[5] = w >> 20 & 0xf, o[6] = w >> 24 & 0xf, o[7] = w >> 28;
		}
		for (; i < en1; ++i) seq[i - st1] = (uint8_t)base(i);
		return (int)(en - st);
	}
};

// one query of a batch (mm_bseq1_t, src/bseq.h:14-17)
struct wm_read {
	std::string name, comment;
	std::string seq;   // ASCII
	std::string qual;
	int64_t dev_off = -1; // >= 0: the bases are also resident in the device pool given to Backend::set_resident_pool, at this offset
	bool has_name = true; // false: mm_map with qname == 0 (the name tests of -D / --dual=no are off; `name` is "")
};
