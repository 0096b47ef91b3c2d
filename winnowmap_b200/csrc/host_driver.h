// The file-level mapping driver (mm_map_file / mm_split_merge, reference src/map.c:1107-1321 and src/main.c:384-424): plain
// host C++ over an index of one or more parts that the caller provides (IndexParts).  The library runs it over its GPU
// context (capi_map.cu), the CPU test harness over oracle backends.
#pragma once
#include <stdint.h>
#include <string>
#include <vector>
#include "host_types.h"

namespace wmh {

// Where mm_idx_gen ends an index part (src/index.c:289-297 and :660-671, src/bseq.c:80-119): a part is read in mini-batches
// of min(mini_batch_size, batch_size) bases, each mini-batch whole sequences until it holds at least that many bases, and
// no further mini-batch is started once the part holds more than batch_size bases.
struct PartCutter {
	uint64_t batch, mb, part_sum = 0, mb_sum = 0;
	bool open = false; // a mini-batch is being filled
	int part = -1;
	PartCutter(uint64_t batch_size, int mini_batch_size) : batch(batch_size), mb((uint64_t)mini_batch_size < batch_size ? (uint64_t)mini_batch_size : batch_size) {}
	int next(uint64_t len) // the part of the next sequence
	{
		if (!open) {
			if (part < 0 || part_sum > batch) ++part, part_sum = 0;
			open = true, mb_sum = 0;
		}
		mb_sum += len;
		if (mb_sum >= mb) part_sum += mb_sum, open = false;
		return part;
	}
};

// What the driver needs of an index: its parts, the options each part maps with and the mapping itself.
class IndexParts {
public:
	virtual ~IndexParts() {}
	virtual int n_parts() const = 0;
	virtual const wm_host_idx *part(int p) const = 0; // the sequence table of part p (rid restarts at 0 in every part)
	virtual const wm_host_idx *all() const = 0;       // the sequence table of all parts in part order (part(0) for one part)
	// the options part p maps with: under -f, mid_occ of that part (mm_mapopt_update, src/main.c:403); false when refused
	virtual bool part_opt(int p, const wm_mapopt_t *opt, wm_mapopt_t *o) = 0;
	// regs (each p malloc()ed) and rep_len of every read against part p
	virtual void map(int p, const wm_mapopt_t *opt, const std::vector<const wm_read*> &reads, std::vector<std::vector<wm_reg1_t>> &regs,
	                 std::vector<int> &rep_len, int n_threads) = 0;
};

// The output step of one read (src/map.c:1189-1206): its hits as PAF or SAM lines (opt_flag says which), appended to dst.
// prefix (if not null) starts every line.
// rg_id is the @RG ID the SAM records carry ("" or null: none).
void format_read(std::string &dst, const wm_host_idx *mi, int64_t opt_flag, const wm_read *t, int n_reg, const wm_reg1_t *regs, int rep_len,
                 const char *prefix = 0, const char *rg_id = 0);

// --split-prefix: every read mapped against every part, then merge_hits (src/map.c:1050-1105).  false when a part's options
// are refused.
bool map_merged(IndexParts &ix, const wm_mapopt_t *opt, const std::vector<const wm_read*> &reads, std::vector<std::vector<wm_reg1_t>> &regs,
                int n_threads);

// mm_map_file over the parts of ix, written to out_fn ("-" or null: stdout) with the SAM header when opt asks for SAM.  With
// world > 1 only the reads whose position in their length-sorted mini-batch is rank mod world are mapped and written, and
// tag_order prefixes every line with "<batch>\t<position>\t".  max_batch_bases bounds the reads mapped in one call.
// 0, or -1 after an error.
int map_file(IndexParts &ix, const wm_mapopt_t *opt, const char *reads_fn, const char *out_fn, const char *sam_cl, int n_threads, int rank, int world,
             int tag_order, int64_t max_batch_bases);

// The loop of the reference's main() over the parts and the query files (src/main.c:384-424): the SAM header once, then part
// by part every file in argument order (or, with split_prefix, every file merged over all parts).  rg is the -R line
// (null: none), checked and unescaped as sam_write_rg_line does; under SAM its ID tags every record.  A query file that
// cannot be opened is reported and skipped, as mm_map_file skips it.  The rest as map_file, which is this call with one file
// that is checked before the output is created.
int map_files(IndexParts &ix, const wm_mapopt_t *opt, const std::vector<const char*> &reads_fns, const char *out_fn, const char *sam_cl, const char *rg,
              int n_threads, int rank, int world, int tag_order, int64_t max_batch_bases);

} // namespace wmh
