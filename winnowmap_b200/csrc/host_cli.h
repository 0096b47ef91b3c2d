// The winnowmap command line (reference src/main.c:45-430): option parsing with the reference's semantics and the run over
// an index of one or more parts (host_driver.h).  Plain host C++: the library runs it over GPU-built parts (wm_cli_main in
// capi_map.cu), the CPU test harness over oracle-backed parts.
#pragma once
#include <stdint.h>
#include <functional>
#include <memory>
#include <string>
#include <vector>
#include "host_driver.h"
#include "host_types.h"

namespace wmh {

#define WM_I_NO_SEQ 0x2 // MM_I_NO_SEQ (src/minimap.h:20): set by main() when nothing is aligned

// What main() holds once its two option passes are done (src/main.c:145-275)
struct CliArgs {
	wm_idxopt_t ipt;
	wm_mapopt_t opt;
	int n_threads;
	bool threads_set;                 // -t was given
	std::vector<std::string> files;   // the positional arguments: the reference first, then the query files
	std::string out_fn, rg, kmer_fn, split_prefix;
	bool has_out, has_rg, has_kmer, has_split;
	bool help;                        // -h
};

// Parses argv as the reference's main() does, up to the point where it opens the index (src/main.c:327).  n_cpu is the
// processor count the default thread count derives from (<= 0: the affinity mask's).  Returns -1 when the run should go
// on, else the exit status main() returns at that point (0 for -V and -h, 1 on every error).  Options the mapper does not
// implement are refused here, naming the option, with status 1.
int cli_parse(int argc, char **argv, CliArgs &a, int n_cpu = 0);

// mm_mapopt_update without the index-dependent -f step (src/options.c:71-81): the splice flag that -u implies and the
// --min-occ-floor clamp.  -f is resolved per index part by IndexParts::part_opt.
void cli_update_opt(wm_mapopt_t *opt);

// Builds the index of a parsed command line (its reference and -W file), cut into parts under -I; null after an error
// (already reported).
typedef std::function<std::unique_ptr<IndexParts>(const CliArgs &a)> IndexBuilder;

// main(): parse, refuse, build the index through `build` and map every query file part by part (or merged under
// --split-prefix) to stdout or -o.  Returns the exit status.
int cli_main(int argc, char **argv, const IndexBuilder &build);

} // namespace wmh
