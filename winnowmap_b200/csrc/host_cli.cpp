// The winnowmap command line (host_cli.h).  Options are read with glibc getopt_long, which takes the same syntax as the
// reference's parser: permuted positional arguments, bundled short options (-ax map-ont), attached values (-t8) and
// --opt=value.  main()'s order is kept: a first pass applies -x (and reports unknown options and missing values), a
// second applies every other option in argument order, then the checks.
#include <errno.h>
#include <getopt.h>
#include <sched.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <unistd.h>
#include <algorithm>
#include "host_cli.h"
#include "host_io.h"

namespace wmh {

static const char *kVersion = "2.03";
// opt_str of src/main.c:128; the leading ':' makes a missing value return ':' instead of '?'
static const char *kOptStr = ":2aSDw:W:k:K:t:r:f:Vv:g:G:I:XT:s:x:Hcp:M:n:z:A:B:O:E:m:N:Qu:R:hF:LC:yYPo:";
enum { O_CAP_SW_MEM = 337, O_MAX_QLEN = 338 };
// long_options of src/main.c:45-100, with the reference's option codes
static const struct option kLong[] = {
	{ "bucket-bits", required_argument, 0, 300 }, { "mb-size", required_argument, 0, 'K' }, { "seed", required_argument, 0, 302 },
	{ "no-kalloc", no_argument, 0, 303 }, { "print-qname", no_argument, 0, 304 }, { "dbg-polish", no_argument, 0, 305 },
	{ "no-self", no_argument, 0, 'D' }, { "print-seeds", no_argument, 0, 306 }, { "max-chain-skip", required_argument, 0, 307 },
	{ "min-dp-len", required_argument, 0, 308 }, { "print-aln-seq", no_argument, 0, 309 }, { "splice", no_argument, 0, 310 },
	{ "cost-non-gt-ag", required_argument, 0, 'C' }, { "no-long-join", no_argument, 0, 312 }, { "sr", no_argument, 0, 313 },
	{ "frag", required_argument, 0, 314 }, { "secondary", required_argument, 0, 315 }, { "cs", optional_argument, 0, 316 },
	{ "end-bonus", required_argument, 0, 317 }, { "no-pairing", no_argument, 0, 318 }, { "splice-flank", required_argument, 0, 319 },
	{ "idx-no-seq", no_argument, 0, 320 }, { "end-seed-pen", required_argument, 0, 321 }, { "for-only", no_argument, 0, 322 },
	{ "rev-only", no_argument, 0, 323 }, { "heap-sort", required_argument, 0, 324 }, { "all-chain", no_argument, 0, 'P' },
	{ "dual", required_argument, 0, 326 }, { "max-clip-ratio", required_argument, 0, 327 }, { "min-occ-floor", required_argument, 0, 328 },
	{ "MD", no_argument, 0, 329 }, { "lj-min-ratio", required_argument, 0, 330 }, { "score-N", required_argument, 0, 331 },
	{ "eqx", no_argument, 0, 332 }, { "paf-no-hit", no_argument, 0, 333 }, { "split-prefix", required_argument, 0, 334 },
	{ "no-end-flt", no_argument, 0, 335 }, { "hard-mask-level", no_argument, 0, 336 }, { "cap-sw-mem", required_argument, 0, O_CAP_SW_MEM },
	{ "max-qlen", required_argument, 0, O_MAX_QLEN }, { "max-chain-iter", required_argument, 0, 339 }, { "junc-bed", required_argument, 0, 340 },
	{ "junc-bonus", required_argument, 0, 341 }, { "sam-hit-only", no_argument, 0, 342 }, { "sv-off", no_argument, 0, 343 },
	{ "help", no_argument, 0, 'h' }, { "max-intron-len", required_argument, 0, 'G' }, { "version", no_argument, 0, 'V' },
	{ "min-count", required_argument, 0, 'n' }, { "min-chain-score", required_argument, 0, 'm' }, { "mask-level", required_argument, 0, 'M' },
	{ "min-dp-score", required_argument, 0, 's' }, { "sam", no_argument, 0, 'a' }, { 0, 0, 0, 0 }
};

// mm_parse_num (src/main.c:102-111): a number with an optional K/M/G suffix, rounded
static int64_t parse_num(const char *str)
{
	char *p;
	double x = strtod(str, &p);
	if (*p == 'G' || *p == 'g') x *= 1e9;
	else if (*p == 'M' || *p == 'm') x *= 1e6;
	else if (*p == 'K' || *p == 'k') x *= 1e3;
	return (int64_t)(x + .499);
}

// yes_or_no (src/main.c:113-125): yes_to_set says whether "yes" sets the flag or clears it
static void yes_or_no(wm_mapopt_t *opt, int64_t flag, int long_idx, const char *arg, bool yes_to_set)
{
	const bool yes = strcmp(arg, "yes") == 0 || strcmp(arg, "y") == 0, no = strcmp(arg, "no") == 0 || strcmp(arg, "n") == 0;
	if (!yes && !no) { fprintf(stderr, "[WARNING] option '--%s' only accepts 'yes' or 'no'.\n", kLong[long_idx].name); return; }
	if (yes == yes_to_set) opt->flag |= flag;
	else opt->flag &= ~flag;
}

static int cpu_count()
{
	cpu_set_t cs;
	if (sched_getaffinity(0, sizeof(cpu_set_t), &cs) != 0) return 1;
	return CPU_COUNT(&cs);
}

static void usage(FILE *fp, const CliArgs &a)
{
	fprintf(fp, "Usage: winnowmap-b200 [options] <target.fa> <query.fa> [...]\n");
	fprintf(fp, "Maps long reads on an NVIDIA GPU with the options and output of Winnowmap %s.\n", kVersion);
	fprintf(fp, "Indexing:\n");
	fprintf(fp, "  -H          homopolymer-compressed k-mers\n");
	fprintf(fp, "  -k INT      k-mer size, at most 28 [%d]\n", a.ipt.k);
	fprintf(fp, "  -w INT      minimizer window size [%d]\n", a.ipt.w);
	fprintf(fp, "  -I NUM      split the index every ~NUM input bases [4G]\n");
	fprintf(fp, "  -W FILE     list of high-frequency k-mers to down-weight\n");
	fprintf(fp, "Mapping:\n");
	fprintf(fp, "  -f FLOAT    filter out the top FLOAT (< 1) fraction of repetitive minimizers\n");
	fprintf(fp, "  -g NUM      stop chain elongation after NUM bp without minimizers [%d]\n", a.opt.max_gap);
	fprintf(fp, "  -G NUM      max intron length (with -x splice) [200k]\n");
	fprintf(fp, "  -r NUM      bandwidth of chaining and alignment [%d]\n", a.opt.bw);
	fprintf(fp, "  -n INT      minimal number of minimizers on a chain [%d]\n", a.opt.min_cnt);
	fprintf(fp, "  -m INT      minimal chaining score [%d]\n", a.opt.min_chain_score);
	fprintf(fp, "  -X          skip self and dual mappings (all-vs-all)\n");
	fprintf(fp, "  -p FLOAT    min secondary-to-primary score ratio [%g]\n", a.opt.pri_ratio);
	fprintf(fp, "  --sv-off    turn off the SV-aware mode\n");
	fprintf(fp, "  --max-qlen NUM    skip reads (and stage-1 windows) longer than NUM\n");
	fprintf(fp, "  --cap-sw-mem NUM  skip alignment DPs with more than NUM cells\n");
	fprintf(fp, "Alignment:\n");
	fprintf(fp, "  -A INT -B INT     match score and mismatch penalty [%d, %d]\n", a.opt.a, a.opt.b);
	fprintf(fp, "  -O INT[,INT]      gap open penalties [%d,%d]\n", a.opt.q, a.opt.q2);
	fprintf(fp, "  -E INT[,INT]      gap extension penalties [%d,%d]\n", a.opt.e, a.opt.e2);
	fprintf(fp, "  -z INT[,INT]      Z-drop and inversion Z-drop scores [%d,%d]\n", a.opt.zdrop, a.opt.zdrop_inv);
	fprintf(fp, "  -s INT            minimal peak DP alignment score [%d]\n", a.opt.min_dp_max);
	fprintf(fp, "Input/output:\n");
	fprintf(fp, "  -a          SAM output (PAF by default)\n");
	fprintf(fp, "  -o FILE     write the output to FILE [stdout]\n");
	fprintf(fp, "  -c          CIGAR in PAF\n");
	fprintf(fp, "  --cs[=STR]  cs tag, 'short' or 'long'\n");
	fprintf(fp, "  --MD        MD tag\n");
	fprintf(fp, "  --eqx       =/X CIGAR operators\n");
	fprintf(fp, "  -R STR      SAM read group line, like '@RG\\tID:foo\\tSM:bar'\n");
	fprintf(fp, "  -t INT      host threads\n");
	fprintf(fp, "  -K NUM      mini-batch size [1000M]\n");
	fprintf(fp, "  --split-prefix STR  merge the hits of a multi-part index per read\n");
	fprintf(fp, "  --version   print the version of Winnowmap this build follows\n");
	fprintf(fp, "Presets (-x, applied before the other options):\n");
	fprintf(fp, "  map-ont, map-pb, map-pb-clr, asm5, asm10, asm20, splice, splice:hq, cdna\n");
}

void cli_update_opt(wm_mapopt_t *opt)
{
	if (opt->flag & (WM_F_SPLICE_FOR | WM_F_SPLICE_REV)) opt->flag |= WM_F_SPLICE;
	if (!(opt->mid_occ_frac >= 0 && opt->mid_occ_frac < 1) && opt->mid_occ < opt->min_mid_occ) opt->mid_occ = opt->min_mid_occ;
}

int cli_parse(int argc, char **argv, CliArgs &a, int n_cpu)
{
	a.n_threads = std::max(3, n_cpu > 0 ? n_cpu : cpu_count());
	a.threads_set = a.has_out = a.has_rg = a.has_kmer = a.has_split = a.help = false;
	a.files.clear();
	set_opt(0, &a.ipt, &a.opt);
	int c, long_idx, old_best_n = -1;
	opterr = 0;
	// pass 1: -x before everything else, and the parse errors (src/main.c:145-158)
	optind = 0;
	while ((c = getopt_long(argc, argv, kOptStr, kLong, &long_idx)) >= 0) {
		if (c == 'x') {
			if (set_opt(optarg, &a.ipt, &a.opt) < 0) { fprintf(stderr, "[ERROR] unknown preset '%s'\n", optarg); return 1; }
		} else if (c == ':') {
			fprintf(stderr, "[ERROR] missing option argument\n");
			return 1;
		} else if (c == '?') {
			fprintf(stderr, "[ERROR] unknown option in \"%s\"\n", argv[optind - 1]);
			return 1;
		}
	}
	// pass 2 (src/main.c:161-274)
	optind = 0;
	wm_mapopt_t &opt = a.opt;
	wm_idxopt_t &ipt = a.ipt;
	while ((c = getopt_long(argc, argv, kOptStr, kLong, &long_idx)) >= 0) {
		char *s;
		switch (c) {
		case 'w': ipt.w = (short)atoi(optarg); break;
		case 'W': a.kmer_fn = optarg, a.has_kmer = true; break;
		case 'k': ipt.k = (short)atoi(optarg); break;
		case 'H': ipt.flag |= WM_I_HPC; break;
		case 'r': opt.bw = (int)parse_num(optarg); break;
		case 't': a.n_threads = atoi(optarg), a.threads_set = true; break;
		case 'v': break; // verbosity of the reference's progress messages
		case 'g': opt.max_gap = (int)parse_num(optarg); break;
		case 'G': mapopt_max_intron_len(&opt, (int)parse_num(optarg)); break;
		case 'F': opt.max_frag_len = (int)parse_num(optarg); break;
		case 'N': old_best_n = opt.best_n, opt.best_n = atoi(optarg); break;
		case 'p': opt.pri_ratio = (float)atof(optarg); break;
		case 'M': opt.mask_level = (float)atof(optarg); break;
		case 'c': opt.flag |= WM_F_OUT_CG | WM_F_CIGAR; break;
		case 'D': opt.flag |= WM_F_NO_DIAG; break;
		case 'P': opt.flag |= WM_F_ALL_CHAINS; break;
		case 'X': opt.flag |= WM_F_ALL_CHAINS | WM_F_NO_DIAG | WM_F_NO_DUAL | WM_F_NO_LJOIN; break;
		case 'a': opt.flag |= WM_F_OUT_SAM | WM_F_CIGAR; break;
		case 'Q': opt.flag |= WM_F_NO_QUAL; break;
		case 'Y': opt.flag |= WM_F_SOFTCLIP; break;
		case 'L': opt.flag |= WM_F_LONG_CIGAR; break;
		case 'y': opt.flag |= WM_F_COPY_COMMENT; break;
		case 'T': opt.sdust_thres = atoi(optarg); break;
		case 'n': opt.min_cnt = atoi(optarg); break;
		case 'm': opt.min_chain_score = atoi(optarg); break;
		case 'A': opt.a = atoi(optarg); break;
		case 'B': opt.b = atoi(optarg); break;
		case 's': opt.min_dp_max = atoi(optarg); break;
		case 'C': opt.noncan = atoi(optarg); break;
		case 'I': ipt.batch_size = (uint64_t)parse_num(optarg); break;
		case 'K': opt.mini_batch_size = (int)parse_num(optarg); break;
		case 'R': a.rg = optarg, a.has_rg = true; break;
		case 'h': a.help = true; break;
		case '2': opt.flag |= WM_F_2_IO_THREADS; break;
		case 'o': a.out_fn = optarg, a.has_out = true; break;
		case 300: ipt.bucket_bits = (short)atoi(optarg); break;
		case 302: opt.seed = atoi(optarg); break;
		case 303: case 304: case 305: break; // allocator and debug-print switches of the reference
		case 306: case 309: a.n_threads = 1; break; // debug prints that also run the reference single-threaded
		case 307: opt.max_chain_skip = atoi(optarg); break;
		case 339: opt.max_chain_iter = atoi(optarg); break;
		case 308: opt.min_ksw_len = atoi(optarg); break;
		case 310: opt.flag |= WM_F_SPLICE; break;
		case 312: opt.flag |= WM_F_NO_LJOIN; break;
		case 313: opt.flag |= WM_F_SR; break;
		case 317: opt.end_bonus = atoi(optarg); break;
		case 318: opt.flag |= WM_F_INDEPEND_SEG; break;
		case 320: ipt.flag |= WM_I_NO_SEQ; break;
		case 321: opt.anchor_ext_shift = atoi(optarg); break;
		case 322: opt.flag |= WM_F_FOR_ONLY; break;
		case 323: opt.flag |= WM_F_REV_ONLY; break;
		case 327: opt.max_clip_ratio = (float)atof(optarg); break;
		case 328: opt.min_mid_occ = atoi(optarg); break;
		case 329: opt.flag |= WM_F_OUT_MD; break;
		case 330: opt.min_join_flank_ratio = (float)atof(optarg); break;
		case 331: opt.sc_ambi = atoi(optarg); break;
		case 332: opt.flag |= WM_F_EQX; break;
		case 333: opt.flag |= WM_F_PAF_NO_HIT; break;
		case 334: a.split_prefix = optarg, a.has_split = true; break;
		case 335: opt.flag |= WM_F_NO_END_FLT; break;
		case 336: opt.flag |= WM_F_HARD_MLEVEL; break;
		case O_CAP_SW_MEM: opt.max_sw_mat = parse_num(optarg); break;
		case O_MAX_QLEN: opt.max_qlen = (int)parse_num(optarg); break;
		case 340: break; // --junc-bed: read only for spliced base alignment
		case 341: break; // --junc-bonus: listed, but main() never applies it
		case 342: opt.flag |= WM_F_SAM_HIT_ONLY; break;
		case 343:
			opt.SVaware = false;
			if (!a.threads_set) a.n_threads = std::max(3, n_cpu > 0 ? n_cpu : cpu_count());
			break;
		case 314: yes_or_no(&opt, WM_F_FRAG_MODE, long_idx, optarg, true); break;
		case 315: yes_or_no(&opt, WM_F_NO_PRINT_2ND, long_idx, optarg, false); break;
		case 316:
			opt.flag |= WM_F_OUT_CS | WM_F_CIGAR;
			if (optarg == 0 || strcmp(optarg, "short") == 0) opt.flag &= ~(int64_t)WM_F_OUT_CS_LONG;
			else if (strcmp(optarg, "long") == 0) opt.flag |= WM_F_OUT_CS_LONG;
			else if (strcmp(optarg, "none") == 0) opt.flag &= ~(int64_t)WM_F_OUT_CS;
			else fprintf(stderr, "[WARNING] --cs only takes 'short' or 'long'. Invalid values are assumed to be 'short'.\n");
			break;
		case 319: yes_or_no(&opt, WM_F_SPLICE_FLANK, long_idx, optarg, true); break;
		case 324: yes_or_no(&opt, WM_F_HEAP_SORT, long_idx, optarg, true); break;
		case 326: yes_or_no(&opt, WM_F_NO_DUAL, long_idx, optarg, false); break;
		case 'S':
			opt.flag |= WM_F_OUT_CS | WM_F_CIGAR | WM_F_OUT_CS_LONG;
			fprintf(stderr, "[WARNING] option -S is deprecated. Please use --cs=long instead.\n");
			break;
		case 'V': puts(kVersion); return 0;
		case 'f': {
			const double x = strtod(optarg, &s);
			if (x >= 0.0 && x < 1.0) opt.mid_occ_frac = (float)x;
			break;
		}
		case 'u':
			if (*optarg == 'b') opt.flag |= WM_F_SPLICE_FOR | WM_F_SPLICE_REV;
			else if (*optarg == 'f') opt.flag |= WM_F_SPLICE_FOR, opt.flag &= ~(int64_t)WM_F_SPLICE_REV;
			else if (*optarg == 'r') opt.flag |= WM_F_SPLICE_REV, opt.flag &= ~(int64_t)WM_F_SPLICE_FOR;
			else if (*optarg == 'n') opt.flag &= ~(int64_t)(WM_F_SPLICE_FOR | WM_F_SPLICE_REV);
			else { fprintf(stderr, "[ERROR] unrecognized cDNA direction\n"); return 1; }
			break;
		case 'z':
			opt.zdrop = opt.zdrop_inv = (int)strtol(optarg, &s, 10);
			if (*s == ',') opt.zdrop_inv = (int)strtol(s + 1, &s, 10);
			break;
		case 'O':
			opt.q = opt.q2 = (int)strtol(optarg, &s, 10);
			if (*s == ',') opt.q2 = (int)strtol(s + 1, &s, 10);
			break;
		case 'E':
			opt.e = opt.e2 = (int)strtol(optarg, &s, 10);
			if (*s == ',') opt.e2 = (int)strtol(s + 1, &s, 10);
			break;
		default: break; // -x: applied in pass 1
		}
	}
	for (int i = optind; i < argc; ++i) a.files.push_back(argv[i]);
	// the struct's string fields point into argv, as the reference's do
	opt.kmer_freq_filename = a.has_kmer ? a.kmer_fn.c_str() : 0;
	opt.split_prefix = a.has_split ? a.split_prefix.c_str() : 0;
	if ((opt.flag & WM_F_SPLICE) && (opt.flag & WM_F_FRAG_MODE)) {
		fprintf(stderr, "[ERROR] --splice and --frag should not be specified at the same time.\n");
		return 1;
	}
	if (!(opt.flag & WM_F_CIGAR)) ipt.flag |= WM_I_NO_SEQ; // src/main.c:280 (no prebuilt index: fnw is never set)
	// mm_check_opt; check_opt also refuses what the mapper does not build (k > 28, w >= 256, wrapping dual gap costs, spliced
	// base alignment), where the reference would go on
	const int rc = check_opt(&ipt, &opt);
	if (rc < 0) {
		static const char *msg[] = { "", "-O and -E must be positive and ({-O}+{-E})+({-O2}+{-E2}) <= 127",
		                             "dual gap penalties violating E1>E2 and O1+E1<O2+E2", "--for-only and --rev-only can't be applied at the same time",
		                             "-N must be no less than 0 and -p within 0 and 1", "-k and -w must be positive (k <= 28, w < 256), Z-drop not less than inversion Z-drop, and -X/-P not with --secondary=no",
		                             "--cs or --MD doesn't work with --split-prefix", "dual gap penalties with -A + O1 + 2*E1 > 128 are not supported",
		                             "spliced base-level alignment (-c, -a or --cs with -x splice, cdna or --splice) is not supported by the command line: it is a library path (Mapper(spliced_alignment=True), wm_map_file)" };
		fprintf(stderr, "[ERROR] %s\n", -rc < (int)(sizeof(msg) / sizeof(msg[0])) ? msg[-rc] : "invalid options");
		return 1;
	}
	if (opt.best_n == 0) {
		fprintf(stderr, "[WARNING] changed '-N 0' to '-N %d --secondary=no'.\n", old_best_n);
		opt.best_n = old_best_n, opt.flag |= WM_F_NO_PRINT_2ND;
	}
	if (a.files.empty() || a.help) {
		usage(a.help ? stdout : stderr, a);
		return a.help ? 0 : 1;
	}
	// the reference opens the index here (a file that cannot be read is reported by cli_main) and then checks these
	if (a.files.size() < 2) { fprintf(stderr, "[ERROR] missing input: please specify a query file to map\n"); return 1; }
	if ((opt.flag & WM_F_CIGAR) && (ipt.flag & WM_I_NO_SEQ)) { // src/main.c:336-341, --idx-no-seq with alignment
		fprintf(stderr, "[ERROR] the prebuilt index doesn't contain sequences.\n");
		return 1;
	}
	// what the mapper does not build: refused before any index is read
	const char *refused = 0;
	if (opt.flag & WM_F_HEAP_SORT) refused = "--heap-sort=yes";
	else if (opt.flag & WM_F_SR) refused = "--sr";
	else if (opt.sdust_thres > 0) refused = "-T (SDUST) above 0";
	else if (opt.flag & WM_F_FRAG_MODE) refused = "--frag=yes (Winnowmap maps single-segment reads only)";
	else if (a.files.size() > 1 && (opt.flag & (WM_F_SPLICE | WM_F_SPLICE_FOR | WM_F_SPLICE_REV)) && (opt.flag & (WM_F_CIGAR | WM_F_OUT_MD)))
		refused = "spliced mapping with -c, -a, --cs or --MD (spliced base-level alignment)";
	else if (a.has_split && a.files.size() > 2) refused = "--split-prefix with more than one query file";
	if (refused) { fprintf(stderr, "[ERROR] winnowmap-b200 does not support %s\n", refused); return 1; }
	return -1;
}

int cli_main(int argc, char **argv, const IndexBuilder &build)
{
	CliArgs a;
	std::string cl = "winnowmap"; // the @PG CL: of the reference names its own program (src/format.c:130-135)
	int rc = cli_parse(argc, argv, a);
	if (rc >= 0) return rc;
	for (int i = 1; i < argc; ++i) cl += ' ', cl += argv[i]; // argv as getopt left it: options first, then the files
	if (a.has_out && a.out_fn != "-" && freopen(a.out_fn.c_str(), "wb", stdout) == 0) {
		fprintf(stderr, "[ERROR] failed to write the output to file '%s': %s\n", a.out_fn.c_str(), strerror(errno));
		return 1;
	}
	{
		SeqReader rd;
		if (!rd.open(a.files[0].c_str())) {
			fprintf(stderr, "[ERROR] failed to open file '%s': %s\n", a.files[0].c_str(), strerror(errno));
			return 1;
		}
	}
	std::unique_ptr<IndexParts> ix = build(a);
	if (!ix) return 1;
	cli_update_opt(&a.opt);
	std::vector<const char*> queries;
	for (size_t i = 1; i < a.files.size(); ++i) queries.push_back(a.files[i].c_str());
	rc = map_files(*ix, &a.opt, queries, 0, cl.c_str(), a.has_rg ? a.rg.c_str() : 0, a.n_threads, 0, 1, 0, 200000000);
	if (fflush(stdout) == EOF) { perror("[ERROR] failed to write the results"); return 1; }
	return rc < 0 ? 1 : 0;
}

} // namespace wmh
