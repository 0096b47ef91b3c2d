/* TEST INFRASTRUCTURE ONLY -- never linked, imported or executed by the product path.
 *
 * Linked with the reference's own main.o (oracle/build_cli_ref.sh) through -Wl,--wrap= for its index-reader and mapping
 * entry points: the reference's real option handling runs, and instead of building an index and mapping, the wrappers
 * record what main() hands to them -- mm_idx_reader_open's file and mm_idxopt_t, mm_map_file's mm_mapopt_t, thread count
 * and query files, mm_write_sam_hdr's read group -- and write it at exit, in the format of cli_dump.h, to the file named by
 * $WM_CLI_DUMP.  Nothing is written when main() returns before mapping.  mm_mapopt_update keeps its index-free steps (the
 * splice flag of -u and the --min-occ-floor clamp); -f stays unresolved.  The processor count is fixed at 8 so that the
 * default thread count does not depend on the machine.  Compiled as C++: minimap.h includes C++ headers. */
#include <sched.h>
#include <stdlib.h>
#include <string.h>
#include "minimap.h"
#include "cli_dump.h"

extern "C" {

static mm_idxopt_t g_ipt;
static mm_mapopt_t g_opt;
static int g_threads, g_mapped, g_n_files;
static const char *g_files[256];
static const char *g_rg;

static void dump_at_exit(void)
{
	const char *fn = getenv("WM_CLI_DUMP");
	FILE *fp;
	if (!g_mapped || !fn || !(fp = fopen(fn, "w"))) return;
	wm_cli_dump(fp, &g_ipt, sizeof(g_ipt), &g_opt, sizeof(g_opt), offsetof(mm_mapopt_t, kmer_freq_filename), offsetof(mm_mapopt_t, split_prefix),
	            g_threads, g_rg, g_n_files, g_files);
	fclose(fp);
}

int __wrap_sched_getaffinity(pid_t pid, size_t size, cpu_set_t *cs)
{
	int i;
	(void)pid;
	CPU_ZERO_S(size, cs);
	for (i = 0; i < 8; ++i) CPU_SET_S(i, size, cs);
	return 0;
}

mm_idx_reader_t *__wrap_mm_idx_reader_open(const char *fn, const mm_idxopt_t *opt, const char *fn_out)
{
	mm_idx_reader_t *r = (mm_idx_reader_t*)calloc(1, sizeof(mm_idx_reader_t));
	(void)fn_out;
	g_ipt = *opt;
	g_files[g_n_files++] = fn;
	atexit(dump_at_exit);
	return r;
}

mm_idx_t *__wrap_mm_idx_reader_read(mm_idx_reader_t *r, int n_threads, const char *kmer_fn)
{
	mm_idx_t *mi;
	(void)n_threads, (void)kmer_fn;
	if (r->n_parts > 0) return 0;
	++r->n_parts;
	mi = (mm_idx_t*)calloc(1, sizeof(mm_idx_t));
	mi->flag = g_ipt.flag, mi->k = g_ipt.k, mi->w = g_ipt.w;
	return mi;
}

int __wrap_mm_idx_reader_eof(const mm_idx_reader_t *r) { (void)r; return 1; }
void __wrap_mm_idx_reader_close(mm_idx_reader_t *r) { free(r); }
void __wrap_mm_idx_destroy(mm_idx_t *mi) { free(mi); }
void __wrap_mm_idx_stat(const mm_idx_t *mi) { (void)mi; }
int __wrap_mm_idx_bed_read(mm_idx_t *mi, const char *fn, int read_junc) { (void)mi, (void)fn, (void)read_junc; return 0; }

void __wrap_mm_mapopt_update(mm_mapopt_t *opt, const mm_idx_t *mi)
{
	(void)mi;
	if ((opt->flag & MM_F_SPLICE_FOR) || (opt->flag & MM_F_SPLICE_REV)) opt->flag |= MM_F_SPLICE;
	if (!(opt->mid_occ_frac >= 0 && opt->mid_occ_frac < 1) && opt->mid_occ < opt->min_mid_occ) opt->mid_occ = opt->min_mid_occ;
}

int __wrap_mm_write_sam_hdr(const mm_idx_t *mi, const char *rg, const char *ver, int argc, char *argv[])
{
	(void)mi, (void)ver, (void)argc, (void)argv;
	g_rg = rg;
	return 0;
}

int __wrap_mm_map_file_frag(const mm_idx_t *idx, int n_segs, const char **fn, const mm_mapopt_t *opt, int n_threads)
{
	int i;
	(void)idx;
	g_opt = *opt, g_threads = n_threads, g_mapped = 1;
	for (i = 0; i < n_segs && g_n_files < 256; ++i) g_files[g_n_files++] = fn[i];
	return 0;
}

int __wrap_mm_map_file(const mm_idx_t *idx, const char *fn, const mm_mapopt_t *opt, int n_threads)
{
	return __wrap_mm_map_file_frag(idx, 1, &fn, opt, n_threads);
}

int __wrap_mm_split_merge(int n, const char **fn, const mm_mapopt_t *opt, int n_split_idx)
{
	(void)n, (void)fn, (void)opt, (void)n_split_idx;
	return 0;
}

} // extern "C"
