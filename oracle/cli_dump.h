/* TEST INFRASTRUCTURE ONLY: the text form of what a winnowmap command line maps with, written the same way by the wrapped
 * reference main() (cli_ref_dump.c) and by the product's parser (tests/hostsim/cli_backend.cpp) so that the two can be
 * compared line by line.  The option structs are dumped as hex bytes with their two pointer fields zeroed; the strings
 * those fields point to follow on lines of their own.  rg is the -R line the SAM header was given (null: none). */
#ifndef WM_CLI_DUMP_H
#define WM_CLI_DUMP_H
#include <stdint.h>
#include <stdio.h>
#include <string.h>

static void wm_cli_dump_hex(FILE *fp, const char *tag, const void *p, size_t n, size_t z0, size_t z1)
{
	const uint8_t *b = (const uint8_t*)p;
	size_t i;
	fprintf(fp, "%s ", tag);
	for (i = 0; i < n; ++i) fprintf(fp, "%02x", (i >= z0 && i < z0 + sizeof(void*)) || (i >= z1 && i < z1 + sizeof(void*)) ? 0 : b[i]);
	fputc('\n', fp);
}

static void wm_cli_dump(FILE *fp, const void *ipt, size_t ipt_size, const void *opt, size_t opt_size, size_t off_kmer, size_t off_split,
                        int n_threads, const char *rg, int n_files, const char *const *files)
{
	const char *kmer, *split;
	int i;
	memcpy(&kmer, (const char*)opt + off_kmer, sizeof(kmer));
	memcpy(&split, (const char*)opt + off_split, sizeof(split));
	wm_cli_dump_hex(fp, "ipt", ipt, ipt_size, (size_t)-1, (size_t)-1);
	wm_cli_dump_hex(fp, "opt", opt, opt_size, off_kmer, off_split);
	fprintf(fp, "kmer_freq_filename %s\n", kmer ? kmer : "(null)");
	fprintf(fp, "split_prefix %s\n", split ? split : "(null)");
	fprintf(fp, "threads %d\n", n_threads);
	fprintf(fp, "rg %s\n", rg ? rg : "(null)");
	for (i = 0; i < n_files; ++i) fprintf(fp, "file %s\n", files[i]);
}
#endif
