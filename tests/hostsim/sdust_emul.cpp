// TEST INFRASTRUCTURE.  The device code of -T (csrc/sdust.cuh: wm_sdust_seq, one thread per sequence, and wm_dust_keep, the
// squeeze test of the sketch's dust pass) compiled for the host on top of cuda_emul.h, so that tests/test_sdust_cpu.py can
// check it against the oracle (oracle/wm_oracle_sdust.c) without a GPU.
#include <vector>
#include "cuda_emul.h"
#include "../../winnowmap_b200/csrc/sdust.cuh"

namespace {
struct AsciiBase { // seq_nt4_table, as the packed pool stores it (csrc/sketch.cu: wm_nt4)
	const unsigned char *s;
	int operator()(int i) const
	{
		switch (s[i]) { case 'A': case 'a': return 0; case 'C': case 'c': return 1; case 'G': case 'g': return 2;
		                case 'T': case 't': case 'U': case 'u': return 3; default: return s[i] < 4 ? s[i] : 4; }
	}
};
}

// the regions of seq[0, len) (at most max_out written, at the device's capacity wm_sdust_reg_cap) with a perfect-interval list of
// pcap entries (0: WM_SDUST_PCAP, the second pass's); -2 when the device code gives the sequence up (the list would outgrow pcap),
// -1 when it reports an overflow of the regions
extern "C" long wmt_sdust_dev(const char *seq, int len, int T, int W, int pcap, uint64_t *out, long max_out)
{
	if (pcap <= 0) pcap = WM_SDUST_PCAP;
	std::vector<wm_sdust_perf> P(pcap);
	std::vector<uint64_t> res(wm_sdust_reg_cap(len, W));
	AsciiBase b; b.s = (const unsigned char*)seq;
	int err = 0;
	const int64_t n = wm_sdust_seq(b, len, T, W, P.data(), pcap, res.data(), (int64_t)res.size(), &err);
	if (n < 0) return -2;
	if (err) return -1;
	for (int64_t i = 0; i < n && i < max_out; ++i) out[i] = res[i];
	return (long)n;
}

// the sketch's dust pass on n minimizers (x, y pairs, position order): squeezed in place as wm_dust_keep decides; returns how
// many are kept
extern "C" long wmt_dust_squeeze_dev(uint64_t *xy, long n, const uint64_t *reg, int n_reg)
{
	long k = 0;
	for (long j = 0; j < n; ++j)
		if (wm_dust_keep(reg, n_reg, (int32_t)((uint32_t)xy[2 * j + 1] >> 1), (int32_t)(xy[2 * j] & 0xff)))
			xy[2 * k] = xy[2 * j], xy[2 * k + 1] = xy[2 * j + 1], ++k;
	return k;
}
