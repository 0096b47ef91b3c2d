// TEST INFRASTRUCTURE.  The device code of the junction annotation (csrc/bed_junc.cuh: wm_bed_junc_window, one warp per target
// window) compiled for the host on top of cuda_emul.h and run on the software warp of kernel_emul.cpp, so that
// tests/test_junc_cpu.py can check it against the oracle (oracle/wm_oracle_junc.c) without a GPU.
#include <vector>
#include "cuda_emul.h"
#include "../../winnowmap_b200/csrc/bed_junc.cuh"

// the annotation of window (rid, off, len, reversed) over intervals st / en / strand with per-sequence offsets off[0..n_seq]
// (strand-0 intervals already dropped, as the upload drops them) into out[0..len); the words it covers start out as garbage
extern "C" void wmt_bed_junc_dev(const int32_t *st, const int32_t *en, const int8_t *strand, const int64_t *off, int n_seq, int rid, int w_off,
                                 int len, int reversed, uint8_t *out)
{
	std::vector<uint32_t> buf((size_t)(len + 3) / 4 + 1, 0xa5a5a5a5u);
	struct Args { wm_junc_dev I; wm_junc_win W; uint8_t *out; } A;
	A.I.st = st, A.I.en = en, A.I.strand = strand, A.I.off = off, A.I.n_seq = n_seq;
	A.W.dst_off = 0, A.W.rid = rid, A.W.off = w_off, A.W.len = len, A.W.reversed = reversed;
	A.out = (uint8_t*)buf.data();
	wm_emul::run_warp([](int l, void *p) { Args &a = *(Args*)p; wm_bed_junc_window(a.I, a.W, a.out, l); }, &A);
	memcpy(out, buf.data(), (size_t)len);
}
