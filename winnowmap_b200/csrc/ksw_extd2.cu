// Banded dual-affine extension DP with traceback on sm_90a.
//
// Computes exactly what ksw_extd2_sse (reference src/ksw2_extd2_sse.c:26-393) computes,
// including the artefacts of its SSE formulation that reach the output (SURVEY.md App. A.1):
// the band is processed in whole 16-cell blocks (:139), the per-diagonal score refresh runs
// in unaligned 16-cell groups past the band end (:158-172), state arrays are int8 with
// wrap-around arithmetic, and the backtrack uses block bounds (src/ksw2.h:119-151).
//
// Mapping to the GPU: one warp owns one DP job and sweeps anti-diagonals r = i + j; lanes
// own consecutive target positions t of the diagonal, the t-1 operand of the recurrence
// comes from the neighbouring lane by shuffle (the SSE code shifts a vector by one byte
// instead).  The production sweep is ksw_extd2_v2.cuh (128 cells per step, 16x2 SIMD with
// tagged maxima); the function in this file is the first-generation sweep (32 cells per
// step, int32 math with int8 wrap casts), kept selectable with WM_DP_V1=1.  State rows live
// in shared memory or, for long targets, in an L2-resident global slice.  Direction bytes
// are streamed to HBM, one row of the rotated matrix per diagonal; a second kernel walks
// them back (one thread per job), emits the CIGAR and, for gap fills, the Z-drop score walk.
#include <mutex>
#include <vector>
#include <algorithm>
#include <utility>
#include "wm_common.cuh"

#define WM_FILL_WARPS 4
#define WM_SMEM_CELLS 1024   // first-generation path: per-warp shared-memory slice covers tlen <= 1024
#define WM_FILL_SLICE (WM_SMEM_CELLS * 11 > WM_V2_SLICE_C ? WM_SMEM_CELLS * 11 : WM_V2_SLICE_C)
#define WM_V2_SLICE_C ((7 * 2 * (512 + 8) + 4 * 512 + (512 + 16) + (640 + 64) + 640 + 16 + 15) / 16 * 16)

#include "ksw_extd2_common.cuh"

__device__ void wm_extd2_fill_job(const wm_dp_job &J, const uint8_t *__restrict__ seq, uint8_t *__restrict__ bt,
                                  wm_extz_dev *out, const wm_dp_params &P, int8_t *S, int lane, unsigned long long *cell_ctr)
{
	unsigned long long cells_acc = 0;
	const unsigned FULL = 0xffffffffu;
	const uint8_t *query = seq + J.q_off, *target = seq + J.t_off;
	const int qlen = J.qlen, tlen = J.tlen, flag = J.flag;
	int w = J.w;
	wm_extz_dev ez;
	ez.max_q = ez.max_t = ez.mqe_t = ez.mte_q = -1;
	ez.max = 0, ez.score = ez.mqe = ez.mte = WM_NEG_INF;
	ez.n_cigar = 0, ez.zdropped = 0, ez.reach_end = 0, ez.reserved = 0;
	if (qlen <= 0 || tlen <= 0 || P.early_out) { if (lane == 0) *out = ez; return; }

	const int q = P.q, e = P.e, q2 = P.q2, e2 = P.e2, qe = q + e, qe2 = q2 + e2;
	const bool approx_max = (flag & 0x08) != 0, right = (flag & 0x02) != 0;
	if (w < 0) w = tlen > qlen ? tlen : qlen;
	const int tlen16 = (tlen + 15) / 16 * 16;
	const int n_col16 = wm_ncol16(qlen, tlen, w);
	int8_t *u = S, *v = u + tlen16, *x = v + tlen16, *y = x + tlen16, *x2 = y + tlen16, *y2 = x2 + tlen16, *s = y2 + tlen16;
	int32_t *H = (int32_t*)(s + tlen16);
	for (int i = lane; i < tlen16; i += 32) {
		u[i] = v[i] = x[i] = y[i] = (int8_t)(-q - e);
		x2[i] = y2[i] = (int8_t)(-q2 - e2);
		s[i] = 0;
		if (!approx_max) H[i] = WM_NEG_INF;
	}
	__syncwarp();

	int32_t H0 = 0, last_H0_t = 0;
	int last_st = -1, last_en = -1;
	const int n_diag = qlen + tlen - 1;
	for (int r = 0; r < n_diag; ++r) {
		const int st0 = wm_band_st(r, qlen, w), en0 = wm_band_en(r, tlen, w);
		if (st0 > en0) { ez.zdropped = 1; break; }
		const int st = st0 / 16 * 16, en = (en0 + 16) / 16 * 16 - 1;
		cells_acc += (unsigned long long)(en - st + 1);
		// boundary operands (src/ksw2_extd2_sse.c:141-151)
		int x1, x21, v1;
		const int bnd = r == 0 ? -q - e : r < P.long_thres ? -e : r == P.long_thres ? P.long_diff : -e2;
		if (st > 0) {
			if (st - 1 >= last_st && st - 1 <= last_en) x1 = x[st - 1], x21 = x2[st - 1], v1 = v[st - 1];
			else x1 = -q - e, x21 = -q2 - e2, v1 = -q - e;
		} else x1 = -q - e, x21 = -q2 - e2, v1 = bnd;
		if (en >= r && lane == 0) { // :152-155
			y[r] = (int8_t)(-q - e), y2[r] = (int8_t)(-q2 - e2);
			u[r] = (int8_t)bnd;
		}
		// score refresh in unaligned 16-cell groups starting at st0 (:158-172)
		{
			const int lim = st0 + ((en0 - st0) / 16 + 1) * 16;
			for (int i = st0 + lane; i < lim; i += 32) {
				if (i < tlen16) { // writes past the s[] row land in sf[] in the reference and are never read back
					int sq = i < tlen ? target[i] : 0;             // sf[] is zero padded up to tlen16
					int j = r - i;                                  // qrr[i] = qr[qlen-1-r+i] = query[r-i]; zero padded
					int sr = (j >= 0 && j < qlen) ? query[j] : 0;
					s[i] = (int8_t)((sq == 4 || sr == 4) ? P.sc_N : (sq == sr ? P.sc_mch : P.sc_mis));
				}
			}
		}
		__syncwarp();
		// the cells of this diagonal, whole 16-cell blocks [st, en]
		{
			int cx = x1, cv = v1, cx2 = x21;
			uint8_t *pr = bt + J.p_off + (size_t)r * n_col16;
			for (int c = st; c <= en; c += 32) {
				const int t = c + lane;
				const bool act = t <= en;
				int z = 0, xo = 0, vo = 0, x2o = 0, uo = 0, yo = 0, y2o = 0;
				if (act) z = s[t], xo = x[t], vo = v[t], x2o = x2[t], uo = u[t], yo = y[t], y2o = y2[t];
				int xl = __shfl_up_sync(FULL, xo, 1), vl = __shfl_up_sync(FULL, vo, 1), x2l = __shfl_up_sync(FULL, x2o, 1);
				if (lane == 0) xl = cx, vl = cv, x2l = cx2;
				cx = __shfl_sync(FULL, xo, 31), cv = __shfl_sync(FULL, vo, 31), cx2 = __shfl_sync(FULL, x2o, 31);
				if (act) {
					int a = (int8_t)(xl + vl), b = (int8_t)(yo + uo), a2 = (int8_t)(x2l + vl), b2 = (int8_t)(y2o + uo), d, tmp;
					if (!right) { // :227-234
						d = 0;
						if (a > z) d = 1, z = a;
						if (b > z) d = 2, z = b;
						if (a2 > z) d = 3, z = a2;
						if (b2 > z) d = 4, z = b2;
					} else { // :274-281
						d = z > a ? 0 : 1; z = max(z, a);
						d = z > b ? d : 2; z = max(z, b);
						d = z > a2 ? d : 3; z = max(z, a2);
						d = z > b2 ? d : 4; z = max(z, b2);
					}
					z = min(z, P.sc_mch);
					u[t] = (int8_t)(z - vl); v[t] = (int8_t)(z - uo);
					tmp = (int8_t)(z - q);  a = (int8_t)(a - tmp);  b = (int8_t)(b - tmp);
					tmp = (int8_t)(z - q2); a2 = (int8_t)(a2 - tmp); b2 = (int8_t)(b2 - tmp);
					if (!right) { // :253-264
						x[t]  = (int8_t)((a  > 0 ? a  : 0) - qe);  d |= a  > 0 ? 0x08 : 0;
						y[t]  = (int8_t)((b  > 0 ? b  : 0) - qe);  d |= b  > 0 ? 0x10 : 0;
						x2[t] = (int8_t)((a2 > 0 ? a2 : 0) - qe2); d |= a2 > 0 ? 0x20 : 0;
						y2[t] = (int8_t)((b2 > 0 ? b2 : 0) - qe2); d |= b2 > 0 ? 0x40 : 0;
					} else { // :300-311
						x[t]  = (int8_t)((a  < 0 ? 0 : a ) - qe);  d |= a  < 0 ? 0 : 0x08;
						y[t]  = (int8_t)((b  < 0 ? 0 : b ) - qe);  d |= b  < 0 ? 0 : 0x10;
						x2[t] = (int8_t)((a2 < 0 ? 0 : a2) - qe2); d |= a2 < 0 ? 0 : 0x20;
						y2[t] = (int8_t)((b2 < 0 ? 0 : b2) - qe2); d |= b2 < 0 ? 0 : 0x40;
					}
					pr[t - st] = (uint8_t)d;
				}
			}
		}
		__syncwarp();
		if (!approx_max) { // exact max with the 32-bit H row (:315-358)
			int32_t max_H, max_t;
			if (r > 0) {
				const int32_t Hm1 = en0 > 0 ? H[en0 - 1] : 0, Hen = H[en0];
				__syncwarp();
				const int en1 = st0 + (en0 - st0) / 4 * 4;
				long long best = (long long)0x8000000000000000LL;
				for (int t = st0 + lane; t < en0; t += 32) {
					int32_t h = H[t] + v[t];
					H[t] = h;
					uint32_t prio = t < en1 ? 1u + ((uint32_t)((t - st0) & 3) << 24) + (uint32_t)((t - st0) >> 2 << 2)
					                        : (1u << 27) + (uint32_t)(t - st0);
					long long key = ((long long)h << 32) | (long long)(0xffffffffu - prio);
					best = key > best ? key : best;
				}
				const int32_t Hn = en0 > 0 ? Hm1 + u[en0] : Hen + v[en0]; // special-cased last element (:319)
				if (lane == 0) H[en0] = Hn;
				{
					long long key = ((long long)Hn << 32) | (long long)0xffffffffu; // prio 0: H[en0] seeds the max
					best = key > best ? key : best;
				}
				#pragma unroll
				for (int o = 16; o; o >>= 1) {
					long long other = __shfl_xor_sync(FULL, best, o);
					best = other > best ? other : best;
				}
				max_H = (int32_t)(best >> 32);
				uint32_t prio = 0xffffffffu - (uint32_t)(best & 0xffffffffLL);
				if (prio == 0) max_t = en0;
				else if (prio < (1u << 27)) max_t = st0 + (int)((prio - 1) & 0xffffffu) + (int)((prio - 1) >> 24); // block base + lane (:342)
				else max_t = st0 + (int)(prio - (1u << 27));
				__syncwarp();
			} else {
				max_H = (int32_t)v[0] - P.qe_h, max_t = 0; // :351
				if (lane == 0) H[0] = max_H;
				__syncwarp();
			}
			const int32_t Hen0 = H[en0], Hst0 = H[st0];
			if (en0 == tlen - 1 && Hen0 > ez.mte) ez.mte = Hen0, ez.mte_q = r - en;
			if (r - st0 == qlen - 1 && Hst0 > ez.mqe) ez.mqe = Hst0, ez.mqe_t = st0;
			if (wm_apply_zdrop(ez, max_H, r, max_t, J.zdrop, e2)) break;
			if (r == qlen + tlen - 2 && en0 == tlen - 1) ez.score = H[tlen - 1];
		} else { // approximate max (:359-375)
			if (r > 0) {
				if (last_H0_t >= st0 && last_H0_t <= en0 && last_H0_t + 1 >= st0 && last_H0_t + 1 <= en0) {
					int32_t d0 = v[last_H0_t], d1 = u[last_H0_t + 1];
					if (d0 > d1) H0 += d0;
					else H0 += d1, ++last_H0_t;
				} else if (last_H0_t >= st0 && last_H0_t <= en0) {
					H0 += v[last_H0_t];
				} else {
					++last_H0_t, H0 += u[last_H0_t];
				}
			} else H0 = (int32_t)v[0] - P.qe_h, last_H0_t = 0;
			if ((flag & 0x10) && wm_apply_zdrop(ez, H0, r, last_H0_t, J.zdrop, e2)) break;
			if (r == qlen + tlen - 2 && en0 == tlen - 1) ez.score = H0;
		}
		last_st = st, last_en = en;
	}
	if (lane == 0) { *out = ez; if (cell_ctr) atomicAdd(cell_ctr, cells_acc); }
}

#include "ksw_extd2_v2.cuh"
#include "ksw_extz2.cuh"
#include "ksw_exts2.cuh"

__global__ void __launch_bounds__(WM_FILL_WARPS * 32, 4)
wm_extd2_fill_kernel(const wm_dp_job *__restrict__ jobs, int n_jobs, const uint8_t *__restrict__ seq, uint8_t *__restrict__ bt,
                     wm_extz_dev *__restrict__ ez, wm_dp_params P, int8_t *gscratch, size_t gscratch_stride, int g_tcap, int g_qcap, int use_v2,
                     unsigned long long *cell_ctr, const uint8_t *__restrict__ junc_pool)
{
	// One job per warp, four consecutive jobs per CTA: jobs come largest first, so the four are of similar size and the
	// CTA leaves its SM as soon as they are done (a persistent grid would hold every SM for the whole launch and keep
	// the short kernels of the other orchestration lanes waiting).
	extern __shared__ __align__(16) int8_t smem[];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	int8_t *my_smem = smem + (size_t)wid * WM_FILL_SLICE;
	const int j = blockIdx.x * WM_FILL_WARPS + wid;
	if (j >= n_jobs) return;
	const wm_dp_job J = jobs[j];
	if (J.flag & WM_DP_COOP) return; // swept by a whole CTA in wm_extd2_fill_coop_kernel
	int8_t *my_g = J.pad >= 0 ? gscratch + (size_t)J.pad * gscratch_stride : (int8_t*)0;
	const int tlen16 = (J.tlen + 15) / 16 * 16;
	if (P.splice) wm_exts2_fill_job(J, seq, junc_pool ? junc_pool + J.t_off : 0, bt, ez + j, P, J.pad < 0 ? my_smem : my_g, lane, cell_ctr);
	else if (P.single) wm_extz2_fill_job(J, seq, bt, ez + j, P, tlen16 <= WM_SMEM_CELLS ? my_smem : my_g, lane, cell_ctr);
	else if (use_v2 && J.qlen > 0 && J.tlen > 0 && !P.early_out) {
		if (J.pad < 0) wm_extd2_fill_job_v2<true>(J, seq, bt, ez + j, P, (uint8_t*)my_smem, 0, 0, lane, cell_ctr ? cell_ctr + 1 : 0);
		else wm_extd2_fill_job_v2<false>(J, seq, bt, ez + j, P, (uint8_t*)my_g, g_tcap, g_qcap, lane, cell_ctr ? cell_ctr + 1 : 0);
	} else
		wm_extd2_fill_job(J, seq, bt, ez + j, P, tlen16 <= WM_SMEM_CELLS ? my_smem : my_g, lane, cell_ctr);
}

// the big jobs, one CTA each (ksw_extd2_v2.cuh: wm_extd2_fill_job_v2_cta)
__global__ void __launch_bounds__(WM_V2_CTA_WARPS * 32)
wm_extd2_fill_coop_kernel(const wm_dp_job *__restrict__ jobs, const int32_t *__restrict__ ids, int n_ids, const uint8_t *__restrict__ seq, uint8_t *__restrict__ bt,
                          wm_extz_dev *__restrict__ ez, wm_dp_params P, int8_t *gscratch, size_t gscratch_stride, int g_tcap, int g_qcap, unsigned long long *cell_ctr)
{
	__shared__ wm_v2_cta_sm SM;
	for (int i = blockIdx.x; i < n_ids; i += gridDim.x) {
		const int j = ids[i];
		const wm_dp_job J = jobs[j];
		wm_extd2_fill_job_v2_cta(J, seq, bt, ez + j, P, (uint8_t*)(gscratch + (size_t)J.pad * gscratch_stride), g_tcap, g_qcap, &SM, cell_ctr ? cell_ctr + 1 : 0);
		__syncthreads();
	}
}

__global__ void wm_extd2_backtrack_kernel(const wm_dp_job *__restrict__ jobs, int n_jobs, const uint8_t *__restrict__ bt,
                                          wm_extz_dev *__restrict__ ezs, uint32_t *__restrict__ cigar_pool,
                                          const uint8_t *__restrict__ seq, wm_zd_params Z, int32_t *__restrict__ zd, int splice, int min_intron_len, int early_out)
{
	const int jid = blockIdx.x * blockDim.x + threadIdx.x;
	if (jid >= n_jobs) return;
	const wm_dp_job J = jobs[jid];
	wm_extd2_backtrack_job(J, ezs + jid, bt, cigar_pool, seq, Z, zd ? zd + 5 * (size_t)jid : 0, splice, min_intron_len, early_out);
}

// ---- host-side launcher on device-resident jobs ----

void wm_dp_params_init(wm_dp_params *P, const int8_t *mat, int q, int e, int q2, int e2)
{ // src/ksw2_extd2_sse.c:61-97
	P->single = q == q2 && e == e2; // src/align.c:328-331: ksw_extz2_sse(q, e) instead
	P->splice = 0, P->noncan = P->junc_bonus = 0; memcpy(P->mat, mat, 25);
	P->qe_h = q + e;
	if (q2 + e2 < q + e) { int t = q; q = q2; q2 = t; t = e; e = e2; e2 = t; }
	P->q = q, P->e = e, P->q2 = q2, P->e2 = e2;
	P->sc_mch = mat[0], P->sc_mis = mat[1];
	P->sc_N = mat[24] == 0 ? -e2 : mat[24];
	int max_sc = mat[0], min_sc = mat[1];
	for (int t = 1; t < 25; ++t) { max_sc = max_sc > mat[t] ? max_sc : mat[t]; min_sc = min_sc < mat[t] ? min_sc : mat[t]; }
	P->early_out = -min_sc > 2 * (q + e);
	int long_thres = e != e2 ? (q2 - q) / (e - e2) - 1 : 0;
	if (q2 + e2 + long_thres * e2 > q + e + long_thres * e) ++long_thres;
	P->long_thres = long_thres;
	P->long_diff = long_thres * (e - e2) - (q2 - q) - e2;
}

void wm_dp_params_init_splice(wm_dp_params *P, const int8_t *mat, int q, int e, int q2, int noncan, int junc_bonus)
{ // src/ksw2_exts2_sse.c:61-84
	memset(P, 0, sizeof(*P));
	P->splice = 1, P->noncan = noncan, P->junc_bonus = junc_bonus; memcpy(P->mat, mat, 25);
	P->q = q, P->e = e, P->q2 = q2, P->e2 = 0, P->qe_h = q + e;
	P->sc_mch = mat[0], P->sc_mis = mat[1];
	P->sc_N = mat[24] == 0 ? -e : mat[24];
	int min_sc = mat[1];
	for (int t = 1; t < 25; ++t) min_sc = min_sc < mat[t] ? min_sc : mat[t];
	P->early_out = q2 <= q + e || -min_sc > 2 * (q + e);
	if (e <= 0) { P->early_out = 1; return; } // (the reference divides by e)
	int long_thres = (q2 - q) / e - 1;
	if (q2 > q + e + long_thres * e) ++long_thres;
	P->long_thres = long_thres;
	P->long_diff = long_thres * e - (q2 - q);
}

size_t wm_extd2_bt_bytes(int qlen, int tlen, int w)
{
	if (qlen <= 0 || tlen <= 0) return 16;
	if (w < 0) w = tlen > qlen ? tlen : qlen;
	int n = qlen < tlen ? qlen : tlen;
	n = ((n < w + 1 ? n : w + 1) + 15) / 16 + 1;
	return ((size_t)(qlen + tlen - 1) * n + 1) * 16;
}

static int wm_use_v2(void)
{
	static int use_v2 = -1;
	if (use_v2 < 0) { const char *e = getenv("WM_DP_V1"); use_v2 = (e && *e == '1') ? 0 : 1; }
	return use_v2;
}

size_t wm_exts2_scratch_bytes(int tlen)
{
	const size_t b = (size_t)(tlen + 15) / 16 * 16 * WM_EXTS2_CELL_BYTES;
	return b <= WM_FILL_SLICE ? 0 : b;
}

wm_extd2_plan_t wm_extd2_plan(wm_dp_job *h_jobs, int n, bool single, bool splice)
{
	wm_extd2_plan_t pl; pl.n_slots = 0, pl.max_tlen = 0, pl.max_qlen = 0, pl.splice_bytes = 0;
	if (splice) { // one slice per job, of the job's own size: J.pad counts WM_EXTS2_PAD_UNIT bytes
		for (int i = 0; i < n; ++i) {
			wm_dp_job &J = h_jobs[i];
			const size_t b = wm_exts2_scratch_bytes(J.tlen);
			J.pad = b == 0 ? -1 : (int32_t)(pl.splice_bytes / WM_EXTS2_PAD_UNIT);
			pl.splice_bytes += b;
		}
		return pl;
	}
	const int use_v2 = single ? 0 : wm_use_v2();
	for (int i = 0; i < n; ++i) {
		wm_dp_job &J = h_jobs[i];
		const int tlen16 = (J.tlen + 15) / 16 * 16;
		const bool fits = use_v2 ? (tlen16 <= WM_V2_T && J.qlen <= WM_V2_Q) : tlen16 <= WM_SMEM_CELLS;
		J.pad = fits ? -1 : pl.n_slots++;
		if (!fits) { if (J.tlen > pl.max_tlen) pl.max_tlen = J.tlen; if (J.qlen > pl.max_qlen) pl.max_qlen = J.qlen; }
	}
	return pl;
}

cudaStream_t wm_stream_create_high_priority(void)
{
	int lo = 0, hi = 0;
	cudaStream_t st;
	WM_CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&lo, &hi)); // numerically: hi <= lo
	WM_CUDA_CHECK(cudaStreamCreateWithPriority(&st, cudaStreamDefault, hi));
	return st;
}

void wm_extd2_launch(wm_extd2_ws *ws, const wm_dp_job *d_jobs, int n_jobs, const wm_extd2_plan_t &plan, const uint8_t *d_seq, uint8_t *d_bt,
                     wm_extz_dev *d_ez, uint32_t *d_cigar, const wm_dp_params &P, cudaStream_t stream, const wm_zd_params *zp, int32_t *d_zd,
                     const int32_t *d_coop_ids, int n_coop, const uint8_t *d_junc, int8_t *d_scratch)
{
	if (n_jobs <= 0) return;
	const size_t smem = (size_t)WM_FILL_WARPS * WM_FILL_SLICE;
	const int use_v2 = P.single || P.splice ? 0 : wm_use_v2();
	const int grid = (n_jobs + WM_FILL_WARPS - 1) / WM_FILL_WARPS;
	// global state slices of the jobs that do not fit the shared-memory slice (wm_extd2_plan gave them slots; a splice job's
	// slot is the offset of its own slice, in WM_EXTS2_PAD_UNIT bytes)
	const int tcap = (plan.max_tlen + 15) / 16 * 16;
	const size_t stride = P.splice ? WM_EXTS2_PAD_UNIT : plan.n_slots == 0 ? 0 : use_v2 ? wm_v2_slice_bytes(tcap, plan.max_qlen) : (size_t)tcap * 11;
	int8_t *gs = d_scratch ? d_scratch : (int8_t*)ws->scratch.need((P.splice ? plan.splice_bytes : stride * (size_t)plan.n_slots) + 16);
	if (!ws->fill_st) {
		int lo = 0, hi = 0;
		WM_CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
		const char *pe = getenv("WM_FILL_PRIO"); // tuning: "high" puts the DP fill on the same priority as the other kernels
		const int prio = (pe && *pe == 'h') ? hi : lo;
		WM_CUDA_CHECK(cudaStreamCreateWithPriority(&ws->fill_st, cudaStreamNonBlocking, prio));
		WM_CUDA_CHECK(cudaStreamCreateWithPriority(&ws->coop_st, cudaStreamNonBlocking, prio));
		WM_CUDA_CHECK(cudaEventCreateWithFlags(&ws->ev_ready, cudaEventDisableTiming));
		WM_CUDA_CHECK(cudaEventCreateWithFlags(&ws->ev_done, cudaEventDisableTiming));
		WM_CUDA_CHECK(cudaEventCreateWithFlags(&ws->ev_coop, cudaEventDisableTiming));
	}
	static bool attr_set = false;
	if (!attr_set) {
		WM_CUDA_CHECK(cudaFuncSetAttribute(wm_extd2_fill_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
		attr_set = true;
	}
	WM_CUDA_CHECK(cudaEventRecord(ws->ev_ready, stream));
	WM_CUDA_CHECK(cudaStreamWaitEvent(ws->fill_st, ws->ev_ready, 0));
	// bench mode: an event pair and a cell-counter slot per launch (prof.cu); nothing is synchronised here, so the
	// timed region runs exactly as it does without profiling
	unsigned long long *cell_ctr = 0;
	const int pslot = wm_prof_launch_begin(WM_PK_FILL, ws->fill_st, ws->fill_st, &cell_ctr);
	if (n_coop > 0 && use_v2) { // the big jobs first, on their own stream: they set the length of the launch
		WM_CUDA_CHECK(cudaStreamWaitEvent(ws->coop_st, ws->ev_ready, 0));
		wm_count_launch(); wm_extd2_fill_coop_kernel<<<n_coop, WM_V2_CTA_WARPS * 32, 0, ws->coop_st>>>(d_jobs, d_coop_ids, n_coop, d_seq, d_bt, d_ez, P, gs, stride, tcap, plan.max_qlen, cell_ctr);
		WM_CUDA_CHECK(cudaGetLastError());
		WM_CUDA_CHECK(cudaEventRecord(ws->ev_coop, ws->coop_st));
	}
	wm_count_launch(); wm_extd2_fill_kernel<<<grid, WM_FILL_WARPS * 32, smem, ws->fill_st>>>(d_jobs, n_jobs, d_seq, d_bt, d_ez, P, gs, stride, tcap, plan.max_qlen, use_v2, cell_ctr, d_junc);
	WM_CUDA_CHECK(cudaGetLastError());
	if (n_coop > 0 && use_v2) WM_CUDA_CHECK(cudaStreamWaitEvent(ws->fill_st, ws->ev_coop, 0));
	wm_prof_launch_end(pslot, ws->fill_st);
	WM_CUDA_CHECK(cudaEventRecord(ws->ev_done, ws->fill_st));
	WM_CUDA_CHECK(cudaStreamWaitEvent(stream, ws->ev_done, 0));
	wm_zd_params Z; memset(&Z, 0, sizeof(Z));
	if (zp && d_zd) Z = *zp;
	wm_count_launch(); wm_extd2_backtrack_kernel<<<(n_jobs + 127) / 128, 128, 0, stream>>>(d_jobs, n_jobs, d_bt, d_ez, d_cigar, d_seq, Z, zp ? d_zd : 0, P.splice, P.splice ? P.long_thres : 0, P.early_out);
	WM_CUDA_CHECK(cudaGetLastError());
}

