// Second-generation fill for jobs whose state fits the per-warp shared-memory slice (the common gap-fill
// case).  Included by ksw_extd2.cu.
//
// Two cells per 32-bit register as signed 16-bit halves, native 16x2 SIMD (VIADD.16x2 / VIMNMX.S16x2 /
// VIADDMNMX.S16x2).  All DP quantities are kept multiplied by 8, and the three free low bits carry tags.  The
// reference keeps them in int8 lanes.  Those stay in [-128, 127] when the gap sum (q + e) + (q2 + e2) is at most 127
// and -A + q + 2e at most 128 (both enforced by check_opt, csrc/host_io.cpp; the second is its return code -7, not in
// the reference) and no score is below -2(q + e) (otherwise the fill returns before the sweep, as the reference does).
// Times 8 that is well inside 16 bits: the sweep never wraps, and neither does the reference.  The tags:
//  * in the max() that picks z, a tie-break tag, so that one max yields both the best state value and WHICH
//    state produced it, in the reference's tie order (left-aligned: first of equals, src/ksw2_extd2_sse.c:227-234;
//    right-aligned: last of equals, :274-281);
//  * in the max() that clamps the four gap states, a tag that records which operand won, i.e. the
//    continuation flag of the direction byte (:253-264 / :300-311).
// A step of the diagonal sweep covers 128 cells (four per lane); the last step of a diagonal covers 64 cells
// (two per lane) when that is enough.  Direction bytes are stored 4 (2) per lane.  Semantics (block rounding,
// stale score cells, H tracking, Z-drop) are those of the first-generation code in ksw_extd2.cu.
#pragma once

#define WM_V2_T 512      // max tlen16 handled in shared memory
#define WM_V2_Q 640      // max qlen
#define WM_V2_TS (WM_V2_T + 8)
// state rows + H + target + reversed query, then (shared-memory slices only) the landing zone of the query's bulk copy and the
// warp's mbarrier
#define WM_V2_SLICE (7 * 2 * WM_V2_TS + 4 * WM_V2_T + (WM_V2_T + 16) + (WM_V2_Q + 64) + WM_V2_Q + 16)

// (bulk-asynchronous staging helpers -- cp.async.bulk + mbarrier -- are in wm_common.cuh)


__device__ __forceinline__ uint32_t wm_pack2(int lo, int hi) { return ((uint32_t)lo & 0xffffu) | ((uint32_t)hi << 16); }
__device__ __forceinline__ uint32_t wm_rep2(int v) { return wm_pack2(v, v); }
// prmt.b32 in its default mode: a selector nibble with bit 3 set replicates the sign bit of the selected byte
// (the __byte_perm intrinsic only defines the low 3 bits of each nibble)
__device__ __forceinline__ uint32_t wm_prmt(uint32_t a, uint32_t b, uint32_t c)
{
#ifdef WM_HOST_EMUL // tests/hostsim/cuda_emul.h: the sweep compiled for the host
	return wm_emul_prmt(a, b, c);
#else
	uint32_t d;
	asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
	return d;
#endif
}
// (a & m) | (b & ~m)
__device__ __forceinline__ uint32_t wm_bitsel(uint32_t m, uint32_t a, uint32_t b) { return (a & m) | (b & ~m); }

// per-job constants of the sweep (registers)
struct wm_v2_k {
	uint32_t KEY_MCH, KEY_MIS, KEY_N;   // score * 8 + TAG_S
	uint32_t TA, TB, TA2, TB2;          // tie-break tags of the four gap states
	uint32_t MCH8;                      // sc_mch * 8
	uint32_t NZ1X, NZ1Y, NZ2X, NZ2Y;    // addends that turn ~z into (-e - z) * 8 + flag tag
	uint32_t C1X, C1Y, C2X, C2Y;        // -(q + e) * 8 (+ tag) / -(q2 + e2) * 8 (+ tag): the clamp operands
	uint32_t DTX;                       // 7 - d for left-aligned gaps
	int16_t *U, *V, *X, *Y, *X2, *Y2, *SK;
	const uint8_t *tg, *qr16;           // target codes; reversed query starting 16 bytes before its first base
};

// One step of a diagonal: NH 32-bit words (2 * NH cells) per lane starting at cell c.  cx/cv/cx2 carry the
// (x, v, x2) values of the cell left of the step in their upper halves.
template <int NH>
__device__ __forceinline__ void wm_v2_step(const wm_v2_k &K, int c, int lane, int st, int en, int st0, int lim, int tlen16, int qoff,
                                           uint8_t *pr, uint32_t &cx, uint32_t &cv, uint32_t &cx2)
{
	const unsigned FULL = 0xffffffffu;
	constexpr int CPL = 2 * NH;
	const int t = c + lane * CPL;
	const bool act = t <= en;                      // cells of the diagonal's blocks
	const bool ref = act || (t < lim && t < tlen16); // score keys: the refresh (:158-172) runs up to 15 cells past en
	uint32_t u_[2], v_[2], x_[2], y_[2], x2_[2], y2_[2], s_[2];
	x_[NH - 1] = v_[NH - 1] = x2_[NH - 1] = 0;
	if (act) {
		if (NH == 2) {
			const uint2 a = *(const uint2*)(K.U + t), b = *(const uint2*)(K.V + t), d = *(const uint2*)(K.X + t), e = *(const uint2*)(K.Y + t);
			const uint2 f = *(const uint2*)(K.X2 + t), g = *(const uint2*)(K.Y2 + t);
			u_[0] = a.x, u_[1] = a.y, v_[0] = b.x, v_[1] = b.y, x_[0] = d.x, x_[1] = d.y, y_[0] = e.x, y_[1] = e.y;
			x2_[0] = f.x, x2_[1] = f.y, y2_[0] = g.x, y2_[1] = g.y;
		} else {
			u_[0] = *(const uint32_t*)(K.U + t), v_[0] = *(const uint32_t*)(K.V + t), x_[0] = *(const uint32_t*)(K.X + t), y_[0] = *(const uint32_t*)(K.Y + t);
			x2_[0] = *(const uint32_t*)(K.X2 + t), y2_[0] = *(const uint32_t*)(K.Y2 + t);
		}
	}
	uint32_t px = __shfl_up_sync(FULL, x_[NH - 1], 1), pv = __shfl_up_sync(FULL, v_[NH - 1], 1), px2 = __shfl_up_sync(FULL, x2_[NH - 1], 1);
	if (lane == 0) px = cx, pv = cv, px2 = cx2;
	if (NH == 2) cx = __shfl_sync(FULL, x_[1], 31), cv = __shfl_sync(FULL, v_[1], 31), cx2 = __shfl_sync(FULL, x2_[1], 31); // a 64-cell step ends its diagonal
	if (ref) {
		// fresh scores for the cells inside [st0, lim); the others keep their stale key.  Codes are 0..4, so a byte of
		// (target ^ query) is non-zero iff adding 0x7f sets its bit 7, and "either is N" is bit 2 of (target | query).
		if (NH == 2) { const uint2 a = *(const uint2*)(K.SK + t); s_[0] = a.x, s_[1] = a.y; } else s_[0] = *(const uint32_t*)(K.SK + t);
		const uint32_t tw = NH == 2 ? *(const uint32_t*)(K.tg + t) : (uint32_t)*(const uint16_t*)(K.tg + t);
		const int o = qoff + t + 16; // index into qr16
		const uint32_t *qw = (const uint32_t*)K.qr16 + (o >> 2);
		const uint32_t qv = __funnelshift_r(qw[0], qw[1], (o & 3) * 8);
		const uint32_t neq = (tw ^ qv) + 0x7f7f7f7fu, nn = (tw | qv) << 5;
		const int rel = t - st0;
		const uint32_t idx0 = __byte_perm((uint32_t)rel, (uint32_t)(rel + 1), 0x5410);
		// cell k of the lane is outside [st0, lim) iff rel + k < 0 or lim - st0 - 1 - (rel + k) < 0: the sign of either half
		uint32_t dlen = __vadd2(wm_rep2(lim - st0), ~idx0); // (lim - st0 - 1) - idx, the "+1" of the negation folded into the constant
		#pragma unroll
		for (int h = 0; h < NH; ++h) {
			const uint32_t ne16 = wm_prmt(neq, 0, h ? 0xbbaa : 0x9988), n16 = wm_prmt(nn, 0, h ? 0xbbaa : 0x9988); // sign replicate
			uint32_t key = K.KEY_MCH ^ ((K.KEY_MCH ^ K.KEY_MIS) & ne16);
			key = key ^ ((key ^ K.KEY_N) & n16);
			const uint32_t idx = h ? __vadd2(idx0, 0x00020002u) : idx0;
			if (h) dlen = __vadd2(dlen, 0xfffefffeu);
			const uint32_t oor = wm_prmt(dlen | idx, 0, 0xbb99); // 0xffff where the cell is out of range
			s_[h] = wm_bitsel(oor, s_[h], key);
		}
		if (NH == 2) *(uint2*)(K.SK + t) = make_uint2(s_[0], s_[1]); else *(uint32_t*)(K.SK + t) = s_[0];
	}
	if (act) {
		uint32_t dd[2], un[2], vn[2], xn[2], yn[2], x2n[2], y2n[2];
		#pragma unroll
		for (int h = 0; h < NH; ++h) {
			const uint32_t uo = u_[h], yo = y_[h], y2o = y2_[h], sk = s_[h];
			const uint32_t xl = h ? __byte_perm(x_[0], x_[1], 0x5432) : __byte_perm(px, x_[0], 0x5432);
			const uint32_t vl = h ? __byte_perm(v_[0], v_[1], 0x5432) : __byte_perm(pv, v_[0], 0x5432);
			const uint32_t x2l = h ? __byte_perm(x2_[0], x2_[1], 0x5432) : __byte_perm(px2, x2_[0], 0x5432);
			const uint32_t a = __vadd2(xl, vl), b = __vadd2(yo, uo), a2 = __vadd2(x2l, vl), b2 = __vadd2(y2o, uo);
			uint32_t m = __viaddmax_s16x2(a, K.TA, sk);
			m = __viaddmax_s16x2(b, K.TB, m);
			m = __viaddmax_s16x2(a2, K.TA2, m);
			m = __viaddmax_s16x2(b2, K.TB2, m);
			uint32_t z = m & 0xfff8fff8u;
			const uint32_t dt = (m & 0x00070007u) ^ K.DTX;
			z = __vmins2(z, K.MCH8);
			const uint32_t notz = ~z;
			// u' = z - v(left), v' = z - u: (~v + 1) + z with the "+1" taken from a shared z + 1
			const uint32_t zp1 = __vadd2(z, 0x00010001u);
			un[h] = __vadd2(zp1, ~vl), vn[h] = __vadd2(zp1, ~uo);
			// x' = max(a - (z - q), 0) - (q + e) = max(a + (-e - z), -(q + e)), likewise the other three (:253-264 / :300-311).
			// Both operands are multiples of 8; the tags in their low bits make bit 0 (x, x2) / bit 1 (y, y2) of the
			// maximum say whether the first operand won, strictly (left-aligned) or not (right-aligned).
			const uint32_t xo = __viaddmax_s16x2(a, __vadd2(notz, K.NZ1X), K.C1X), yo2 = __viaddmax_s16x2(b, __vadd2(notz, K.NZ1Y), K.C1Y);
			const uint32_t x2o = __viaddmax_s16x2(a2, __vadd2(notz, K.NZ2X), K.C2X), y2o2 = __viaddmax_s16x2(b2, __vadd2(notz, K.NZ2Y), K.C2Y);
			const uint32_t f1 = wm_bitsel(0x00010001u, xo, yo2), f2 = wm_bitsel(0x00010001u, x2o, y2o2);
			dd[h] = dt | ((f1 << 3) & 0x00180018u) | ((f2 << 5) & 0x00600060u);
			xn[h] = xo & 0xfff8fff8u, yn[h] = yo2 & 0xfff8fff8u, x2n[h] = x2o & 0xfff8fff8u, y2n[h] = y2o2 & 0xfff8fff8u;
		}
		if (NH == 2) {
			*(uint2*)(K.U + t) = make_uint2(un[0], un[1]); *(uint2*)(K.V + t) = make_uint2(vn[0], vn[1]);
			*(uint2*)(K.X + t) = make_uint2(xn[0], xn[1]); *(uint2*)(K.Y + t) = make_uint2(yn[0], yn[1]);
			*(uint2*)(K.X2 + t) = make_uint2(x2n[0], x2n[1]); *(uint2*)(K.Y2 + t) = make_uint2(y2n[0], y2n[1]);
			*(uint32_t*)(pr + (t - st)) = __byte_perm(dd[0], dd[1], 0x6420);
		} else {
			*(uint32_t*)(K.U + t) = un[0]; *(uint32_t*)(K.V + t) = vn[0]; *(uint32_t*)(K.X + t) = xn[0]; *(uint32_t*)(K.Y + t) = yn[0];
			*(uint32_t*)(K.X2 + t) = x2n[0]; *(uint32_t*)(K.Y2 + t) = y2n[0];
			*(uint16_t*)(pr + (t - st)) = (uint16_t)__byte_perm(dd[0], 0, 0x4420);
		}
	}
}

// bytes of one state slice for jobs of up to tcap (multiple of 16) target and qcap query bases
__host__ __device__ __forceinline__ size_t wm_v2_slice_bytes(int tcap, int qcap)
{
	return ((size_t)7 * 2 * (tcap + 8) + (size_t)4 * tcap + (size_t)(tcap + 16) + (size_t)(qcap + 64) + 15) / 16 * 16;
}

// SM: the slice S8 is the warp's shared-memory slice (capacity WM_V2_T / WM_V2_Q); otherwise it is an L2-resident global
// slice sized for (tcap, qcap) -- the same code, for the few jobs that do not fit shared memory.
template <bool SM>
__device__ void wm_extd2_fill_job_v2(const wm_dp_job &J, const uint8_t *__restrict__ seq, uint8_t *__restrict__ bt,
                                     wm_extz_dev *out, const wm_dp_params &P, uint8_t *S8, int tcap_rt, int qcap_rt, int lane, unsigned long long *cell_ctr)
{
	const int tcap = SM ? WM_V2_T : tcap_rt, qcap = SM ? WM_V2_Q : qcap_rt, ts = tcap + 8;
	const unsigned FULL = 0xffffffffu;
	const uint8_t *query = seq + J.q_off, *target = seq + J.t_off;
	const int qlen = J.qlen, tlen = J.tlen, flag = J.flag;
	int w = J.w;
	wm_extz_dev ez;
	ez.max_q = ez.max_t = ez.mqe_t = ez.mte_q = -1;
	ez.max = 0, ez.score = ez.mqe = ez.mte = WM_NEG_INF;
	ez.n_cigar = 0, ez.zdropped = 0, ez.reach_end = 0, ez.reserved = 0;
	const int q = P.q, e = P.e, q2 = P.q2, e2 = P.e2;
	const bool approx_max = (flag & 0x08) != 0, right = (flag & 0x02) != 0;
	if (w < 0) w = tlen > qlen ? tlen : qlen;
	const int tlen16 = (tlen + 15) / 16 * 16;
	const int n_col16 = wm_ncol16(qlen, tlen, w);
	wm_v2_k K;
	K.U = (int16_t*)S8, K.V = K.U + ts, K.X = K.V + ts, K.Y = K.X + ts, K.X2 = K.Y + ts, K.Y2 = K.X2 + ts, K.SK = K.Y2 + ts;
	int16_t *const U = K.U, *const V = K.V, *const X = K.X, *const Y = K.Y, *const X2 = K.X2, *const Y2 = K.Y2, *const SK = K.SK;
	int32_t *H = (int32_t*)(SK + ts);
	uint8_t *tg = (uint8_t*)(H + tcap);          // target codes, zero padded
	uint8_t *qr = tg + tcap + 16 + 16;             // reversed query with 16 zero bytes in front and 32 behind
	K.tg = tg, K.qr16 = qr - 16;
	{
		const int TAG_S = right ? 0 : 7, TAG_A = right ? 1 : 6, TAG_B = right ? 2 : 5, TAG_A2 = right ? 3 : 4, TAG_B2 = right ? 4 : 3;
		K.KEY_MCH = wm_rep2(P.sc_mch * 8 + TAG_S), K.KEY_MIS = wm_rep2(P.sc_mis * 8 + TAG_S), K.KEY_N = wm_rep2(P.sc_N * 8 + TAG_S);
		K.TA = wm_rep2(TAG_A), K.TB = wm_rep2(TAG_B), K.TA2 = wm_rep2(TAG_A2), K.TB2 = wm_rep2(TAG_B2);
		K.MCH8 = wm_rep2(P.sc_mch * 8);
		K.DTX = right ? 0u : 0x00070007u;
		// ~z + (1 - 8e) = (-e - z) * 8; + 1 (x) or + 2 (y) tags the first operand of the clamp
		K.NZ1X = wm_rep2(-e * 8 + 1 + 1), K.NZ1Y = wm_rep2(-e * 8 + 1 + 2), K.NZ2X = wm_rep2(-e2 * 8 + 1 + 1), K.NZ2Y = wm_rep2(-e2 * 8 + 1 + 2);
		// left-aligned gaps continue only on a strictly positive value: the clamp operand wins ties (tag above the first operand's)
		K.C1X = wm_rep2(-(q + e) * 8 + (right ? 0 : 6)), K.C1Y = wm_rep2(-(q + e) * 8 + (right ? 0 : 5));
		K.C2X = wm_rep2(-(q2 + e2) * 8 + (right ? 0 : 6)), K.C2Y = wm_rep2(-(q2 + e2) * 8 + (right ? 0 : 5));
		const int16_t i1 = (int16_t)(-(q + e) * 8), i2 = (int16_t)(-(q2 + e2) * 8), s0 = (int16_t)TAG_S;
		for (int i = lane; i < tlen16; i += 32) {
			U[i] = V[i] = X[i] = Y[i] = i1; X2[i] = Y2[i] = i2; SK[i] = s0;
			if (!approx_max) H[i] = WM_NEG_INF;
		}
#ifndef WM_HOST_EMUL
		if (SM && ((J.q_off | J.t_off) & 15) == 0) {
			// bulk copies of the 16-byte padded target and query (the pool's padding bytes are zero); the state rows above were
			// being initialised while the copies were in flight
			uint8_t *stage = qr + qcap + 48;                       // landing zone of the forward query
			uint64_t *mbar = (uint64_t*)(stage + qcap);
			const uint32_t tb = (uint32_t)((tlen + 15) & ~15), qb = (uint32_t)((qlen + 15) & ~15);
			if (lane == 0) {
				wm_mbar_init(mbar, 1);
				wm_mbar_expect_tx(mbar, tb + qb);
				wm_bulk_g2s(tg, target, tb, mbar);
				wm_bulk_g2s(stage, query, qb, mbar);
			}
			for (int i = (int)tb + lane; i < tcap + 16; i += 32) tg[i] = 0;
			__syncwarp();
			wm_mbar_wait(mbar, 0);
			for (int i = lane; i < qcap + 48; i += 32) { const int j = i - 16; (qr - 16)[i] = (j >= 0 && j < qlen) ? stage[qlen - 1 - j] : 0; }
		} else
#endif
		{
			for (int i = lane; i < tcap + 16; i += 32) tg[i] = i < tlen ? target[i] : 0;
			for (int i = lane; i < qcap + 48; i += 32) { const int j = i - 16; (qr - 16)[i] = (j >= 0 && j < qlen) ? query[qlen - 1 - j] : 0; }
		}
	}
	__syncwarp();

	const int NQE = -(q + e) * 8, NQE2 = -(q2 + e2) * 8;
	const int bnd_lt = -e * 8, bnd_eq = P.long_diff * 8, bnd_gt = -e2 * 8, long_thres = P.long_thres;
	int32_t H0 = 0, last_H0_t = 0;
	int last_st = -1, last_en = -1;
	unsigned cells_acc = 0;
	const int n_diag = qlen + tlen - 1;
	for (int r = 0; r < n_diag; ++r) {
		const int st0 = wm_band_st(r, qlen, w), en0 = wm_band_en(r, tlen, w);
		if (st0 > en0) { ez.zdropped = 1; break; }
		const int st = st0 & ~15, en = en0 | 15;                    // whole 16-cell blocks (:139)
		const int lim = st0 + (((en0 - st0) >> 4) + 1) * 16;         // end of the score refresh (:158)
		cells_acc += (unsigned)(en - st + 1);
		const int bnd = r == 0 ? NQE : r < long_thres ? bnd_lt : r == long_thres ? bnd_eq : bnd_gt;
		int x1 = NQE, x21 = NQE2, v1 = st > 0 ? NQE : bnd;           // :141-151
		if (st > 0 && st - 1 >= last_st && st - 1 <= last_en) x1 = X[st - 1], x21 = X2[st - 1], v1 = V[st - 1];
		if (en >= r && lane == 0) { Y[r] = (int16_t)NQE, Y2[r] = (int16_t)NQE2; U[r] = (int16_t)bnd; } // :152-155
		__syncwarp();
		{
			uint32_t cx = (uint32_t)x1 << 16, cv = (uint32_t)v1 << 16, cx2 = (uint32_t)x21 << 16;
			uint8_t *pr = bt + J.p_off + (size_t)r * n_col16;
			const int qoff = qlen - 1 - r; // qr index of cell t is qoff + t
			const int last = lim - 1 > en ? lim - 1 : en;
			int c = st;
			for (; last - c >= 64; c += 128) wm_v2_step<2>(K, c, lane, st, en, st0, lim, tlen16, qoff, pr, cx, cv, cx2);
			if (c <= last) wm_v2_step<1>(K, c, lane, st, en, st0, lim, tlen16, qoff, pr, cx, cv, cx2);
		}
		__syncwarp();
		if (!approx_max) {
			int32_t max_H, max_t;
			if (r > 0) {
				const int32_t Hm1 = en0 > 0 ? H[en0 - 1] : 0, Hen = H[en0];
				__syncwarp();
				const int en1 = st0 + (en0 - st0) / 4 * 4;
				long long best = (long long)0x8000000000000000LL;
				for (int t = st0 + lane; t < en0; t += 32) {
					int32_t h = H[t] + (V[t] >> 3);
					H[t] = h;
					uint32_t prio = t < en1 ? 1u + ((uint32_t)((t - st0) & 3) << 24) + (uint32_t)((t - st0) >> 2 << 2)
					                        : (1u << 27) + (uint32_t)(t - st0);
					long long key = ((long long)h << 32) | (long long)(0xffffffffu - prio);
					best = key > best ? key : best;
				}
				const int32_t Hn = en0 > 0 ? Hm1 + (U[en0] >> 3) : Hen + (V[en0] >> 3);
				if (lane == 0) H[en0] = Hn;
				{
					long long key = ((long long)Hn << 32) | (long long)0xffffffffu;
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
				else if (prio < (1u << 27)) max_t = st0 + (int)((prio - 1) & 0xffffffu) + (int)((prio - 1) >> 24);
				else max_t = st0 + (int)(prio - (1u << 27));
				__syncwarp();
			} else {
				max_H = (V[0] >> 3) - P.qe_h, max_t = 0;
				if (lane == 0) H[0] = max_H;
				__syncwarp();
			}
			const int32_t Hen0 = H[en0], Hst0 = H[st0];
			if (en0 == tlen - 1 && Hen0 > ez.mte) ez.mte = Hen0, ez.mte_q = r - en;
			if (r - st0 == qlen - 1 && Hst0 > ez.mqe) ez.mqe = Hst0, ez.mqe_t = st0;
			if (wm_apply_zdrop(ez, max_H, r, max_t, J.zdrop, e2)) break;
			if (r == qlen + tlen - 2 && en0 == tlen - 1) ez.score = H[tlen - 1];
		} else {
			if (r > 0) {
				if (last_H0_t >= st0 && last_H0_t <= en0 && last_H0_t + 1 >= st0 && last_H0_t + 1 <= en0) {
					int32_t d0 = V[last_H0_t] >> 3, d1 = U[last_H0_t + 1] >> 3;
					if (d0 > d1) H0 += d0;
					else H0 += d1, ++last_H0_t;
				} else if (last_H0_t >= st0 && last_H0_t <= en0) {
					H0 += V[last_H0_t] >> 3;
				} else {
					++last_H0_t, H0 += U[last_H0_t] >> 3;
				}
			} else H0 = (V[0] >> 3) - P.qe_h, last_H0_t = 0;
			if ((flag & 0x10) && wm_apply_zdrop(ez, H0, r, last_H0_t, J.zdrop, e2)) break;
			if (r == qlen + tlen - 2 && en0 == tlen - 1) ez.score = H0;
		}
		last_st = st, last_en = en;
	}
	if (lane == 0) { *out = ez; if (cell_ctr) atomicAdd(cell_ctr, (unsigned long long)cells_acc); }
}


// ---- CTA-cooperative sweep for the few big jobs ------------------------------------------------------------------
// One warp per job leaves a launch waiting for its largest job: an end extension of 16 kb x 17 kb at w = 3001 is ~10^8
// cells on one warp.  Here the NW warps of a CTA share one job: the 128-cell steps of a diagonal are dealt round-robin to
// the warps.  A step needs the (x, v, x2) values of the cell left of it on the PREVIOUS diagonal, which the neighbouring
// step is about to overwrite, so every diagonal starts by saving those carry-in values (one per step) in shared memory;
// then: barrier, steps, barrier, H tracking (spread over all threads, reduced through shared memory), barrier.  State
// rows live in the job's global (L2-resident) slice, as for every job that does not fit a warp's shared-memory slice.
#ifndef WM_HOST_EMUL // (CTA-level code: not part of the single-warp CPU emulation of the tests; checked on the device)
#define WM_V2_CTA_WARPS 8
#define WM_V2_CTA_MAXSTEPS 1024 // diagonals of up to 131072 cells
struct wm_v2_cta_sm {
	int16_t cx[WM_V2_CTA_MAXSTEPS], cv[WM_V2_CTA_MAXSTEPS], cx2[WM_V2_CTA_MAXSTEPS];
	long long best[WM_V2_CTA_WARPS];
};

__device__ void wm_extd2_fill_job_v2_cta(const wm_dp_job &J, const uint8_t *__restrict__ seq, uint8_t *__restrict__ bt,
                                         wm_extz_dev *out, const wm_dp_params &P, uint8_t *S8, int tcap, int qcap, wm_v2_cta_sm *SM, unsigned long long *cell_ctr)
{
	constexpr int NW = WM_V2_CTA_WARPS, NT = NW * 32;
	const unsigned FULL = 0xffffffffu;
	const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
	const int ts = tcap + 8;
	const uint8_t *query = seq + J.q_off, *target = seq + J.t_off;
	const int qlen = J.qlen, tlen = J.tlen, flag = J.flag;
	int w = J.w;
	wm_extz_dev ez;
	ez.max_q = ez.max_t = ez.mqe_t = ez.mte_q = -1;
	ez.max = 0, ez.score = ez.mqe = ez.mte = WM_NEG_INF;
	ez.n_cigar = 0, ez.zdropped = 0, ez.reach_end = 0, ez.reserved = 0;
	// a mismatch score above 2(q+e) makes the reference return before the sweep (src/ksw2_extd2_sse.c:92), as the warp
	// kernel does (wm_extd2_fill_job); P is uniform, so the whole CTA returns here
	if (P.early_out) { if (tid == 0) *out = ez; return; }
	const int q = P.q, e = P.e, q2 = P.q2, e2 = P.e2;
	const bool approx_max = (flag & 0x08) != 0, right = (flag & 0x02) != 0;
	if (w < 0) w = tlen > qlen ? tlen : qlen;
	const int tlen16 = (tlen + 15) / 16 * 16;
	const int n_col16 = wm_ncol16(qlen, tlen, w);
	wm_v2_k K;
	K.U = (int16_t*)S8, K.V = K.U + ts, K.X = K.V + ts, K.Y = K.X + ts, K.X2 = K.Y + ts, K.Y2 = K.X2 + ts, K.SK = K.Y2 + ts;
	int16_t *const U = K.U, *const V = K.V, *const X = K.X, *const Y = K.Y, *const X2 = K.X2, *const Y2 = K.Y2, *const SK = K.SK;
	int32_t *H = (int32_t*)(SK + ts);
	uint8_t *tg = (uint8_t*)(H + tcap);
	uint8_t *qr = tg + tcap + 16 + 16;
	K.tg = tg, K.qr16 = qr - 16;
	{
		const int TAG_S = right ? 0 : 7, TAG_A = right ? 1 : 6, TAG_B = right ? 2 : 5, TAG_A2 = right ? 3 : 4, TAG_B2 = right ? 4 : 3;
		K.KEY_MCH = wm_rep2(P.sc_mch * 8 + TAG_S), K.KEY_MIS = wm_rep2(P.sc_mis * 8 + TAG_S), K.KEY_N = wm_rep2(P.sc_N * 8 + TAG_S);
		K.TA = wm_rep2(TAG_A), K.TB = wm_rep2(TAG_B), K.TA2 = wm_rep2(TAG_A2), K.TB2 = wm_rep2(TAG_B2);
		K.MCH8 = wm_rep2(P.sc_mch * 8);
		K.DTX = right ? 0u : 0x00070007u;
		K.NZ1X = wm_rep2(-e * 8 + 1 + 1), K.NZ1Y = wm_rep2(-e * 8 + 1 + 2), K.NZ2X = wm_rep2(-e2 * 8 + 1 + 1), K.NZ2Y = wm_rep2(-e2 * 8 + 1 + 2);
		K.C1X = wm_rep2(-(q + e) * 8 + (right ? 0 : 6)), K.C1Y = wm_rep2(-(q + e) * 8 + (right ? 0 : 5));
		K.C2X = wm_rep2(-(q2 + e2) * 8 + (right ? 0 : 6)), K.C2Y = wm_rep2(-(q2 + e2) * 8 + (right ? 0 : 5));
		const int16_t i1 = (int16_t)(-(q + e) * 8), i2 = (int16_t)(-(q2 + e2) * 8), s0 = (int16_t)TAG_S;
		for (int i = tid; i < tlen16; i += NT) {
			U[i] = V[i] = X[i] = Y[i] = i1; X2[i] = Y2[i] = i2; SK[i] = s0;
			if (!approx_max) H[i] = WM_NEG_INF;
		}
		for (int i = tid; i < tcap + 16; i += NT) tg[i] = i < tlen ? target[i] : 0;
		for (int i = tid; i < qcap + 48; i += NT) { const int j = i - 16; (qr - 16)[i] = (j >= 0 && j < qlen) ? query[qlen - 1 - j] : 0; }
	}
	__syncthreads();

	const int NQE = -(q + e) * 8, NQE2 = -(q2 + e2) * 8;
	const int bnd_lt = -e * 8, bnd_eq = P.long_diff * 8, bnd_gt = -e2 * 8, long_thres = P.long_thres;
	int32_t H0 = 0, last_H0_t = 0;
	int last_st = -1, last_en = -1;
	unsigned long long cells_acc = 0;
	const int n_diag = qlen + tlen - 1;
	for (int r = 0; r < n_diag; ++r) {
		const int st0 = wm_band_st(r, qlen, w), en0 = wm_band_en(r, tlen, w);
		if (st0 > en0) { ez.zdropped = 1; break; }
		const int st = st0 & ~15, en = en0 | 15;
		const int lim = st0 + (((en0 - st0) >> 4) + 1) * 16;
		cells_acc += (unsigned long long)(en - st + 1);
		const int bnd = r == 0 ? NQE : r < long_thres ? bnd_lt : r == long_thres ? bnd_eq : bnd_gt;
		const int last = lim - 1 > en ? lim - 1 : en;
		const int nf = last - st >= 64 ? (last - st - 64) / 128 + 1 : 0; // full 128-cell steps; then at most one 64-cell step
		const int c_tail = st + 128 * nf, n_steps = nf + (c_tail <= last ? 1 : 0);
		// carry-in of every step: the (x, v, x2) of the cell left of it, previous diagonal (src/ksw2_extd2_sse.c:141-151 for step 0)
		for (int sidx = tid; sidx < n_steps; sidx += NT) {
			int x1 = NQE, x21 = NQE2, v1 = st > 0 ? NQE : bnd;
			const int c = st + 128 * sidx;
			if (sidx == 0) { if (st > 0 && st - 1 >= last_st && st - 1 <= last_en) x1 = X[st - 1], x21 = X2[st - 1], v1 = V[st - 1]; }
			else if (c - 1 <= en) x1 = X[c - 1], x21 = X2[c - 1], v1 = V[c - 1];
			else x1 = x21 = v1 = 0;
			SM->cx[sidx] = (int16_t)x1, SM->cx2[sidx] = (int16_t)x21, SM->cv[sidx] = (int16_t)v1;
		}
		const int32_t Hm1 = (!approx_max && r > 0 && en0 > 0) ? H[en0 - 1] : 0, Hen = (!approx_max && r > 0) ? H[en0] : 0; // before anybody adds to H[]
		if (en >= r && tid == 0) { Y[r] = (int16_t)NQE, Y2[r] = (int16_t)NQE2; U[r] = (int16_t)bnd; } // :152-155
		__syncthreads();
		{
			uint8_t *pr = bt + J.p_off + (size_t)r * n_col16;
			const int qoff = qlen - 1 - r;
			for (int sidx = wid; sidx < n_steps; sidx += NW) {
				uint32_t cx = (uint32_t)(uint16_t)SM->cx[sidx] << 16, cv = (uint32_t)(uint16_t)SM->cv[sidx] << 16, cx2 = (uint32_t)(uint16_t)SM->cx2[sidx] << 16;
				const int c = st + 128 * sidx;
				if (sidx < nf) wm_v2_step<2>(K, c, lane, st, en, st0, lim, tlen16, qoff, pr, cx, cv, cx2);
				else wm_v2_step<1>(K, c, lane, st, en, st0, lim, tlen16, qoff, pr, cx, cv, cx2);
			}
		}
		__syncthreads();
		if (!approx_max) {
			int32_t max_H, max_t;
			if (r > 0) {
				const int en1 = st0 + (en0 - st0) / 4 * 4;
				long long best = (long long)0x8000000000000000LL;
				for (int t = st0 + tid; t < en0; t += NT) {
					const int32_t h = H[t] + (V[t] >> 3);
					H[t] = h;
					const uint32_t prio = t < en1 ? 1u + ((uint32_t)((t - st0) & 3) << 24) + (uint32_t)((t - st0) >> 2 << 2)
					                              : (1u << 27) + (uint32_t)(t - st0);
					const long long key = ((long long)h << 32) | (long long)(0xffffffffu - prio);
					best = key > best ? key : best;
				}
				if (tid == 0) {
					const int32_t Hn = en0 > 0 ? Hm1 + (U[en0] >> 3) : Hen + (V[en0] >> 3);
					H[en0] = Hn;
					const long long key = ((long long)Hn << 32) | (long long)0xffffffffu;
					best = key > best ? key : best;
				}
				#pragma unroll
				for (int o = 16; o; o >>= 1) {
					const long long other = __shfl_xor_sync(FULL, best, o);
					best = other > best ? other : best;
				}
				if (lane == 0) SM->best[wid] = best;
				__syncthreads();
				best = SM->best[0];
				#pragma unroll
				for (int k2 = 1; k2 < NW; ++k2) { const long long other = SM->best[k2]; best = other > best ? other : best; }
				max_H = (int32_t)(best >> 32);
				const uint32_t prio = 0xffffffffu - (uint32_t)(best & 0xffffffffLL);
				if (prio == 0) max_t = en0;
				else if (prio < (1u << 27)) max_t = st0 + (int)((prio - 1) & 0xffffffu) + (int)((prio - 1) >> 24);
				else max_t = st0 + (int)(prio - (1u << 27));
			} else {
				max_H = (V[0] >> 3) - P.qe_h, max_t = 0;
				if (tid == 0) H[0] = max_H;
				__syncthreads();
			}
			const int32_t Hen0 = H[en0], Hst0 = H[st0];
			if (en0 == tlen - 1 && Hen0 > ez.mte) ez.mte = Hen0, ez.mte_q = r - en;
			if (r - st0 == qlen - 1 && Hst0 > ez.mqe) ez.mqe = Hst0, ez.mqe_t = st0;
			if (wm_apply_zdrop(ez, max_H, r, max_t, J.zdrop, e2)) break;
			if (r == qlen + tlen - 2 && en0 == tlen - 1) ez.score = H[tlen - 1];
		} else {
			if (r > 0) {
				if (last_H0_t >= st0 && last_H0_t <= en0 && last_H0_t + 1 >= st0 && last_H0_t + 1 <= en0) {
					const int32_t d0 = V[last_H0_t] >> 3, d1 = U[last_H0_t + 1] >> 3;
					if (d0 > d1) H0 += d0;
					else H0 += d1, ++last_H0_t;
				} else if (last_H0_t >= st0 && last_H0_t <= en0) {
					H0 += V[last_H0_t] >> 3;
				} else {
					++last_H0_t, H0 += U[last_H0_t] >> 3;
				}
			} else H0 = (V[0] >> 3) - P.qe_h, last_H0_t = 0;
			if ((flag & 0x10) && wm_apply_zdrop(ez, H0, r, last_H0_t, J.zdrop, e2)) break;
			if (r == qlen + tlen - 2 && en0 == tlen - 1) ez.score = H0;
		}
		last_st = st, last_en = en;
	}
	if (tid == 0) { *out = ez; if (cell_ctr) atomicAdd(cell_ctr, cells_acc); }
}
#endif // WM_HOST_EMUL
