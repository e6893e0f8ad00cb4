// ssq_warp.cuh — warp-cooperative forms of the two Smith-Waterman variants of the second half of `bwa mem` (device only):
//
//   sw_local_warp    upstream ksw_align2 (mate rescue, mem_matesw; SURVEY §8a a11).  The reference evaluates the DP in the order of
//                    its 128-bit striped SSE2 kernel (16 byte lanes, or 8 word lanes when the score can exceed 255) including the
//                    "lazy F" loop and the byte saturation, and the results depend on that order; ssq_dev2.cuh::sw_local_pass
//                    emulates it lane by lane in scalar code.  Here the SSE lanes ARE warp lanes: lane s owns segment s of the
//                    striped query, a row is one lock-step sweep over the segment, the cross-segment carries are shuffles and the
//                    lazy-F exit test is a ballot.  One warp per problem: the latency of one alignment drops by the lane count,
//                    which is what matters — a batch has few rescue alignments (a few 10^4 per 2 M reads), but each is 10^5 cells.
//                    The byte kernel has 16 lanes: the register form that runs by default gives every segment to TWO warp lanes
//                    (sw_local_pass_warp_split), so all 32 lanes work and the values stay those of the 16-lane kernel.
//   sw_global_warp   upstream ksw_global2 + traceback (CIGAR generation, mem_reg2aln / bwa_gen_cigar2; a14).  Plain banded global
//                    affine-gap DP: a cell depends on the row above (H diagonal, E) and on the cell to its left only through F,
//                    and F along a row is a max-plus prefix scan of the gap-open candidates of that row.  Lanes = columns of the
//                    band, rows sequential, F by a 5-step shuffle scan; the traceback byte of every cell is the same function of
//                    the same integers as in the scalar loop, rows of it are written coalesced.
// Both keep everything hot in shared memory (DP rows, query profile / sequences); only the traceback matrix and the list of
// sub-optimal rows live in per-warp global scratch.  Results are bit-identical to the scalar routines (tests against the oracle:
// test_gpu_sw_kernels.py through the kernel-level entries ssq_sw_global_batch / ssq_sw_local_batch, test_gpu_parity.py::
// test_sw_local_striped_order, and whole records in test_gpu_pipe.py; test_sw_kernels_cpu.py checks the scalar routines on the
// same problems).
#pragma once
#include "ssq_dev3.cuh"

#define WFULL 0xffffffffu
#define QMAX_W 256

// --------------------------------------------------------------------------------- local SW ----
struct WarpSwSmem { // per warp
	int16_t H[2][256], E[256], Hmax[256];
	int8_t prof[5][256];
	uint8_t q[256 + 16], q2[256 + 16];
};
struct TgtPac { const DevIndex *ix; i64 rb; __device__ __forceinline__ int operator()(int i) const { return ref_base(*ix, rb + i); } };
struct TgtBuf { const uint8_t *t; __device__ __forceinline__ int operator()(int i) const { return t[i]; } };
// the reference reverses the target prefix [0, te] in place and still passes the full length: rows past te see the unreversed tail
template <class T> struct TgtRev { T t; int te; __device__ __forceinline__ int operator()(int i) const { return i <= te ? t(te - i) : t(i); } };

template <class TGT>
__device__ LocalRes sw_local_pass_warp_smem(const ssq_opts_t &o, bool bytes, int qlen, const uint8_t *q /* shared */, int tlen, TGT tgt, int xtra, WarpSwSmem &W, u64 *b, int b_cap, int lane, unsigned long long *cnt = 0)
{
	const int P = bytes ? 16 : 8, slen = (qlen + P - 1) / P, n = slen * P;
	const int oe_del = o.o_del + o.e_del, oe_ins = o.o_ins + o.e_ins, e_del = o.e_del, e_ins = o.e_ins;
	const int shift = o.b > 1 ? o.b : 1, maxsc = o.a;
	const int minsc = (xtra & SSQ_XSUBO) ? xtra & 0xffff : 0x10000;
	const int endsc = (xtra & SSQ_XSTOP) ? xtra & 0xffff : 0x10000;
	const bool act = lane < P;
	LocalRes r;
	r.score = 0; r.te = r.qe = -1; r.score2 = -1; r.te2 = -1; r.tb = r.qb = -1;
	if (qlen <= 0) return r; // (the reversed pass after a saturated byte-mode score: no cells, nothing found — what the scalar loop yields)
	// query profile in the striped memory order: entry k*P + s = position s*slen + k
	for (int idx = lane; idx < n; idx += 32) {
		const int pos = (idx % P) * slen + idx / P;
		const int qc = pos < qlen ? q[pos] : -1;
#pragma unroll
		for (int c = 0; c < 5; ++c) W.prof[c][idx] = (int8_t)(qc < 0 ? 0 : score_of(o, qc, c));
		W.H[0][idx] = W.H[1][idx] = W.E[idx] = W.Hmax[idx] = 0;
	}
	__syncwarp();
	int gmax = 0, te = -1, n_b = 0, cur = 0, tcache = 0;
	for (int i = 0; i < tlen; ++i) {
		if ((i & 31) == 0) tcache = i + lane < tlen ? tgt(i + lane) : 0;
		const int tb = __shfl_sync(WFULL, tcache, i & 31);
		const int16_t *H0 = W.H[cur]; int16_t *H1 = W.H[cur ^ 1];
		const int8_t *pf = W.prof[tb];
		int f = 0, imax = 0;
		int hd = act ? H0[(slen - 1) * P + lane] : 0;
		hd = __shfl_up_sync(WFULL, hd, 1);
		if (lane == 0) hd = 0;
		if (act) {
			for (int k = 0; k < slen; ++k) { // main pass: every lane sweeps its own segment
				const int idx = k * P + lane;
				const int hn = H0[idx];
				int h = hd + pf[idx], e = W.E[idx], tt;
				if (bytes) { h += shift; if (h > 255) h = 255; h -= shift; if (h < 0) h = 0; }
				else if (h > 32767) h = 32767;
				h = h > e ? h : e;
				h = h > f ? h : f;
				imax = imax > h ? imax : h;
				H1[idx] = (int16_t)h;
				tt = h - oe_del; if (tt < 0) tt = 0;
				e -= e_del; if (e < 0) e = 0;
				W.E[idx] = (int16_t)(e > tt ? e : tt);
				tt = h - oe_ins; if (tt < 0) tt = 0;
				f -= e_ins; if (f < 0) f = 0;
				f = f > tt ? f : tt;
				hd = hn;
			}
		}
		{ // lazy F: carry F across segment boundaries, lock-step over the lanes; stops at the first step where no lane improves
			int fl = f;
			bool done = false;
			for (int round = 0; round < 16 && !done; ++round) {
				fl = __shfl_up_sync(WFULL, fl, 1);
				if (lane == 0) fl = 0;
				for (int k = 0; k < slen; ++k) {
					bool gt = false;
					if (act) {
						const int idx = k * P + lane;
						int h = H1[idx], tt;
						h = h > fl ? h : fl;
						H1[idx] = (int16_t)h;
						tt = h - oe_ins; if (tt < 0) tt = 0;
						fl -= e_ins; if (fl < 0) fl = 0;
						gt = fl > tt;
					}
					if (!__any_sync(WFULL, gt)) { done = true; break; }
				}
			}
		}
		imax = __reduce_max_sync(WFULL, imax);
		if (imax >= minsc && lane == 0) {
			if (n_b == 0 || (i32)b[n_b - 1] + 1 != i) { if (n_b < b_cap) b[n_b++] = (u64)imax << 32 | (u32)i; }
			else if ((int)(b[n_b - 1] >> 32) < imax) b[n_b - 1] = (u64)imax << 32 | (u32)i;
		}
		if (imax > gmax) {
			gmax = imax; te = i;
			if (act) for (int k = 0; k < slen; ++k) W.Hmax[k * P + lane] = H1[k * P + lane];
			if (bytes ? (gmax + shift >= 255 || gmax >= endsc) : gmax >= endsc) break;
		}
		cur ^= 1;
	}
	n_b = __shfl_sync(WFULL, n_b, 0);
	if (cnt && lane == 0) { atomicAdd(cnt + 2, 1ull); atomicAdd(cnt + 3, (unsigned long long)(te < 0 ? tlen : (te + 1 < tlen ? te + 1 : tlen)) * qlen); }
	r.score = bytes ? (gmax + shift < 255 ? gmax : 255) : gmax;
	r.te = te;
	if (!bytes || r.score != 255) {
		int vmax = -1, qe = 0x7fffffff;
		if (act) for (int k = 0; k < slen; ++k) { const int v = W.Hmax[k * P + lane], pos = lane * slen + k; if (v > vmax) { vmax = v; qe = pos; } else if (v == vmax && pos < qe) qe = pos; }
		const int m = __reduce_max_sync(WFULL, vmax);
		r.qe = __reduce_min_sync(WFULL, vmax == m ? qe : 0x7fffffff);
		if (n_b) {
			int s2 = -1, te2 = -1;
			if (lane == 0) {
				const int d = (r.score + maxsc - 1) / maxsc, low = te - d, high = te + d;
				for (int i = 0; i < n_b; ++i) {
					const int e = (i32)b[i];
					if ((e < low || e > high) && (int)(b[i] >> 32) > s2) { s2 = (int)(b[i] >> 32); te2 = e; }
				}
			}
			r.score2 = __shfl_sync(WFULL, s2, 0); r.te2 = __shfl_sync(WFULL, te2, 0);
		}
	}
	__syncwarp();
	return r;
}


// Byte mode with the whole striped state of a lane in registers: a segment has at most 16 cells (queries up to 255 bases over 16
// lanes), so H, E and the query profile of a lane are 16-entry register arrays swept by a fully unrolled loop — no shared-memory
// traffic and no index arithmetic in the inner loop (the profiler attributed 85 % of k_rescue's instructions to that loop).  The
// profile of cell k is one word: the scores against target bases A, C, G, T in its four bytes.  Same arithmetic, same order,
// same results as the shared-memory form above; targets holding N take that form.
template <int SLEN, class TGT>
__device__ __noinline__ LocalRes sw_local_pass_warp_reg(const ssq_opts_t &o, int qlen, const uint8_t *q /* shared */, int tlen, TGT tgt, int xtra, WarpSwSmem &W, u64 *b, int b_cap, int lane, unsigned long long *cnt, bool *has_n)
{
	const int P = 16, slen = SLEN;
	const int oe_del = o.o_del + o.e_del, oe_ins = o.o_ins + o.e_ins, e_del = o.e_del, e_ins = o.e_ins;
	const int shift = o.b > 1 ? o.b : 1, maxsc = o.a;
	const int minsc = (xtra & SSQ_XSUBO) ? xtra & 0xffff : 0x10000;
	const int endsc = (xtra & SSQ_XSTOP) ? xtra & 0xffff : 0x10000;
	const bool act = lane < P;
	LocalRes r;
	r.score = 0; r.te = r.qe = -1; r.score2 = -1; r.te2 = -1; r.tb = r.qb = -1;
	*has_n = false;
	if (qlen <= 0) return r;
	int H[SLEN], E[SLEN], HM[SLEN]; u32 PF[SLEN];
#pragma unroll
	for (int k = 0; k < SLEN; ++k) {
		const int pos = lane * slen + k;
		const int qc = (act && pos < qlen) ? q[pos] : -1;
		u32 w = 0;
#pragma unroll
		for (int c = 0; c < 4; ++c) w |= (u32)(uint8_t)(int8_t)(qc < 0 ? 0 : score_of(o, qc, c)) << (8 * c);
		PF[k] = w; H[k] = E[k] = HM[k] = 0;
	}
	int gmax = 0, te = -1, n_b = 0, tcache = 0, rows = 0;
	for (int i = 0; i < tlen; ++i) {
		if ((i & 31) == 0) tcache = i + lane < tlen ? tgt(i + lane) : 0;
		const int tb = __shfl_sync(WFULL, tcache, i & 31);
		if (tb > 3) { *has_n = true; return r; } // (uniform) the caller redoes the pass with the general form
		++rows;
		const int sh = 8 * tb;
		int f = 0, imax = 0;
		int hd;
		{ // H of the last cell of the lane below
			hd = __shfl_up_sync(WFULL, H[SLEN - 1], 1);
			if (lane == 0) hd = 0;
		}
#pragma unroll
		for (int k = 0; k < SLEN; ++k) {
			{
				const int hn = H[k];
				int h = hd + (int)(int8_t)(PF[k] >> sh), e = E[k], tt;
				h += shift; if (h > 255) h = 255; h -= shift; if (h < 0) h = 0;
				h = h > e ? h : e;
				h = h > f ? h : f;
				imax = imax > h ? imax : h;
				H[k] = h;
				tt = h - oe_del; if (tt < 0) tt = 0;
				e -= e_del; if (e < 0) e = 0;
				E[k] = e > tt ? e : tt;
				tt = h - oe_ins; if (tt < 0) tt = 0;
				f -= e_ins; if (f < 0) f = 0;
				f = f > tt ? f : tt;
				hd = hn;
			}
		}
		if (!act) { imax = 0; f = 0; }
		{ // lazy F
			int fl = f;
			bool done = false;
			for (int round = 0; round < 16 && !done; ++round) {
				fl = __shfl_up_sync(WFULL, fl, 1);
				if (lane == 0) fl = 0;
#pragma unroll
				for (int k = 0; k < SLEN; ++k) {
					if (!done) {
						bool gt = false;
						if (act) {
							int h = H[k], tt;
							h = h > fl ? h : fl;
							H[k] = h;
							tt = h - oe_ins; if (tt < 0) tt = 0;
							fl -= e_ins; if (fl < 0) fl = 0;
							gt = fl > tt;
						}
						if (!__any_sync(WFULL, gt)) done = true;
					}
				}
			}
		}
		imax = __reduce_max_sync(WFULL, imax);
		if (imax >= minsc && lane == 0) {
			if (n_b == 0 || (i32)b[n_b - 1] + 1 != i) { if (n_b < b_cap) b[n_b++] = (u64)imax << 32 | (u32)i; }
			else if ((int)(b[n_b - 1] >> 32) < imax) b[n_b - 1] = (u64)imax << 32 | (u32)i;
		}
		if (imax > gmax) {
			gmax = imax; te = i;
#pragma unroll
			for (int k = 0; k < SLEN; ++k) HM[k] = H[k];
			if (gmax + shift >= 255 || gmax >= endsc) break;
		}
	}
	n_b = __shfl_sync(WFULL, n_b, 0);
	if (cnt && lane == 0) { atomicAdd(cnt + 2, 1ull); atomicAdd(cnt + 3, (unsigned long long)rows * qlen); }
	r.score = gmax + shift < 255 ? gmax : 255;
	r.te = te;
	if (r.score != 255) {
		int vmax = -1, qe = 0x7fffffff;
		if (act) {
#pragma unroll
			for (int k = 0; k < SLEN; ++k) { const int v = HM[k], pos = lane * slen + k; if (v > vmax) { vmax = v; qe = pos; } else if (v == vmax && pos < qe) qe = pos; }
		}
		const int m = __reduce_max_sync(WFULL, vmax);
		r.qe = __reduce_min_sync(WFULL, vmax == m ? qe : 0x7fffffff);
		if (n_b) {
			int s2 = -1, te2 = -1;
			if (lane == 0) {
				const int d = (r.score + maxsc - 1) / maxsc, low = te - d, high = te + d;
				for (int i = 0; i < n_b; ++i) {
					const int e = (i32)b[i];
					if ((e < low || e > high) && (int)(b[i] >> 32) > s2) { s2 = (int)(b[i] >> 32); te2 = e; }
				}
			}
			r.score2 = __shfl_sync(WFULL, s2, 0); r.te2 = __shfl_sync(WFULL, te2, 0);
		}
	}
	return r;
}

// The same pass with all 32 lanes at work: the striped kernel has 16 byte lanes, so the form above leaves half the warp idle.
// Here every segment is shared by two lanes — lane s sweeps cells [0, HA) of segment s, lane 16 + s cells [HA, SLEN) — and the
// values stay those of the 16-lane kernel:
//   * main pass: within a segment only F runs from cell to cell, F' = max(F - e_ins, H - oe_ins, 0), a max-plus recurrence.  The
//     second half starts with F = 0; when the first half's F arrives, F_true(j) = max(F_local(j), F_in decayed by j * e_ins), so
//     its cells are repaired by H = max(H, decayed F_in) (and E, which was derived from H) — a pass that only runs when some
//     segment hands a positive F across its middle;
//   * lazy F: the 16-lane loop tests after every cell whether any lane could still raise an H; here the first halves sweep their
//     cells (exit test over those 16 lanes), then the second halves theirs — the same sequence of cells and tests.
// tests/hostsim/split_emul.cpp runs this algorithm lane by lane on the host against the scalar restatement (sw_local_pass).
__device__ int ssq_rescue_split = 1; // SSQ_RESCUE_SPLIT=0 keeps the 16-lane form (A/B measurements)
template <int SLEN, class TGT>
__device__ __noinline__ LocalRes sw_local_pass_warp_split(const ssq_opts_t &o, int qlen, const uint8_t *q /* shared */, int tlen, TGT tgt, int xtra, WarpSwSmem &W, u64 *b, int b_cap, int lane, unsigned long long *cnt, bool *has_n)
{
	constexpr int HA = (SLEN + 1) / 2, HB = SLEN / 2;
	const int slen = SLEN, s = lane & 15, half = lane >> 4, nloc = half ? HB : HA, base = half ? HA : 0;
	const int oe_del = o.o_del + o.e_del, oe_ins = o.o_ins + o.e_ins, e_del = o.e_del, e_ins = o.e_ins;
	const int shift = o.b > 1 ? o.b : 1, maxsc = o.a;
	const int minsc = (xtra & SSQ_XSUBO) ? xtra & 0xffff : 0x10000;
	const int endsc = (xtra & SSQ_XSTOP) ? xtra & 0xffff : 0x10000;
	LocalRes r;
	r.score = 0; r.te = r.qe = -1; r.score2 = -1; r.te2 = -1; r.tb = r.qb = -1;
	*has_n = false;
	if (qlen <= 0) return r;
	int H[HA], E[HA], HM[HA]; u32 PF[HA];
#pragma unroll
	for (int j = 0; j < HA; ++j) {
		const int pos = s * slen + base + j;
		const int qc = (j < nloc && pos < qlen) ? q[pos] : -1;
		u32 w = 0;
#pragma unroll
		for (int c = 0; c < 4; ++c) w |= (u32)(uint8_t)(int8_t)(qc < 0 ? 0 : score_of(o, qc, c)) << (8 * c);
		PF[j] = w; H[j] = E[j] = HM[j] = 0;
	}
	int gmax = 0, te = -1, n_b = 0, tcache = 0, rows = 0;
	for (int i = 0; i < tlen; ++i) {
		if ((i & 31) == 0) tcache = i + lane < tlen ? tgt(i + lane) : 0;
		const int tb = __shfl_sync(WFULL, tcache, i & 31);
		if (tb > 3) { *has_n = true; return r; } // (uniform) the caller redoes the pass with the general form
		++rows;
		const int sh = 8 * tb;
		int f = 0, imax = 0, hd;
		{ // H (previous row) of the cell before this lane's first one: the end of the segment below / of this segment's first half
			const int last = half ? H[HB - 1] : H[HA - 1];
			hd = __shfl_sync(WFULL, last, half ? s : (15 + s) & 31);
			if (lane == 0) hd = 0;
		}
#pragma unroll
		for (int j = 0; j < HA; ++j) {
			if (j < HB || !half) { // (a second half has one cell less when SLEN is odd)
				const int hn = H[j];
				int h = hd + (int)(int8_t)(PF[j] >> sh), e = E[j], tt;
				h += shift; if (h > 255) h = 255; h -= shift; if (h < 0) h = 0;
				h = h > e ? h : e;
				h = h > f ? h : f;
				imax = imax > h ? imax : h;
				H[j] = h;
				tt = h - oe_del; if (tt < 0) tt = 0;
				e -= e_del; if (e < 0) e = 0;
				E[j] = e > tt ? e : tt;
				tt = h - oe_ins; if (tt < 0) tt = 0;
				f -= e_ins; if (f < 0) f = 0;
				f = f > tt ? f : tt;
				hd = hn;
			}
		}
		{ // the first half's F reaches into the second half
			int g = __shfl_sync(WFULL, f, s);
			if (!half) g = 0;
			if (__any_sync(WFULL, g > 0)) {
#pragma unroll
				for (int j = 0; j < HB; ++j) { // (first halves: g = 0 never exceeds an H)
					if (g > H[j]) { H[j] = g; int tt = g - oe_del; if (tt < 0) tt = 0; if (tt > E[j]) E[j] = tt; if (g > imax) imax = g; }
					g -= e_ins; if (g < 0) g = 0;
				}
				if (g > f) f = g;
			}
		}
		{ // lazy F: first halves, then second halves; the exit test after a cell looks at the 16 lanes that own it
			int fl = f;
			bool done = false;
			for (int round = 0; round < 16 && !done; ++round) {
				const int in = __shfl_sync(WFULL, fl, (15 + s) & 31); // the F the segment below ended its sweep with
				if (!half) fl = s == 0 ? 0 : in;
#pragma unroll
				for (int j = 0; j < HA; ++j) {
					if (!done) {
						bool gt = false;
						if (!half) {
							int h = H[j], tt;
							h = h > fl ? h : fl;
							H[j] = h;
							tt = h - oe_ins; if (tt < 0) tt = 0;
							fl -= e_ins; if (fl < 0) fl = 0;
							gt = fl > tt;
						}
						if (!__any_sync(WFULL, gt)) done = true;
					}
				}
				if (done) break;
				const int fa = __shfl_sync(WFULL, fl, s);
				if (half) fl = fa;
#pragma unroll
				for (int j = 0; j < HB; ++j) {
					if (!done) {
						bool gt = false;
						if (half) {
							int h = H[j], tt;
							h = h > fl ? h : fl;
							H[j] = h;
							tt = h - oe_ins; if (tt < 0) tt = 0;
							fl -= e_ins; if (fl < 0) fl = 0;
							gt = fl > tt;
						}
						if (!__any_sync(WFULL, gt)) done = true;
					}
				}
			}
		}
		imax = __reduce_max_sync(WFULL, imax);
		if (imax >= minsc && lane == 0) {
			if (n_b == 0 || (i32)b[n_b - 1] + 1 != i) { if (n_b < b_cap) b[n_b++] = (u64)imax << 32 | (u32)i; }
			else if ((int)(b[n_b - 1] >> 32) < imax) b[n_b - 1] = (u64)imax << 32 | (u32)i;
		}
		if (imax > gmax) {
			gmax = imax; te = i;
#pragma unroll
			for (int j = 0; j < HA; ++j) HM[j] = H[j];
			if (gmax + shift >= 255 || gmax >= endsc) break;
		}
	}
	n_b = __shfl_sync(WFULL, n_b, 0);
	if (cnt && lane == 0) { atomicAdd(cnt + 2, 1ull); atomicAdd(cnt + 3, (unsigned long long)rows * qlen); }
	r.score = gmax + shift < 255 ? gmax : 255;
	r.te = te;
	if (r.score != 255) {
		int vmax = -1, qe = 0x7fffffff;
#pragma unroll
		for (int j = 0; j < HA; ++j) if (j < nloc) { const int v = HM[j], pos = s * slen + base + j; if (v > vmax) { vmax = v; qe = pos; } else if (v == vmax && pos < qe) qe = pos; }
		const int m = __reduce_max_sync(WFULL, vmax);
		r.qe = __reduce_min_sync(WFULL, vmax == m ? qe : 0x7fffffff);
		if (n_b) {
			int s2 = -1, te2 = -1;
			if (lane == 0) {
				const int d = (r.score + maxsc - 1) / maxsc, low = te - d, high = te + d;
				for (int i = 0; i < n_b; ++i) {
					const int e = (i32)b[i];
					if ((e < low || e > high) && (int)(b[i] >> 32) > s2) { s2 = (int)(b[i] >> 32); te2 = e; }
				}
			}
			r.score2 = __shfl_sync(WFULL, s2, 0); r.te2 = __shfl_sync(WFULL, te2, 0);
		}
	}
	return r;
}

template <class TGT>
__device__ LocalRes sw_local_pass_warp(const ssq_opts_t &o, bool bytes, int qlen, const uint8_t *q /* shared */, int tlen, TGT tgt, int xtra, WarpSwSmem &W, u64 *b, int b_cap, int lane, unsigned long long *cnt = 0)
{
	if (bytes && qlen > 0 && qlen <= 256) {
		bool has_n = false;
		LocalRes r;
		if (ssq_rescue_split && qlen > 16) switch ((qlen + 15) / 16) {
#define SSQ_SLEN_CASE(n_) case n_: r = sw_local_pass_warp_split<n_>(o, qlen, q, tlen, tgt, xtra, W, b, b_cap, lane, cnt, &has_n); break;
		SSQ_SLEN_CASE(2) SSQ_SLEN_CASE(3) SSQ_SLEN_CASE(4) SSQ_SLEN_CASE(5) SSQ_SLEN_CASE(6) SSQ_SLEN_CASE(7) SSQ_SLEN_CASE(8)
		SSQ_SLEN_CASE(9) SSQ_SLEN_CASE(10) SSQ_SLEN_CASE(11) SSQ_SLEN_CASE(12) SSQ_SLEN_CASE(13) SSQ_SLEN_CASE(14) SSQ_SLEN_CASE(15) SSQ_SLEN_CASE(16)
#undef SSQ_SLEN_CASE
		default: has_n = true;
		}
		else switch ((qlen + 15) / 16) {
#define SSQ_SLEN_CASE(n_) case n_: r = sw_local_pass_warp_reg<n_>(o, qlen, q, tlen, tgt, xtra, W, b, b_cap, lane, cnt, &has_n); break;
		SSQ_SLEN_CASE(1) SSQ_SLEN_CASE(2) SSQ_SLEN_CASE(3) SSQ_SLEN_CASE(4) SSQ_SLEN_CASE(5) SSQ_SLEN_CASE(6) SSQ_SLEN_CASE(7) SSQ_SLEN_CASE(8)
		SSQ_SLEN_CASE(9) SSQ_SLEN_CASE(10) SSQ_SLEN_CASE(11) SSQ_SLEN_CASE(12) SSQ_SLEN_CASE(13) SSQ_SLEN_CASE(14) SSQ_SLEN_CASE(15) SSQ_SLEN_CASE(16)
#undef SSQ_SLEN_CASE
		default: has_n = true;
		}
		if (!has_n) return r;
	}
	return sw_local_pass_warp_smem(o, bytes, qlen, q, tlen, tgt, xtra, W, b, b_cap, lane, cnt);
}

// forward pass for score/end, then a pass over the reversed prefixes for the start.  q: the query in shared memory (W.q)
template <class TGT>
__device__ LocalRes sw_local_warp(const ssq_opts_t &o, int qlen, int tlen, TGT tgt, int xtra, WarpSwSmem &W, u64 *b, int b_cap, int lane, unsigned long long *cnt = 0)
{
	const bool bytes = (xtra & SSQ_XBYTE) != 0;
	LocalRes r = sw_local_pass_warp(o, bytes, qlen, W.q, tlen, tgt, xtra, W, b, b_cap, lane, cnt);
	if ((xtra & SSQ_XSTART) == 0 || ((xtra & SSQ_XSUBO) && r.score < (xtra & 0xffff))) return r;
	for (int i = lane; i <= r.qe; i += 32) W.q2[i] = W.q[r.qe - i];
	__syncwarp();
	TgtRev<TGT> rt; rt.t = tgt; rt.te = r.te;
	const LocalRes rr = sw_local_pass_warp(o, bytes, r.qe + 1, W.q2, tlen, rt, SSQ_XSTOP | r.score, W, b, b_cap, lane, cnt);
	if (r.score == rr.score) { r.tb = r.te - rr.te; r.qb = r.qe - rr.qe; }
	return r;
}

// one mem_matesw() by a warp: control flow is uniform (every lane evaluates the same scalars), lane 0 owns the writes to the
// mate's region list.  Same contract as ssq_dev2.cuh::mate_rescue
__device__ int mate_rescue_warp(const DevIndex &ix, const ssq_opts_t &o, const PeStat *pes, const AlnReg &a, int l_ms, const uint8_t *ms, AlnReg *ma, int *n_ma, int ma_cap,
                                WarpSwSmem &W, u64 *bl, int b_cap, int lane, unsigned long long *wcnt = 0, i32 *idx = 0, RCache *rc = 0, u32 key = 0)
{
	const i64 l_pac = ix.l_pac;
	int i, r, skip[4], n = 0, cnt = *n_ma; // cnt: the list length, kept uniform across the lanes (lane 0 changes the list, then broadcasts)
	{ // the skip test looks at every hit of the mate: lanes take hits round-robin, one vote per orientation
		int mine = 0;
		for (i = lane; i < cnt; i += 32) {
			i64 dist;
			r = infer_dir(l_pac, a.rb, ma[i].rb, &dist);
			if (dist >= pes[r].low && dist <= pes[r].high) mine |= 1 << r;
		}
		mine = __reduce_or_sync(WFULL, mine);
		for (r = 0; r < 4; ++r) skip[r] = (pes[r].failed || (mine >> r & 1)) ? 1 : 0;
	}
	if (skip[0] + skip[1] + skip[2] + skip[3] == 4) return 0;
	AlnScratch noA; noA.qbuf = noA.rbuf = 0; noA.rcap = 0; noA.g.h = noA.g.e = 0; noA.g.z = 0; noA.g.zcap = 0;
	for (r = 0; r < 4; ++r) {
		if (skip[r]) continue;
		const int is_rev = (r >> 1 != (r & 1));
		i64 rb, re;
		if (rescue_window(ix, o, pes, a, l_ms, r, &rb, &re)) {
			if (re - rb > b_cap) { *n_ma = cnt; return -1; }
			const int tlen = (int)(re - rb);
			const LocalRes *ahead = rc ? rcache_find(*rc, key | (u32)r, rb, tlen) : 0; // (uniform: every lane walks its own copy of the cursor)
			LocalRes aln;
			if (ahead) aln = *ahead;
			else { // not computed ahead: here and now
				if (rc && rc->miss && lane == 0) atomicAdd(rc->miss, 1u);
				__syncwarp();
				for (i = lane; i < l_ms; i += 32) W.q[is_rev ? l_ms - 1 - i : i] = is_rev ? (ms[i] < 4 ? 3 - ms[i] : 4) : ms[i];
				__syncwarp();
				TgtPac tg; tg.ix = &ix; tg.rb = rb;
				aln = sw_local_warp(o, l_ms, tlen, tg, rescue_xtra(o, l_ms), W, bl, b_cap, lane, wcnt);
			}
			if (aln.score >= o.min_seed_len && aln.qb >= 0) {
				if (lane == 0 && cnt < ma_cap) {
					AlnReg b;
					b.rid = a.rid;
					b.qb = is_rev ? l_ms - (aln.qe + 1) : aln.qb;
					b.qe = is_rev ? l_ms - aln.qb : aln.qe + 1;
					b.rb = is_rev ? (l_pac << 1) - (rb + aln.te + 1) : rb + aln.tb;
					b.re = is_rev ? (l_pac << 1) - (rb + aln.tb) : rb + aln.te + 1;
					b.score = aln.score; b.truesc = 0; b.sub = 0; b.csub = aln.score2; b.sub_n = 0; b.w = 0;
					b.secondary = -1; b.secondary_all = 0; b.seedlen0 = 0; b.n_comp = 0; b.frac_rep = 0.f; b.hash = 0;
					b.seedcov = (int)((b.re - b.rb < b.qe - b.qb ? b.re - b.rb : b.qe - b.qb) >> 1);
					for (i = 0; i < cnt; ++i) if (ma[i].score < b.score) break;
					const int at = i;
					for (i = cnt; i > at; --i) ma[i] = ma[i - 1];
					ma[at] = b;
				}
				if (cnt < ma_cap) ++cnt;
			}
			++n;
		}
		if (n) {
			int c2 = cnt;
			if (lane == 0) c2 = sort_dedup_patch(ix, o, 0, cnt, ma, noA, idx);
			cnt = __shfl_sync(WFULL, c2, 0);
			__syncwarp();
		}
	}
	*n_ma = cnt;
	return n;
}
// one rescue alignment computed ahead of the replay (RTask, ssq_dev2.cuh): the mate's sequence in the orientation's strand against
// the task's window
__device__ LocalRes rescue_task_warp(const PipeView &V, const RTask &t, int p, WarpSwSmem &W, u64 *bl, int b_cap, int lane)
{
	const int i = (int)(t.key >> 16), r = (int)(t.key & 3), is_rev = (r >> 1 != (r & 1)), l_ms = t.l_ms;
	const uint8_t *ms = V.tc.seq + V.tc.read_off[2 * p + !i];
	__syncwarp();
	for (int x = lane; x < l_ms; x += 32) W.q[is_rev ? l_ms - 1 - x : x] = is_rev ? (ms[x] < 4 ? 3 - ms[x] : 4) : ms[x];
	__syncwarp();
	TgtPac tg; tg.ix = &V.ix; tg.rb = t.rb;
	return sw_local_warp(V.opt, l_ms, t.tlen, tg, rescue_xtra(V.opt, l_ms), W, bl, b_cap, lane, V.cnt);
}
// -------------------------------------------------------------------------------- global DP ----
#define WG_RCAP 2048
struct WarpGlSmem { i32 H[2][QMAX_W + 16], E[QMAX_W + 16]; uint8_t q[QMAX_W], r[WG_RCAP]; };

// banded global alignment of W.q[0..qlen) vs W.r[0..tlen), traceback into cig (lane 0 writes).  z: per-warp global scratch of
// zcap bytes (null / too small: score only when cig == null, else *n_cig = -1); *n_cig = -1 as well when the operations do not fit
// in cig_cap.  Same contract and results as sw_global()
__device__ int sw_global_warp(const ssq_opts_t &o, int qlen, int tlen, int w, WarpGlSmem &W, uint8_t *z, long zcap, u32 *cig, int cig_cap, int *n_cig, int lane, unsigned long long *cells = 0)
{
	const int o_del = o.o_del, e_del = o.e_del, o_ins = o.o_ins, e_ins = o.e_ins, oe_del = o_del + e_del, oe_ins = o_ins + e_ins;
	const int n_col = qlen < 2 * w + 1 ? qlen : 2 * w + 1;
	const bool tb = cig != 0 && n_cig != 0;
	if (cells && lane == 0) atomicAdd(cells, (unsigned long long)n_col * tlen);
	if (n_cig) *n_cig = 0;
	if (tb && (long)n_col * tlen > zcap) { *n_cig = -1; return 0; }
	for (int j = lane; j <= qlen; j += 32) {
		W.H[0][j] = j == 0 ? 0 : j <= w ? -(o_ins + e_ins * j) : SSQ_MINUS_INF;
		W.E[j] = SSQ_MINUS_INF;
	}
	__syncwarp();
	int cur = 0;
	for (int i = 0; i < tlen; ++i) {
		const i32 *Hp = W.H[cur]; i32 *Hc = W.H[cur ^ 1];
		const int tbase = W.r[i];
		const int beg = i > w ? i - w : 0, end = i + w + 1 < qlen ? i + w + 1 : qlen;
		i32 carry = SSQ_MINUS_INF; // F entering the chunk's first column
		if (lane == 0) Hc[beg] = beg == 0 ? -(o_del + e_del * (i + 1)) : SSQ_MINUS_INF;
		for (int c0 = beg; c0 < end; c0 += 32) {
			const int j = c0 + lane;
			const bool act = j < end;
			i32 m = SSQ_MINUS_INF, e = SSQ_MINUS_INF;
			if (act) { m = Hp[j] + score_of(o, W.q[j], tbase); e = W.E[j]; }
			// F entering column j: f(c0) = carry, f(j+1) = max(f(j) - e_ins, m(j) - oe_ins)  ==  a max-plus prefix scan
			i32 s = act ? m - oe_ins : SSQ_MINUS_INF; // candidate opened at column j, seen by column j + 1
#pragma unroll
			for (int d = 1; d < 32; d <<= 1) {
				const i32 up = __shfl_up_sync(WFULL, s, d);
				if (lane >= d) { const i32 v = up - e_ins * d; s = s > v ? s : v; }
			}
			i32 f = __shfl_up_sync(WFULL, s, 1); // best candidate opened at a column < j of this chunk, decayed to column j
			const i32 fc = carry - e_ins * lane;
			f = lane == 0 ? fc : (f > fc ? f : fc);
			if (act) {
				uint8_t d = m >= e ? 0 : 1;
				i32 h = m >= e ? m : e, tt;
				d = h >= f ? d : 2;
				h = h >= f ? h : f;
				tt = m - oe_del;
				e -= e_del;
				d |= e > tt ? 1 << 2 : 0;
				e = e > tt ? e : tt;
				W.E[j] = e;
				tt = m - oe_ins;
				const i32 fx = f - e_ins;
				d |= fx > tt ? 2 << 4 : 0;
				Hc[j + 1] = h;
				if (tb) z[(size_t)i * n_col + (j - beg)] = d;
			}
			// F entering the next chunk = the scan's value one column past lane 31
			const i32 fx31 = (f - e_ins) > (m - oe_ins) ? (f - e_ins) : (m - oe_ins);
			carry = __shfl_sync(WFULL, fx31, 31);
		}
		if (lane == 0) W.E[end] = SSQ_MINUS_INF;
		__syncwarp();
		cur ^= 1;
	}
	const int score = W.H[cur][qlen];
	if (tb) { // traceback by lane 0 (the matrix rows were written by all lanes: make them visible first)
		__syncwarp();
		int n = 0;
		if (lane == 0) {
			int which = 0, i = tlen - 1, k = (i + w + 1 < qlen ? i + w + 1 : qlen) - 1;
			bool full = false;
#define PUSH_OP(op_, len_) do { if (n == 0 || (int)(cig[n - 1] & 0xf) != (op_)) { if (n < cig_cap) cig[n++] = (u32)(len_) << 4 | (op_); else full = true; } else cig[n - 1] += (u32)(len_) << 4; } while (0)
			while (i >= 0 && k >= 0) {
				which = z[(size_t)i * n_col + (k - (i > w ? i - w : 0))] >> (which << 1) & 3;
				if (which == 0) { PUSH_OP(0, 1); --i; --k; }
				else if (which == 1) { PUSH_OP(2, 1); --i; }
				else { PUSH_OP(1, 1); --k; }
			}
			if (i >= 0) PUSH_OP(2, i + 1);
			if (k >= 0) PUSH_OP(1, k + 1);
#undef PUSH_OP
			for (i = 0; i < n >> 1; ++i) { const u32 x = cig[i]; cig[i] = cig[n - 1 - i]; cig[n - 1 - i] = x; }
			if (full) n = -1; // more operations than cig_cap: reported, never cut short (gen_cigar_warp returns false)
		}
		n = __shfl_sync(WFULL, n, 0);
		*n_cig = n;
	}
	return score;
}

// bwa_gen_cigar2 by a warp; same contract as ssq_dev2.cuh::gen_cigar.  Text/CIGAR outputs are written by lane 0
__device__ bool gen_cigar_warp(const DevIndex &ix, const ssq_opts_t &o, int w_, int l_query, const uint8_t *query, i64 rb, i64 re, WarpGlSmem &W, uint8_t *z, long zcap,
                               int *score, u32 *cig, int cig_cap, int *n_cig, int *NM, TextOut *md, int lane)
{
	const i64 l_pac = ix.l_pac;
	int i;
	if (n_cig) *n_cig = 0;
	if (NM) *NM = -1;
	if (l_query <= 0 || rb >= re || (rb < l_pac && re > l_pac)) return false;
	const int rlen = (int)(re - rb);
	if (rlen > WG_RCAP) { if (n_cig) *n_cig = -1; return false; }
	const bool rev = rb >= l_pac;
	__syncwarp();
	for (i = lane; i < rlen; i += 32) W.r[rev ? rlen - 1 - i : i] = (uint8_t)ref_base(ix, rb + i);
	for (i = lane; i < l_query; i += 32) W.q[rev ? l_query - 1 - i : i] = query[i];
	__syncwarp();
	if (l_query == rlen && w_ == 0) {
		int sc = 0;
		for (i = lane; i < l_query; i += 32) sc += score_of(o, W.q[i], W.r[i]);
		*score = __reduce_add_sync(WFULL, sc);
		if (cig && n_cig) { if (lane == 0) cig[0] = (u32)l_query << 4; *n_cig = 1; }
	} else {
		int w, max_gap, max_ins, max_del, min_w;
		max_ins = (int)((double)(((l_query + 1) >> 1) * o.a - o.o_ins) / o.e_ins + 1.);
		max_del = (int)((double)(((l_query + 1) >> 1) * o.a - o.o_del) / o.e_del + 1.);
		max_gap = max_ins > max_del ? max_ins : max_del;
		max_gap = max_gap > 1 ? max_gap : 1;
		w = (max_gap + iabs(rlen - l_query) + 1) >> 1;
		w = w < w_ ? w : w_;
		min_w = iabs(rlen - l_query) + 3;
		w = w > min_w ? w : min_w;
		*score = sw_global_warp(o, l_query, rlen, w, W, z, zcap, cig, cig_cap, n_cig, lane);
		if (cig && n_cig && *n_cig < 0) return false;
	}
	if (NM && cig && n_cig) {
		int nm = 0;
		if (lane == 0) {
			int k, x, y, u, n_mm = 0, n_gap = 0;
			const char *int2base = rb < l_pac ? "ACGTN" : "TGCAN";
			for (k = 0, x = y = u = 0; k < *n_cig; ++k) {
				const int op = cig[k] & 0xf, len = (int)(cig[k] >> 4);
				if (op == 0) {
					for (i = 0; i < len; ++i) {
						if (W.q[x + i] != W.r[y + i]) { if (md) { tputn(*md, u); tput(*md, int2base[W.r[y + i]]); } ++n_mm; u = 0; }
						else ++u;
					}
					x += len; y += len;
				} else if (op == 2) {
					if (k > 0 && k < *n_cig - 1) {
						if (md) { tputn(*md, u); tput(*md, '^'); for (i = 0; i < len; ++i) tput(*md, int2base[W.r[y + i]]); }
						u = 0; n_gap += len;
					}
					y += len;
				} else if (op == 1) { x += len; n_gap += len; }
			}
			if (md) tputn(*md, u);
			nm = n_mm + n_gap;
		}
		*NM = __shfl_sync(WFULL, nm, 0);
		if (md) md->n = __shfl_sync(WFULL, md->n, 0);
	}
	return true;
}

// mem_reg2aln by a warp; lane 0 writes a / cig / md.  Same contract as ssq_dev2.cuh::reg2aln
__device__ void reg2aln_warp(const DevIndex &ix, const ssq_opts_t &o, int l_query, const uint8_t *query, const AlnReg &ar, WarpGlSmem &W, uint8_t *z, long zcap,
                             AlnOut &a, u32 *cig, int cig_cap, char *md, int md_cap, int lane)
{
	int i, w2, tmp, NM = -1, score = 0, is_rev, last_sc = -(1 << 30), n_cigar = 0;
	const int qb = ar.qb, qe = ar.qe;
	const i64 rb = ar.rb, re = ar.re;
	TextOut t; t.s = md; t.n = 0; t.cap = md_cap;
	a.flag = ar.secondary >= 0 ? 0x100 : 0;
	tmp = infer_bw(qe - qb, (int)(re - rb), ar.truesc, o.a, o.o_del, o.e_del);
	w2 = infer_bw(qe - qb, (int)(re - rb), ar.truesc, o.a, o.o_ins, o.e_ins);
	w2 = w2 > tmp ? w2 : tmp;
	if (w2 > o.w) w2 = w2 < ar.w ? w2 : ar.w;
	i = 0;
	do {
		w2 = w2 < o.w << 2 ? w2 : o.w << 2;
		t.n = 0;
		gen_cigar_warp(ix, o, w2, qe - qb, query + qb, rb, re, W, z, zcap, &score, cig, cig_cap - 2, &n_cigar, &NM, &t, lane);
		if (score == last_sc || w2 == o.w << 2) break;
		last_sc = score;
		w2 <<= 1;
	} while (++i < 3 && score < ar.truesc - o.a);
	a.NM = NM;
	i64 pos = depos(ix, rb < ix.l_pac ? rb : re - 1, is_rev);
	a.is_rev = is_rev;
	__syncwarp();
	if (n_cigar > 0) {
		const u32 c0 = cig[0], cl = cig[n_cigar - 1];
		__syncwarp();
		if ((c0 & 0xf) == 2) { pos += c0 >> 4; --n_cigar; if (lane == 0) for (i = 0; i < n_cigar; ++i) cig[i] = cig[i + 1]; }
		else if ((cl & 0xf) == 2) --n_cigar;
	}
	if (n_cigar >= 0 && (qb != 0 || qe != l_query)) {
		const int clip5 = is_rev ? l_query - qe : qb, clip3 = is_rev ? qb : l_query - qe;
		if (clip5) { if (lane == 0) { for (i = n_cigar; i > 0; --i) cig[i] = cig[i - 1]; cig[0] = (u32)clip5 << 4 | 3; } ++n_cigar; }
		if (clip3) { if (lane == 0) cig[n_cigar] = (u32)clip3 << 4 | 3; ++n_cigar; }
	}
	__syncwarp();
	a.n_cigar = n_cigar;
	if (n_cigar < 0) { a.rid = ar.rid; a.pos = 0; a.score = ar.score; a.sub = 0; a.md_len = 0; a.mapq_unused = 0; a.pad = 0; return; }
	a.rid = pos2rid(ix, pos);
	a.pos = pos - ix.ann_off[a.rid];
	a.score = ar.score; a.sub = ar.sub > ar.csub ? ar.sub : ar.csub;
	a.md_len = t.n < md_cap ? t.n : md_cap;
	a.mapq_unused = 0; a.pad = 0;
}

// mem_sam_pe's rescue block for one pair by a warp (the warp form of ssq_dev3.cuh::body_rescue).  bbuf: per-warp global scratch for
// 2 x 64 regions, bl: per-warp list of b_cap sub-optimal rows
__device__ void body_rescue_warp(const PipeView &V, int p, AlnReg *bbuf, WarpSwSmem &W, u64 *bl, int b_cap, int lane, RCache *rc = 0)
{
	AlnReg *b[2] = {bbuf, bbuf + 64};
	int nb[2] = {0, 0}, na[2];
	AlnReg *a[2];
	for (int i = 0; i < 2; ++i) { // snapshot of the near-best hits of both ends: lanes pick the qualifying hits by ballot and copy one record each
		a[i] = V.areg + V.areg_off[2 * p + i]; na[i] = (int)V.n_areg[2 * p + i];
		const int thr = na[i] ? a[i][0].score - V.opt.pen_unpaired : 0;
		for (int j0 = 0; j0 < na[i] && nb[i] < 64; j0 += 32) {
			const int j = j0 + lane;
			const bool q = j < na[i] && a[i][j].score >= thr;
			const unsigned m = __ballot_sync(WFULL, q);
			const int at = nb[i] + __popc(m & ((1u << lane) - 1));
			if (q && at < 64) b[i][at] = a[i][j];
			nb[i] += __popc(m); if (nb[i] > 64) nb[i] = 64;
		}
	}
	__syncwarp();
	for (int i = 0; i < 2; ++i) {
		const int cap = (int)(V.areg_off[2 * p + !i + 1] - V.areg_off[2 * p + !i]);
		for (int j = 0; j < nb[i] && j < V.opt.max_matesw; ++j) {
			const int before = na[!i];
			if (mate_rescue_warp(V.ix, V.opt, V.pes, b[i][j], (int)(V.tc.read_off[2 * p + !i + 1] - V.tc.read_off[2 * p + !i]), V.tc.seq + V.tc.read_off[2 * p + !i], a[!i], &na[!i], cap, W, bl, b_cap, lane, V.cnt, V.xcnt + V.areg_off[2 * p + !i], rc, (u32)(i << 16 | j << 2)) < 0 && lane == 0) PIPE_ERR(V, 8);
			if (na[!i] >= cap && before < cap && lane == 0) PIPE_ERR(V, 1);
		}
	}
	if (lane == 0) { V.n_areg[2 * p] = (u32)na[0]; V.n_areg[2 * p + 1] = (u32)na[1]; }
}
