// ssq_dev2.cuh — second half of the single-end / paired-end core as SSQ_HD routines:
//   sw_global      banded global affine-gap DP + traceback            (upstream ksw_global2; SURVEY §8a a8/a14)
//   gen_cigar      CIGAR + NM + MD of a region                       (upstream bwa_gen_cigar2)
//   sort_dedup_patch                                                 (upstream mem_sort_dedup_patch / mem_patch_reg; a8)
//   sw_local       local SW in the evaluation order of the 16/8-lane striped kernel (upstream ksw_align2; a11)
//   mate_rescue    one mem_matesw() call                                                          (a11)
//   reg2aln        region -> position / CIGAR / NM / MD with the band-doubling loop              (upstream mem_reg2aln; a14)
// Call site in the reference: inside `$BWA mem`, speedseq/bin/speedseq:438.  Used by the kernels of
// ssq_kernels2.cu (one thread per read / pair / alignment) and, for CPU-side checking only, by tests/hostsim.
#pragma once
#include "ssq_dev.cuh"

struct AlnReg { // full alignment-region record (upstream mem_alnreg_t)
	i64 rb, re;
	i32 qb, qe, rid, score, truesc, sub, csub, sub_n, w, seedcov, secondary, secondary_all, seedlen0, n_comp;
	float frac_rep;
	u64 hash;
};

SSQ_HD void reg_from_cand(const RegCand &c, AlnReg &a)
{
	a.rb = c.rb; a.re = c.re; a.qb = c.qb; a.qe = c.qe; a.rid = c.rid; a.score = c.score; a.truesc = c.truesc;
	a.sub = 0; a.csub = 0; a.sub_n = 0; a.w = c.w; a.seedcov = c.seedcov; a.secondary = 0; a.secondary_all = 0;
	a.seedlen0 = c.seedlen0; a.n_comp = 0; a.frac_rep = c.frac_rep; a.hash = 0;
}

SSQ_HD int score_of(const ssq_opts_t &o, int a, int b) { return (a > 3 || b > 3) ? -1 : (a == b ? o.a : -o.b); }

// ------------------------------------------------------------------------------ global DP ----
#define SSQ_MINUS_INF (-0x40000000)
struct GlobalScratch { i32 *h, *e; uint8_t *z; long zcap; }; // h/e: qlen+1 each; z: n_col*tlen (may be null when no CIGAR is wanted)

// query q[0..qlen), target t[0..tlen) (arrays of codes). cigar (op | len<<4) written reversed-then-fixed into cig[0..*n_cig);
// *n_cig = -1 when the operations do not fit in cig_cap (reported, never cut short)
SSQ_HD int sw_global(const ssq_opts_t &o, int qlen, const uint8_t *q, int tlen, const uint8_t *t, int w, const GlobalScratch &S, u32 *cig, int cig_cap, int *n_cig)
{
	const int o_del = o.o_del, e_del = o.e_del, o_ins = o.o_ins, e_ins = o.e_ins, oe_del = o_del + e_del, oe_ins = o_ins + e_ins;
	const int n_col = qlen < 2 * w + 1 ? qlen : 2 * w + 1;
	int i, j, k;
	if (n_cig) *n_cig = 0;
	S.h[0] = 0; S.e[0] = SSQ_MINUS_INF;
	for (j = 1; j <= qlen && j <= w; ++j) { S.h[j] = -(o_ins + e_ins * j); S.e[j] = SSQ_MINUS_INF; }
	for (; j <= qlen; ++j) S.h[j] = S.e[j] = SSQ_MINUS_INF;
	for (i = 0; i < tlen; ++i) {
		i32 f = SSQ_MINUS_INF, h1, beg, end, tt;
		const int tb = t[i];
		beg = i > w ? i - w : 0;
		end = i + w + 1 < qlen ? i + w + 1 : qlen;
		h1 = beg == 0 ? -(o_del + e_del * (i + 1)) : SSQ_MINUS_INF;
		for (j = beg; j < end; ++j) {
			i32 h, m = S.h[j], e = S.e[j];
			uint8_t d;
			S.h[j] = h1;
			m += score_of(o, q[j], tb);
			d = m >= e ? 0 : 1;
			h = m >= e ? m : e;
			d = h >= f ? d : 2;
			h = h >= f ? h : f;
			h1 = h;
			tt = m - oe_del;
			e -= e_del;
			d |= e > tt ? 1 << 2 : 0;
			e = e > tt ? e : tt;
			S.e[j] = e;
			tt = m - oe_ins;
			f -= e_ins;
			d |= f > tt ? 2 << 4 : 0;
			f = f > tt ? f : tt;
			if (S.z) S.z[(size_t)i * n_col + (j - beg)] = d;
		}
		S.h[end] = h1; S.e[end] = SSQ_MINUS_INF;
	}
	const int score = S.h[qlen];
	if (S.z && cig && n_cig) { // traceback, operations collected from the end then reversed
		int n = 0, which = 0;
		bool full = false;
		i = tlen - 1; k = (i + w + 1 < qlen ? i + w + 1 : qlen) - 1;
#define PUSH_OP(op_, len_) do { if (n == 0 || (int)(cig[n - 1] & 0xf) != (op_)) { if (n < cig_cap) cig[n++] = (u32)(len_) << 4 | (op_); else full = true; } else cig[n - 1] += (u32)(len_) << 4; } while (0)
		while (i >= 0 && k >= 0) {
			which = S.z[(size_t)i * n_col + (k - (i > w ? i - w : 0))] >> (which << 1) & 3;
			if (which == 0) { PUSH_OP(0, 1); --i; --k; }
			else if (which == 1) { PUSH_OP(2, 1); --i; }
			else { PUSH_OP(1, 1); --k; }
		}
		if (i >= 0) PUSH_OP(2, i + 1);
		if (k >= 0) PUSH_OP(1, k + 1);
#undef PUSH_OP
		for (i = 0; i < n >> 1; ++i) { u32 x = cig[i]; cig[i] = cig[n - 1 - i]; cig[n - 1 - i] = x; }
		*n_cig = full ? -1 : n;
	}
	return score;
}

SSQ_HD int iabs(int x) { return x < 0 ? -x : x; }

// small text sink for MD strings
struct TextOut { char *s; int n, cap; };
SSQ_HD void tput(TextOut &t, char c) { if (t.n < t.cap) t.s[t.n] = c; ++t.n; }
SSQ_HD void tputn(TextOut &t, int v)
{
	char b[12]; int k = 0;
	do { b[k++] = (char)('0' + v % 10); v /= 10; } while (v);
	while (k) tput(t, b[--k]);
}

// Per-thread scratch for everything that needs sequences of one read: qbuf (read length), rbuf (reference window), DP rows.
struct AlnScratch { uint8_t *qbuf, *rbuf; GlobalScratch g; int rcap; };

// global alignment of query[0,l_query) against reference [rb,re) of the doubled coordinate space.
// score always; CIGAR/NM/MD when cig != null.  Returns false if the region is invalid.
SSQ_HD bool gen_cigar(const DevIndex &ix, const ssq_opts_t &o, int w_, int l_query, const uint8_t *query, i64 rb, i64 re, const AlnScratch &S,
                      int *score, u32 *cig, int cig_cap, int *n_cig, int *NM, TextOut *md)
{
	const i64 l_pac = ix.l_pac;
	int i;
	if (n_cig) *n_cig = 0;
	if (NM) *NM = -1;
	if (l_query <= 0 || rb >= re || (rb < l_pac && re > l_pac)) return false;
	const int rlen = (int)(re - rb);
	if (rlen > S.rcap) return false;
	const bool rev = rb >= l_pac; // reverse both so that gaps end up left-aligned on the forward strand
	for (i = 0; i < rlen; ++i) S.rbuf[rev ? rlen - 1 - i : i] = (uint8_t)ref_base(ix, rb + i);
	for (i = 0; i < l_query; ++i) S.qbuf[rev ? l_query - 1 - i : i] = query[i];
	if (l_query == rlen && w_ == 0) { // ungapped
		if (cig && n_cig) { cig[0] = (u32)l_query << 4; *n_cig = 1; }
		int sc = 0;
		for (i = 0; i < l_query; ++i) sc += score_of(o, S.qbuf[i], S.rbuf[i]);
		*score = sc;
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
		GlobalScratch g = S.g;
		if (!cig) g.z = 0;
		else if ((long)(l_query < 2 * w + 1 ? l_query : 2 * w + 1) * rlen > g.zcap) { if (n_cig) *n_cig = -1; return false; } // traceback matrix would not fit: reported, never silent
		*score = sw_global(o, l_query, S.qbuf, rlen, S.rbuf, w, g, cig, cig_cap, n_cig);
		if (cig && n_cig && *n_cig < 0) return false; // more operations than cig_cap: reported like the matrix overflow above
	}
	if (NM && cig && n_cig) {
		int k, x, y, u, n_mm = 0, n_gap = 0;
		const char *int2base = rb < l_pac ? "ACGTN" : "TGCAN";
		for (k = 0, x = y = u = 0; k < *n_cig; ++k) {
			const int op = cig[k] & 0xf, len = (int)(cig[k] >> 4);
			if (op == 0) {
				for (i = 0; i < len; ++i) {
					if (S.qbuf[x + i] != S.rbuf[y + i]) { if (md) { tputn(*md, u); tput(*md, int2base[S.rbuf[y + i]]); } ++n_mm; u = 0; }
					else ++u;
				}
				x += len; y += len;
			} else if (op == 2) {
				if (k > 0 && k < *n_cig - 1) { // terminal deletions get squeezed out later
					if (md) { tputn(*md, u); tput(*md, '^'); for (i = 0; i < len; ++i) tput(*md, int2base[S.rbuf[y + i]]); }
					u = 0; n_gap += len;
				}
				y += len;
			} else if (op == 1) { x += len; n_gap += len; }
		}
		if (md) tputn(*md, u);
		*NM = n_mm + n_gap;
	}
	return true;
}

// ---------------------------------------------------------------------- sort / dedup / patch ----
struct Ars2Lt { SSQ_HD bool operator()(const AlnReg &a, const AlnReg &b) const { return a.re < b.re; } };
struct ArsLt { SSQ_HD bool operator()(const AlnReg &a, const AlnReg &b) const { return a.score > b.score || (a.score == b.score && (a.rb < b.rb || (a.rb == b.rb && a.qb < b.qb))); } };
struct ArsHashLt { SSQ_HD bool operator()(const AlnReg &a, const AlnReg &b) const { return a.score > b.score || (a.score == b.score && a.hash < b.hash); } };

SSQ_HD int patch_reg(const DevIndex &ix, const ssq_opts_t &o, const uint8_t *query, const AlnReg &a, const AlnReg &b, const AlnScratch &S, int *w_out)
{
	int w, score = 0, q_s, r_s;
	double r;
	if (a.rb < ix.l_pac && b.rb >= ix.l_pac) return 0;
	if (a.qb >= b.qb || a.qe >= b.qe || a.re >= b.re) return 0; // not colinear
	w = (int)((a.re - b.rb) - (a.qe - b.qb));
	w = w > 0 ? w : -w;
	r = (double)(a.re - b.rb) / (b.re - a.rb) - (double)(a.qe - b.qb) / (b.qe - a.qb);
	r = r > 0. ? r : -r;
	if (a.re < b.rb || a.qe < b.qb) { if (w > o.w << 1 || r >= 0.05f) return 0; }
	else if (w > o.w << 2 || r >= 0.05f * 2) return 0;
	w += a.w + b.w;
	w = w < o.w << 2 ? w : o.w << 2;
	if (!gen_cigar(ix, o, w, b.qe - a.qb, query + a.qb, a.rb, b.re, S, &score, 0, 0, 0, 0, 0)) score = 0;
	q_s = (int)((double)(b.qe - a.qb) / ((b.qe - b.qb) + (a.qe - a.qb)) * (b.score + a.score) + .499);
	r_s = (int)((double)(b.re - a.rb) / ((b.re - b.rb) + (a.re - a.rb)) * (b.score + a.score) + .499);
	if ((double)score / (q_s > r_s ? q_s : r_s) < 0.90f) return 0;
	*w_out = w;
	return score;
}

// The reference sorts the 96-byte records themselves; the order it leaves equal keys in is part of its behaviour, so the SAME
// introsort runs here — on an index array, comparing through it (identical comparisons and swaps, hence the identical
// permutation) — and the records are then moved once, cycle by cycle.  idx: n scratch ints; null: sort the records directly
template <class LT> struct IdxLt { const AlnReg *a; LT lt; SSQ_HD bool operator()(i32 x, i32 y) const { return lt(a[x], a[y]); } };
template <class LT>
SSQ_HD void sort_regs(int n, AlnReg *a, i32 *idx, LT lt)
{
	if (!idx || n < 8) { ks_introsort((long)n, a, lt); return; }
	for (int i = 0; i < n; ++i) idx[i] = i;
	IdxLt<LT> il; il.a = a; il.lt = lt;
	ks_introsort((long)n, idx, il);
	for (int s = 0; s < n; ++s) { // position k takes record idx[k]
		if (idx[s] == s) continue;
		const AlnReg tmp = a[s];
		int j = s;
		while (idx[j] != s) { const int nj = idx[j]; a[j] = a[nj]; idx[j] = j; j = nj; }
		a[j] = tmp; idx[j] = j;
	}
}

// query == null disables patching (the call made from mate rescue); idx: optional n scratch ints (see sort_regs)
SSQ_HD int sort_dedup_patch(const DevIndex &ix, const ssq_opts_t &o, const uint8_t *query, int n, AlnReg *a, const AlnScratch &S, i32 *idx = 0)
{
	int m, i, j;
	if (n <= 1) return n;
	sort_regs(n, a, idx, Ars2Lt());
	for (i = 0; i < n; ++i) a[i].n_comp = 1;
	for (i = 1; i < n; ++i) {
		AlnReg &p = a[i];
		if (p.rid != a[i - 1].rid || p.rb >= a[i - 1].re + o.max_chain_gap) continue;
		for (j = i - 1; j >= 0 && p.rid == a[j].rid && p.rb < a[j].re + o.max_chain_gap; --j) {
			AlnReg &q = a[j];
			i64 orr, oq, mr, mq;
			int score, w;
			if (q.qe == q.qb) continue;
			orr = q.re - p.rb;
			oq = q.qb < p.qb ? q.qe - p.qb : p.qe - q.qb;
			mr = q.re - q.rb < p.re - p.rb ? q.re - q.rb : p.re - p.rb;
			mq = q.qe - q.qb < p.qe - p.qb ? q.qe - q.qb : p.qe - p.qb;
			if (orr > o.mask_level_redun * mr && oq > o.mask_level_redun * mq) {
				if (p.score < q.score) { p.qe = p.qb; break; }
				else q.qe = q.qb;
			} else if (query && q.rb < p.rb && (score = patch_reg(ix, o, query, q, p, S, &w)) > 0) {
				p.n_comp += q.n_comp + 1;
				p.seedcov = p.seedcov > q.seedcov ? p.seedcov : q.seedcov;
				p.sub = p.sub > q.sub ? p.sub : q.sub;
				p.csub = p.csub > q.csub ? p.csub : q.csub;
				p.qb = q.qb; p.rb = q.rb;
				p.truesc = p.score = score;
				p.w = w;
				q.qb = q.qe;
			}
		}
	}
	for (i = 0, m = 0; i < n; ++i) if (a[i].qe > a[i].qb) { if (m != i) a[m++] = a[i]; else ++m; }
	n = m;
	sort_regs(n, a, idx, ArsLt());
	for (i = 1; i < n; ++i) if (a[i].score == a[i - 1].score && a[i].rb == a[i - 1].rb && a[i].qb == a[i - 1].qb) a[i].qe = a[i].qb;
	for (i = 1, m = 1; i < n; ++i) if (a[i].qe > a[i].qb) { if (m != i) a[m++] = a[i]; else ++m; }
	return m;
}

// --------------------------------------------------------------------------- local SW (mate rescue) ----
// Scalar emulation of the 128-bit striped kernel: padded query of slen*P cells in P segments; within a row F is first
// carried inside a segment (E of the next row is taken from that partial H), then up to 16 "lazy F" rounds carry F across
// segment boundaries into H only.  Byte mode saturates at 255 around a bias `shift`.
struct LocalRes { int score, te, qe, score2, te2, tb, qb; };
struct LocalScratch { i32 *H0, *H1, *E, *Hmax; u64 *b; int b_cap; }; // 4 x (qlen padded) ints, b: sub-optimal row list

#define SSQ_XBYTE 0x10000
#define SSQ_XSTOP 0x20000
#define SSQ_XSUBO 0x40000
#define SSQ_XSTART 0x80000

SSQ_HD LocalRes sw_local_pass(const ssq_opts_t &o, bool bytes, int qlen, const uint8_t *q, int tlen, const uint8_t *t, int xtra, const LocalScratch &S)
{
	const int P = bytes ? 16 : 8, slen = (qlen + P - 1) / P, n = slen * P;
	const int oe_del = o.o_del + o.e_del, oe_ins = o.o_ins + o.e_ins, e_del = o.e_del, e_ins = o.e_ins;
	const int shift = o.b > 1 ? o.b : 1, maxsc = o.a; // most negative matrix entry is -b (or -1 for N); largest is a
	i32 *H0 = S.H0, *H1 = S.H1, *E = S.E, *Hmax = S.Hmax;
	int i, k, s, te = -1, gmax = 0, n_b = 0;
	LocalRes r;
	r.score = 0; r.te = r.qe = -1; r.score2 = -1; r.te2 = -1; r.tb = r.qb = -1;
	const int minsc = (xtra & SSQ_XSUBO) ? xtra & 0xffff : 0x10000;
	const int endsc = (xtra & SSQ_XSTOP) ? xtra & 0xffff : 0x10000;
	for (i = 0; i < n; ++i) H0[i] = H1[i] = E[i] = Hmax[i] = 0;
	for (i = 0; i < tlen; ++i) {
		int imax = 0, fl[16];
		const int tb = t[i];
		for (s = 0; s < P; ++s) { // main pass, one segment after the other
			int f = 0;
			const int base = s * slen;
			for (k = 0; k < slen; ++k) {
				const int pos = base + k;
				int h = pos > 0 ? H0[pos - 1] : 0, e, tt;
				const int sc = pos < qlen ? score_of(o, q[pos], tb) : 0;
				if (bytes) { h += sc + shift; if (h > 255) h = 255; h -= shift; if (h < 0) h = 0; }
				else { h += sc; if (h > 32767) h = 32767; }
				e = E[pos];
				h = h > e ? h : e;
				h = h > f ? h : f;
				imax = imax > h ? imax : h;
				H1[pos] = h;
				tt = h - oe_del; if (tt < 0) tt = 0;
				e -= e_del; if (e < 0) e = 0;
				E[pos] = e > tt ? e : tt;
				tt = h - oe_ins; if (tt < 0) tt = 0;
				f -= e_ins; if (f < 0) f = 0;
				f = f > tt ? f : tt;
			}
			fl[s] = f;
		}
		{ // lazy F across segments, lock-step over the P lanes
			bool done = false;
			for (int round = 0; round < 16 && !done; ++round) {
				for (s = P - 1; s > 0; --s) fl[s] = fl[s - 1];
				fl[0] = 0;
				for (k = 0; k < slen; ++k) {
					bool all = true;
					for (s = 0; s < P; ++s) {
						const int pos = s * slen + k;
						int h = H1[pos], tt;
						h = h > fl[s] ? h : fl[s];
						H1[pos] = h;
						tt = h - oe_ins; if (tt < 0) tt = 0;
						fl[s] -= e_ins; if (fl[s] < 0) fl[s] = 0;
						if (fl[s] > tt) all = false;
					}
					if (all) { done = true; break; }
				}
			}
		}
		if (imax >= minsc) {
			if (n_b == 0 || (i32)S.b[n_b - 1] + 1 != i) { if (n_b < S.b_cap) S.b[n_b++] = (u64)imax << 32 | (u32)i; }
			else if ((int)(S.b[n_b - 1] >> 32) < imax) S.b[n_b - 1] = (u64)imax << 32 | (u32)i;
		}
		if (imax > gmax) {
			gmax = imax; te = i;
			for (k = 0; k < n; ++k) Hmax[k] = H1[k];
			if (bytes ? (gmax + shift >= 255 || gmax >= endsc) : gmax >= endsc) break;
		}
		{ i32 *x = H1; H1 = H0; H0 = x; }
	}
	r.score = bytes ? (gmax + shift < 255 ? gmax : 255) : gmax;
	r.te = te;
	if (!bytes || r.score != 255) {
		int max = -1;
		for (i = 0; i < n; ++i) { // memory order of the striped vectors
			const int pos = i / P + (i % P) * slen, v = Hmax[pos];
			if (v > max) { max = v; r.qe = pos; }
			else if (v == max && pos < r.qe) r.qe = pos;
		}
		if (n_b) {
			const int d = (r.score + maxsc - 1) / maxsc, low = te - d, high = te + d;
			for (i = 0; i < n_b; ++i) {
				const int e = (i32)S.b[i];
				if ((e < low || e > high) && (int)(S.b[i] >> 32) > r.score2) { r.score2 = (int)(S.b[i] >> 32); r.te2 = e; }
			}
		}
	}
	return r;
}

// forward pass for score/end, then a reversed pass for the start (q and t are modified in place and restored)
SSQ_HD LocalRes sw_local(const ssq_opts_t &o, int qlen, uint8_t *q, int tlen, uint8_t *t, int xtra, const LocalScratch &S)
{
	const bool bytes = (xtra & SSQ_XBYTE) != 0;
	LocalRes r = sw_local_pass(o, bytes, qlen, q, tlen, t, xtra, S), rr;
	if ((xtra & SSQ_XSTART) == 0 || ((xtra & SSQ_XSUBO) && r.score < (xtra & 0xffff))) return r;
	int i;
#define REV(p_, l_) for (i = 0; i < (l_) >> 1; ++i) { uint8_t x_ = (p_)[i]; (p_)[i] = (p_)[(l_) - 1 - i]; (p_)[(l_) - 1 - i] = x_; }
	REV(q, r.qe + 1) REV(t, r.te + 1)
	rr = sw_local_pass(o, bytes, r.qe + 1, q, tlen, t, SSQ_XSTOP | r.score, S);
	REV(q, r.qe + 1) REV(t, r.te + 1)
#undef REV
	if (r.score == rr.score) { r.tb = r.te - rr.te; r.qb = r.qe - rr.qe; }
	return r;
}

struct PeStat { i32 low, high, failed, pad; double avg, std; };

SSQ_HD int infer_dir(i64 l_pac, i64 b1, i64 b2, i64 *dist)
{
	const int r1 = b1 >= l_pac, r2 = b2 >= l_pac;
	const i64 p2 = r1 == r2 ? b2 : (l_pac << 1) - 1 - b2;
	*dist = p2 > b1 ? p2 - b1 : b1 - p2;
	return (r1 == r2 ? 0 : 1) ^ (p2 > b1 ? 0 : 3);
}

struct MateScratch { uint8_t *seq, *ref; int ref_cap; LocalScratch L; AlnScratch A; };

// the window orientation r of one mem_matesw() aligns the mate in: [*rb, *re) on the doubled reference; false when the orientation
// aligns nothing (window outside the hit's contig, or shorter than a seed)
SSQ_HD bool rescue_window(const DevIndex &ix, const ssq_opts_t &o, const PeStat *pes, const AlnReg &a, int l_ms, int r, i64 *rb_, i64 *re_)
{
	const i64 l_pac = ix.l_pac;
	const int is_rev = (r >> 1 != (r & 1)), is_larger = !(r >> 1);
	i64 rb, re;
	int rid = -1;
	if (!is_rev) {
		rb = is_larger ? a.rb + pes[r].low : a.rb - pes[r].high;
		re = (is_larger ? a.rb + pes[r].high : a.rb - pes[r].low) + l_ms;
	} else {
		rb = (is_larger ? a.rb + pes[r].low : a.rb - pes[r].high) - l_ms;
		re = is_larger ? a.rb + pes[r].high : a.rb - pes[r].low;
	}
	if (rb < 0) rb = 0;
	if (re > l_pac << 1) re = l_pac << 1;
	if (rb < re) { // clamp to the contig/strand holding the window's midpoint
		int rv;
		const i64 mid = (rb + re) >> 1;
		rid = pos2rid(ix, depos(ix, mid, rv));
		i64 far_beg = ix.ann_off[rid], far_end = far_beg + ix.ann_len[rid];
		if (rv) { i64 t = far_beg; far_beg = (l_pac << 1) - far_end; far_end = (l_pac << 1) - t; }
		rb = rb > far_beg ? rb : far_beg;
		re = re < far_end ? re : far_end;
	}
	*rb_ = rb; *re_ = re;
	return a.rid == rid && re - rb >= o.min_seed_len;
}

// Speculative mate rescue.  What a rescue alignment computes depends only on the hit it starts from (taken from the snapshot of
// near-best hits made before any rescue), the orientation and the mate's sequence — not on the mate's region list, which only
// decides whether the alignment is SKIPPED.  So every alignment the initial lists do not skip can be computed ahead, one task each,
// spread evenly over the machine; the sequential replay (mate_rescue below, in the reference's order, with the lists evolving as
// the reference's do) then looks its alignments up instead of computing them.  A replay step whose alignment was not computed
// ahead (possible when de-duplication removed the hit that had made the initial list skip it) computes it on the spot.
struct RTask { u32 slot, key; i64 rb; i32 tlen, l_ms; }; // key = end << 16 | snapshot index << 2 | orientation: ascending in replay order
struct RCache { const RTask *t; const LocalRes *res; int n, cur; unsigned int *miss; };
SSQ_HD const LocalRes *rcache_find(RCache &c, u32 key, i64 rb, int tlen)
{
	while (c.cur < c.n && c.t[c.cur].key < key) ++c.cur;
	if (c.cur < c.n && c.t[c.cur].key == key && c.t[c.cur].rb == rb && c.t[c.cur].tlen == tlen) return &c.res[c.cur];
	return 0;
}
SSQ_HD int rescue_xtra(const ssq_opts_t &o, int l_ms) { return SSQ_XSUBO | SSQ_XSTART | (l_ms * o.a < 250 ? SSQ_XBYTE : 0) | (o.min_seed_len * o.a); }

// one mem_matesw(): rescue the mate `ms` of hit `a` inside the windows the insert-size bounds allow; ma[0..*n_ma) is the mate's
// region list (capacity ma_cap), kept sorted by score and de-duplicated.  Returns the number of windows aligned, -1 when a window
// does not fit S.ref_cap (callers size the scratch from the batch's insert-size bounds and treat -1 as an error)
SSQ_HD int mate_rescue(const DevIndex &ix, const ssq_opts_t &o, const PeStat pes[4], const AlnReg &a, int l_ms, const uint8_t *ms, AlnReg *ma, int *n_ma, int ma_cap,
                       const MateScratch &S, i32 *idx = 0, RCache *rc = 0, u32 key = 0)
{
	const i64 l_pac = ix.l_pac;
	int i, r, skip[4], n = 0;
	for (r = 0; r < 4; ++r) skip[r] = pes[r].failed ? 1 : 0;
	for (i = 0; i < *n_ma; ++i) {
		i64 dist;
		r = infer_dir(l_pac, a.rb, ma[i].rb, &dist);
		if (dist >= pes[r].low && dist <= pes[r].high) skip[r] = 1;
	}
	if (skip[0] + skip[1] + skip[2] + skip[3] == 4) return 0;
	for (r = 0; r < 4; ++r) {
		if (skip[r]) continue;
		const int is_rev = (r >> 1 != (r & 1));
		i64 rb, re;
		if (rescue_window(ix, o, pes, a, l_ms, r, &rb, &re)) {
			if (re - rb > S.ref_cap) return -1; // window beyond the caller's scratch: reported, never skipped silently (the reference has no limit)
			const int tlen = (int)(re - rb);
			const LocalRes *ahead = rc ? rcache_find(*rc, key | (u32)r, rb, tlen) : 0;
			LocalRes aln;
			if (ahead) aln = *ahead;
			else {
				if (rc && rc->miss) ++*rc->miss;
				for (i = 0; i < l_ms; ++i) S.seq[is_rev ? l_ms - 1 - i : i] = is_rev ? (ms[i] < 4 ? 3 - ms[i] : 4) : ms[i];
				for (i = 0; i < tlen; ++i) S.ref[i] = (uint8_t)ref_base(ix, rb + i);
				aln = sw_local(o, l_ms, S.seq, tlen, S.ref, rescue_xtra(o, l_ms), S.L);
			}
			if (aln.score >= o.min_seed_len && aln.qb >= 0) {
				AlnReg b;
				b.rid = a.rid;
				b.qb = is_rev ? l_ms - (aln.qe + 1) : aln.qb;
				b.qe = is_rev ? l_ms - aln.qb : aln.qe + 1;
				b.rb = is_rev ? (l_pac << 1) - (rb + aln.te + 1) : rb + aln.tb;
				b.re = is_rev ? (l_pac << 1) - (rb + aln.tb) : rb + aln.te + 1;
				b.score = aln.score; b.truesc = 0; b.sub = 0; b.csub = aln.score2; b.sub_n = 0; b.w = 0;
				b.secondary = -1; b.secondary_all = 0; b.seedlen0 = 0; b.n_comp = 0; b.frac_rep = 0.f; b.hash = 0;
				b.seedcov = (int)((b.re - b.rb < b.qe - b.qb ? b.re - b.rb : b.qe - b.qb) >> 1);
				if (*n_ma < ma_cap) {
					++*n_ma;
					for (i = 0; i < *n_ma - 1; ++i) if (ma[i].score < b.score) break;
					const int at = i;
					for (i = *n_ma - 1; i > at; --i) ma[i] = ma[i - 1];
					ma[at] = b;
				}
			}
			++n;
		}
		if (n) *n_ma = sort_dedup_patch(ix, o, 0, *n_ma, ma, S.A, idx);
	}
	return n;
}

// ---------------------------------------------------------------------------------- region -> alignment ----
struct AlnOut { // fixed-size result of reg2aln; CIGAR ops and MD text live in per-alignment slices of two pools
	i64 pos;
	i32 rid, flag, is_rev, mapq_unused, NM, n_cigar, score, sub, md_len, pad;
};

SSQ_HD int infer_bw(int l1, int l2, int score, int a, int q, int r)
{
	int w;
	if (l1 == l2 && l1 * a - score < (q + r - a) << 1) return 0;
	w = (int)((double)((l1 < l2 ? l1 : l2) * a - score - q) / r + 2.);
	if (w < iabs(l1 - l2)) w = iabs(l1 - l2);
	return w;
}

// cig has room for cig_cap ops (>= 2 spare for clipping); md for md_cap chars
SSQ_HD void reg2aln(const DevIndex &ix, const ssq_opts_t &o, int l_query, const uint8_t *query, const AlnReg &ar, const AlnScratch &S,
                    AlnOut &a, u32 *cig, int cig_cap, char *md, int md_cap)
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
	do { // widen the band until the global score catches up with the extension score
		w2 = w2 < o.w << 2 ? w2 : o.w << 2;
		t.n = 0;
		gen_cigar(ix, o, w2, qe - qb, query + qb, rb, re, S, &score, cig, cig_cap - 2, &n_cigar, &NM, &t);
		if (score == last_sc || w2 == o.w << 2) break;
		last_sc = score;
		w2 <<= 1;
	} while (++i < 3 && score < ar.truesc - o.a);
	a.NM = NM;
	i64 pos = depos(ix, rb < ix.l_pac ? rb : re - 1, is_rev);
	a.is_rev = is_rev;
	if (n_cigar > 0) { // squeeze out a leading or trailing deletion (n_cigar < 0 = capacity error, passed through)
		if ((cig[0] & 0xf) == 2) { pos += cig[0] >> 4; --n_cigar; for (i = 0; i < n_cigar; ++i) cig[i] = cig[i + 1]; }
		else if ((cig[n_cigar - 1] & 0xf) == 2) --n_cigar;
	}
	if (n_cigar >= 0 && (qb != 0 || qe != l_query)) {
		const int clip5 = is_rev ? l_query - qe : qb, clip3 = is_rev ? qb : l_query - qe;
		if (clip5) { for (i = n_cigar; i > 0; --i) cig[i] = cig[i - 1]; cig[0] = (u32)clip5 << 4 | 3; ++n_cigar; }
		if (clip3) cig[n_cigar++] = (u32)clip3 << 4 | 3;
	}
	a.n_cigar = n_cigar;
	if (n_cigar < 0) { a.rid = ar.rid; a.pos = 0; a.score = ar.score; a.sub = 0; a.md_len = 0; a.mapq_unused = 0; a.pad = 0; return; }
	a.rid = pos2rid(ix, pos);
	a.pos = pos - ix.ann_off[a.rid];
	a.score = ar.score; a.sub = ar.sub > ar.csub ? ar.sub : ar.csub;
	a.md_len = t.n < md_cap ? t.n : md_cap;
	a.mapq_unused = 0; a.pad = 0;
}
