/*
 * ssqo_ksw.c — ORACLE (test infrastructure): the three Smith-Waterman flavours of BWA-MEM.
 * SURVEY.md §8a rows a7 (ksw_extend2, banded affine-gap extension with per-row band trimming and
 * z-drop), a14 (ksw_global2, banded global DP + traceback), a11 (ksw_align2 = Farrar-striped local
 * SW, u8 then i16 — restated here as a scalar emulation of the striped evaluation order, including
 * its lane/segment artefacts, so that scores, end points and the 2nd-best score agree).
 * Call sites in the reference: inside `$BWA mem`, speedseq/bin/speedseq:438,468.
 */
#include <stdlib.h>
#include <string.h>
#include "ssqo.h"

typedef struct { int32_t h, e; } eh_t;

int ssqo_ksw_extend2(int qlen, const uint8_t *query, int tlen, const uint8_t *target, int m, const int8_t *mat,
                     int o_del, int e_del, int o_ins, int e_ins, int w, int end_bonus, int zdrop, int h0,
                     int *_qle, int *_tle, int *_gtle, int *_gscore, int *_max_off)
{
	eh_t *eh;
	int8_t *qp;
	int i, j, k, oe_del = o_del + e_del, oe_ins = o_ins + e_ins, beg, end, max, max_i, max_j, max_ins, max_del, max_ie, gscore, max_off;
	++ssqo_cnt.n_sw_calls;
	ssqo_cnt.sw_bytes += (uint64_t)qlen + (uint64_t)(tlen + 3) / 4 + 24;
	qp = (int8_t*)malloc((size_t)qlen * m);
	eh = (eh_t*)calloc(qlen + 1, sizeof(eh_t));
	for (k = i = 0; k < m; ++k) {
		const int8_t *p = &mat[k * m];
		for (j = 0; j < qlen; ++j) qp[i++] = p[query[j]];
	}
	/* row -1: only insertions from h0 */
	eh[0].h = h0; eh[1].h = h0 > oe_ins ? h0 - oe_ins : 0;
	for (j = 2; j <= qlen && eh[j - 1].h > e_ins; ++j) eh[j].h = eh[j - 1].h - e_ins;
	/* the band can never usefully exceed the longest gap the scores can pay for */
	for (i = 0, max = 0; i < m * m; ++i) max = max > mat[i] ? max : mat[i];
	max_ins = (int)((double)(qlen * max + end_bonus - o_ins) / e_ins + 1.);
	max_ins = max_ins > 1 ? max_ins : 1;
	w = w < max_ins ? w : max_ins;
	max_del = (int)((double)(qlen * max + end_bonus - o_del) / e_del + 1.);
	max_del = max_del > 1 ? max_del : 1;
	w = w < max_del ? w : max_del;
	max = h0; max_i = max_j = -1; max_ie = -1; gscore = -1; max_off = 0;
	beg = 0; end = qlen;
	for (i = 0; i < tlen; ++i) {
		int t, f = 0, h1, mrow = 0, mj = -1;
		const int8_t *q = &qp[target[i] * qlen];
		if (beg < i - w) beg = i - w;
		if (end > i + w + 1) end = i + w + 1;
		if (end > qlen) end = qlen;
		if (beg == 0) { h1 = h0 - (o_del + e_del * (i + 1)); if (h1 < 0) h1 = 0; } else h1 = 0;
		for (j = beg; j < end; ++j) {
			/* eh[j] holds H(i-1,j-1) and E(i,j); f = F(i,j); h1 = H(i,j-1) */
			eh_t *p = &eh[j];
			int h, M = p->h, e = p->e;
			p->h = h1;
			M = M ? M + q[j] : 0; /* a dead diagonal stays dead */
			h = M > e ? M : e;
			h = h > f ? h : f;
			h1 = h;
			mj = mrow > h ? mj : j; /* ties: the later column wins */
			mrow = mrow > h ? mrow : h;
			t = M - oe_del; t = t > 0 ? t : 0;
			e -= e_del; e = e > t ? e : t;
			p->e = e;
			t = M - oe_ins; t = t > 0 ? t : 0;
			f -= e_ins; f = f > t ? f : t;
		}
		ssqo_cnt.sw_cells += (uint64_t)(end > beg ? end - beg : 0);
		eh[end].h = h1; eh[end].e = 0;
		if (j == qlen) { /* reached the end of the query: ties go to the later row */
			max_ie = gscore > h1 ? max_ie : i;
			gscore = gscore > h1 ? gscore : h1;
		}
		if (mrow == 0) break;
		if (mrow > max) {
			max = mrow; max_i = i; max_j = mj;
			max_off = max_off > abs(mj - i) ? max_off : abs(mj - i);
		} else if (zdrop > 0) {
			if (i - max_i > mj - max_j) {
				if (max - mrow - ((i - max_i) - (mj - max_j)) * e_del > zdrop) break;
			} else {
				if (max - mrow - ((mj - max_j) - (i - max_i)) * e_ins > zdrop) break;
			}
		}
		/* shrink the band to the live cells (F is never carried past `end`) */
		for (j = beg; j < end && eh[j].h == 0 && eh[j].e == 0; ++j);
		beg = j;
		for (j = end; j >= beg && eh[j].h == 0 && eh[j].e == 0; --j);
		end = j + 2 < qlen ? j + 2 : qlen;
	}
	free(eh); free(qp);
	if (_qle) *_qle = max_j + 1;
	if (_tle) *_tle = max_i + 1;
	if (_gtle) *_gtle = max_ie + 1;
	if (_gscore) *_gscore = gscore;
	if (_max_off) *_max_off = max_off;
	return max;
}

#define MINUS_INF (-0x40000000)

static uint32_t *push_cigar(int *n, int *m, uint32_t *cigar, int op, int len)
{
	if (*n == 0 || op != (int)(cigar[*n - 1] & 0xf)) {
		if (*n == *m) { *m = *m ? *m << 1 : 4; cigar = (uint32_t*)realloc(cigar, (size_t)*m << 2); }
		cigar[(*n)++] = (uint32_t)len << 4 | op;
	} else cigar[*n - 1] += (uint32_t)len << 4;
	return cigar;
}

int ssqo_ksw_global2(int qlen, const uint8_t *query, int tlen, const uint8_t *target, int m, const int8_t *mat,
                     int o_del, int e_del, int o_ins, int e_ins, int w, int *n_cigar_, uint32_t **cigar_)
{
	eh_t *eh;
	int8_t *qp;
	int i, j, k, oe_del = o_del + e_del, oe_ins = o_ins + e_ins, score, n_col;
	uint8_t *z; /* per cell: bits 0-1 = source of H, bit 2-3 = E continues, bit 4-5 = F continues */
	if (n_cigar_) *n_cigar_ = 0;
	n_col = qlen < 2 * w + 1 ? qlen : 2 * w + 1;
	z = (uint8_t*)malloc((size_t)n_col * tlen + 1);
	qp = (int8_t*)malloc((size_t)qlen * m);
	eh = (eh_t*)calloc(qlen + 1, sizeof(eh_t));
	for (k = i = 0; k < m; ++k) {
		const int8_t *p = &mat[k * m];
		for (j = 0; j < qlen; ++j) qp[i++] = p[query[j]];
	}
	eh[0].h = 0; eh[0].e = MINUS_INF;
	for (j = 1; j <= qlen && j <= w; ++j) eh[j].h = -(o_ins + e_ins * j), eh[j].e = MINUS_INF;
	for (; j <= qlen; ++j) eh[j].h = eh[j].e = MINUS_INF;
	for (i = 0; i < tlen; ++i) {
		int32_t f = MINUS_INF, h1, beg, end, t;
		const int8_t *q = &qp[target[i] * qlen];
		uint8_t *zi = &z[(size_t)i * n_col];
		beg = i > w ? i - w : 0;
		end = i + w + 1 < qlen ? i + w + 1 : qlen;
		h1 = beg == 0 ? -(o_del + e_del * (i + 1)) : MINUS_INF;
		for (j = beg; j < end; ++j) {
			eh_t *p = &eh[j];
			int32_t h, mm = p->h, e = p->e;
			uint8_t d;
			p->h = h1;
			mm += q[j];
			d = mm >= e ? 0 : 1;
			h = mm >= e ? mm : e;
			d = h >= f ? d : 2;
			h = h >= f ? h : f;
			h1 = h;
			t = mm - oe_del;
			e -= e_del;
			d |= e > t ? 1 << 2 : 0;
			e = e > t ? e : t;
			p->e = e;
			t = mm - oe_ins;
			f -= e_ins;
			d |= f > t ? 2 << 4 : 0;
			f = f > t ? f : t;
			zi[j - beg] = d;
		}
		eh[end].h = h1; eh[end].e = MINUS_INF;
	}
	score = eh[qlen].h;
	if (n_cigar_ && cigar_) {
		int n_cigar = 0, m_cigar = 0, which = 0;
		uint32_t *cigar = 0, tmp;
		i = tlen - 1; k = (i + w + 1 < qlen ? i + w + 1 : qlen) - 1;
		while (i >= 0 && k >= 0) {
			which = z[(size_t)i * n_col + (k - (i > w ? i - w : 0))] >> (which << 1) & 3;
			if (which == 0) cigar = push_cigar(&n_cigar, &m_cigar, cigar, 0, 1), --i, --k;
			else if (which == 1) cigar = push_cigar(&n_cigar, &m_cigar, cigar, 2, 1), --i;
			else cigar = push_cigar(&n_cigar, &m_cigar, cigar, 1, 1), --k;
		}
		if (i >= 0) cigar = push_cigar(&n_cigar, &m_cigar, cigar, 2, i + 1);
		if (k >= 0) cigar = push_cigar(&n_cigar, &m_cigar, cigar, 1, k + 1);
		for (i = 0; i < n_cigar >> 1; ++i) tmp = cigar[i], cigar[i] = cigar[n_cigar - 1 - i], cigar[n_cigar - 1 - i] = tmp;
		*n_cigar_ = n_cigar; *cigar_ = cigar;
	}
	free(eh); free(qp); free(z);
	return score;
}

/* ------------------------------------------------------------------------------------------
 * Local SW with the evaluation order of the 128-bit striped kernel: the padded query of
 * slen*P cells (P = 16 lanes for bytes, 8 for words) is cut into P segments of slen cells.
 * Within a row, F is first carried only inside a segment (and E(i+1,.) is taken from that
 * partial H), then the "lazy F" passes carry F across segment boundaries into H only.
 * Byte mode saturates at 255 with a bias `shift`; word mode is plain int16 range.
 * ------------------------------------------------------------------------------------------ */
typedef struct { int size, slen, qlenp, shift, mdiff, max; int *prof; /* 5 x qlenp, unbiased */ } sw_q_t;

static sw_q_t *swq_init(int size, int qlen, const uint8_t *query, int m, const int8_t *mat)
{
	sw_q_t *q = (sw_q_t*)calloc(1, sizeof(sw_q_t));
	int p = size == 1 ? 16 : 8, a, k, lo = 127, hi = 0;
	q->size = size;
	q->slen = (qlen + p - 1) / p;
	q->qlenp = q->slen * p;
	for (a = 0; a < m * m; ++a) { if (mat[a] < lo) lo = mat[a]; if (mat[a] > hi) hi = mat[a]; }
	q->max = hi; q->shift = -lo; q->mdiff = hi - lo;
	q->prof = (int*)calloc((size_t)m * q->qlenp, sizeof(int));
	for (a = 0; a < m; ++a)
		for (k = 0; k < q->qlenp; ++k) q->prof[a * q->qlenp + k] = k < qlen ? mat[a * m + query[k]] : 0;
	return q;
}

static ssqo_kswr_t sw_striped(const sw_q_t *q, int tlen, const uint8_t *target, int o_del, int e_del, int o_ins, int e_ins, int xtra)
{
	const int P = q->size == 1 ? 16 : 8, slen = q->slen, n = q->qlenp, bytes = q->size == 1;
	const int oe_del = o_del + e_del, oe_ins = o_ins + e_ins;
	int *H0 = (int*)calloc(n, sizeof(int)), *H1 = (int*)calloc(n, sizeof(int)), *E = (int*)calloc(n, sizeof(int)), *Hmax = (int*)calloc(n, sizeof(int));
	int *fend = (int*)calloc(P, sizeof(int));
	int i, k, s, te = -1, gmax = 0, minsc, endsc, n_b = 0, m_b = 0;
	uint64_t *b = 0;
	ssqo_kswr_t r;
	r.score = 0; r.te = r.qe = -1; r.score2 = -1; r.te2 = -1; r.tb = r.qb = -1;
	minsc = (xtra & SSQO_KSW_XSUBO) ? xtra & 0xffff : 0x10000;
	endsc = (xtra & SSQO_KSW_XSTOP) ? xtra & 0xffff : 0x10000;
	for (i = 0; i < tlen; ++i) {
		const int *S = q->prof + target[i] * n;
		int imax = 0, *swp;
		/* main pass: per segment s, cells s*slen .. s*slen+slen-1 */
		for (s = 0; s < P; ++s) {
			int f = 0, base = s * slen;
			for (k = 0; k < slen; ++k) {
				int pos = base + k, h, e, t;
				h = pos > 0 ? H0[pos - 1] : 0; /* H(i-1,j-1); the cell before position 0 is 0 */
				if (bytes) { h += S[pos] + q->shift; if (h > 255) h = 255; h -= q->shift; if (h < 0) h = 0; }
				else { h += S[pos]; if (h > 32767) h = 32767; }
				e = E[pos];
				h = h > e ? h : e;
				h = h > f ? h : f;
				imax = imax > h ? imax : h;
				H1[pos] = h;
				t = h - oe_del; if (t < 0) t = 0;
				e -= e_del; if (e < 0) e = 0;
				E[pos] = e > t ? e : t;
				t = h - oe_ins; if (t < 0) t = 0;
				f -= e_ins; if (f < 0) f = 0;
				f = f > t ? f : t;
			}
			fend[s] = f;
		}
		/* lazy F: up to 16 rounds; each round shifts the carried F one segment to the right and walks all cells
		 * in lock-step; stops as soon as no lane can still raise anything */
		{
			int fl[16], round, done = 0;
			for (s = 0; s < P; ++s) fl[s] = fend[s];
			for (round = 0; round < 16 && !done; ++round) {
				for (s = P - 1; s > 0; --s) fl[s] = fl[s - 1];
				fl[0] = 0;
				for (k = 0; k < slen; ++k) {
					int all = 1;
					for (s = 0; s < P; ++s) {
						int pos = s * slen + k, h = H1[pos], t;
						h = h > fl[s] ? h : fl[s];
						H1[pos] = h;
						t = h - oe_ins; if (t < 0) t = 0;
						fl[s] -= e_ins; if (fl[s] < 0) fl[s] = 0;
						if (fl[s] > t) all = 0;
					}
					if (all) { done = 1; break; }
				}
			}
		}
		if (imax >= minsc) {
			if (n_b == 0 || (int32_t)b[n_b - 1] + 1 != i) {
				if (n_b == m_b) { m_b = m_b ? m_b << 1 : 8; b = (uint64_t*)realloc(b, 8 * (size_t)m_b); }
				b[n_b++] = (uint64_t)imax << 32 | (uint32_t)i;
			} else if ((int)(b[n_b - 1] >> 32) < imax) b[n_b - 1] = (uint64_t)imax << 32 | (uint32_t)i;
		}
		if (imax > gmax) {
			gmax = imax; te = i;
			memcpy(Hmax, H1, sizeof(int) * n);
			if (bytes ? (gmax + q->shift >= 255 || gmax >= endsc) : gmax >= endsc) break;
		}
		swp = H1; H1 = H0; H0 = swp;
	}
	r.score = bytes ? (gmax + q->shift < 255 ? gmax : 255) : gmax;
	r.te = te;
	if (!bytes || r.score != 255) {
		int max = -1, low, high;
		/* memory order of the striped vectors: byte index i -> query position i/P + (i%P)*slen */
		for (i = 0; i < n; ++i) {
			int pos = i / P + (i % P) * slen, v = Hmax[pos];
			if (v > max) max = v, r.qe = pos;
			else if (v == max && pos < r.qe) r.qe = pos;
		}
		if (b) {
			i = (r.score + q->max - 1) / q->max;
			low = te - i; high = te + i;
			for (i = 0; i < n_b; ++i) {
				int e = (int32_t)b[i];
				if ((e < low || e > high) && (int)(b[i] >> 32) > r.score2) r.score2 = (int)(b[i] >> 32), r.te2 = e;
			}
		}
	}
	free(b); free(H0); free(H1); free(E); free(Hmax); free(fend);
	return r;
}

static void revseq(int l, uint8_t *s)
{
	int i;
	for (i = 0; i < l >> 1; ++i) { uint8_t t = s[i]; s[i] = s[l - 1 - i]; s[l - 1 - i] = t; }
}

ssqo_kswr_t ssqo_ksw_align2(int qlen, uint8_t *query, int tlen, uint8_t *target, int m, const int8_t *mat,
                            int o_del, int e_del, int o_ins, int e_ins, int xtra)
{
	int size = (xtra & SSQO_KSW_XBYTE) ? 1 : 2;
	sw_q_t *q = swq_init(size, qlen, query, m, mat);
	ssqo_kswr_t r, rr;
	r = sw_striped(q, tlen, target, o_del, e_del, o_ins, e_ins, xtra);
	free(q->prof); free(q);
	if ((xtra & SSQO_KSW_XSTART) == 0 || ((xtra & SSQO_KSW_XSUBO) && r.score < (xtra & 0xffff))) return r;
	revseq(r.qe + 1, query); revseq(r.te + 1, target);
	q = swq_init(size, r.qe + 1, query, m, mat);
	rr = sw_striped(q, tlen, target, o_del, e_del, o_ins, e_ins, SSQO_KSW_XSTOP | r.score);
	revseq(r.qe + 1, query); revseq(r.te + 1, target);
	free(q->prof); free(q);
	if (r.score == rr.score) r.tb = r.te - rr.te, r.qb = r.qe - rr.qe;
	return r;
}
