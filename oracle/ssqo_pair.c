/*
 * ssqo_pair.c — ORACLE (test infrastructure): paired-end half of BWA-MEM and the `bwa mem` driver.
 * SURVEY.md §8a rows a3 (batching), a10 (insert-size statistics per batch), a11 (mate rescue),
 * a12 (pairing), a13 (paired MAPQ), a15 (SAM text + header).
 * Reference call site: speedseq/bin/speedseq:438 (`-p` interleaved) and :468 (two files).
 * Upstream names (not in tree): mem_pestat, mem_matesw, mem_pair, mem_sam_pe, mem_process_seqs,
 * bseq_read, bseq_classify, main_mem, bwa_set_rg, bwa_print_sam_hdr.
 */
#include <stdlib.h>
#include <string.h>
#include <math.h>
#include <ctype.h>
#include <assert.h>
#include <unistd.h>
#include "ssqo.h"
#include "ssqo_kseq.h"
#include "ssqo_sort.h"
#include "ssqo_mem.h"
#include "ssqo_par.h"

typedef struct { uint64_t x, y; } pair64_t;
#define LT_P64(a, b) ((a).x < (b).x || ((a).x == (b).x && (a).y < (b).y))
SSQO_SORT_INIT(p64, pair64_t, LT_P64)

#define MIN_RATIO 0.8
#define MIN_DIR_CNT 10
#define MIN_DIR_RATIO 0.05
#define OUTLIER_BOUND 2.0
#define MAPPING_BOUND 3.0
#define MAX_STDDEV 4.0

static inline int infer_dir(int64_t l_pac, int64_t b1, int64_t b2, int64_t *dist)
{
	int64_t p2;
	int r1 = (b1 >= l_pac), r2 = (b2 >= l_pac);
	p2 = r1 == r2 ? b2 : (l_pac << 1) - 1 - b2; /* mate start seen from read 1's strand */
	*dist = p2 > b1 ? p2 - b1 : b1 - p2;
	return (r1 == r2 ? 0 : 1) ^ (p2 > b1 ? 0 : 3);
}

static int cal_sub(const ssqo_opt_t *opt, const ssqo_alnreg_v *r)
{
	int j;
	for (j = 1; j < (int)r->n; ++j) {
		int b_max = r->a[j].qb > r->a[0].qb ? r->a[j].qb : r->a[0].qb;
		int e_min = r->a[j].qe < r->a[0].qe ? r->a[j].qe : r->a[0].qe;
		if (e_min > b_max) {
			int min_l = r->a[j].qe - r->a[j].qb < r->a[0].qe - r->a[0].qb ? r->a[j].qe - r->a[j].qb : r->a[0].qe - r->a[0].qb;
			if (e_min - b_max >= min_l * opt->mask_level) break;
		}
	}
	return j < (int)r->n ? r->a[j].score : opt->min_seed_len * opt->a;
}

void ssqo_pestat(const ssqo_opt_t *opt, int64_t l_pac, int n, const ssqo_alnreg_v *regs, ssqo_pestat_t pes[4])
{
	int i, d, max;
	struct { size_t n, m; uint64_t *a; } isize[4];
	memset(pes, 0, 4 * sizeof(ssqo_pestat_t));
	memset(isize, 0, sizeof isize);
	for (i = 0; i < n >> 1; ++i) {
		int dir;
		int64_t is;
		const ssqo_alnreg_v *r[2];
		r[0] = &regs[i << 1 | 0]; r[1] = &regs[i << 1 | 1];
		if (r[0]->n == 0 || r[1]->n == 0) continue;
		if (cal_sub(opt, r[0]) > MIN_RATIO * r[0]->a[0].score) continue;
		if (cal_sub(opt, r[1]) > MIN_RATIO * r[1]->a[0].score) continue;
		if (r[0]->a[0].rid != r[1]->a[0].rid) continue;
		dir = infer_dir(l_pac, r[0]->a[0].rb, r[1]->a[0].rb, &is);
		if (is && is <= opt->max_ins) {
			if (isize[dir].n == isize[dir].m) { isize[dir].m = isize[dir].m ? isize[dir].m << 1 : 256; isize[dir].a = (uint64_t*)realloc(isize[dir].a, isize[dir].m * 8); }
			isize[dir].a[isize[dir].n++] = (uint64_t)is;
		}
	}
	fprintf(stderr, "[M::mem_pestat] # candidate unique pairs for (FF, FR, RF, RR): (%ld, %ld, %ld, %ld)\n", (long)isize[0].n, (long)isize[1].n, (long)isize[2].n, (long)isize[3].n);
	for (d = 0; d < 4; ++d) {
		ssqo_pestat_t *r = &pes[d];
		uint64_t *q = isize[d].a;
		size_t qn = isize[d].n;
		int p25, p50, p75, x;
		if (qn < MIN_DIR_CNT) {
			fprintf(stderr, "[M::mem_pestat] skip orientation %c%c as there are not enough pairs\n", "FR"[d >> 1 & 1], "FR"[d & 1]);
			r->failed = 1;
			continue;
		} else fprintf(stderr, "[M::mem_pestat] analyzing insert size distribution for orientation %c%c...\n", "FR"[d >> 1 & 1], "FR"[d & 1]);
		ssqo_sort_u64(qn, q);
		p25 = (int)q[(int)(.25 * qn + .499)];
		p50 = (int)q[(int)(.50 * qn + .499)];
		p75 = (int)q[(int)(.75 * qn + .499)];
		r->low = (int)(p25 - OUTLIER_BOUND * (p75 - p25) + .499);
		if (r->low < 1) r->low = 1;
		r->high = (int)(p75 + OUTLIER_BOUND * (p75 - p25) + .499);
		fprintf(stderr, "[M::mem_pestat] (25, 50, 75) percentile: (%d, %d, %d)\n", p25, p50, p75);
		fprintf(stderr, "[M::mem_pestat] low and high boundaries for computing mean and std.dev: (%d, %d)\n", r->low, r->high);
		for (i = x = 0, r->avg = 0; i < (int)qn; ++i)
			if (q[i] >= (uint64_t)r->low && q[i] <= (uint64_t)r->high) r->avg += q[i], ++x;
		r->avg /= x;
		for (i = 0, r->std = 0; i < (int)qn; ++i)
			if (q[i] >= (uint64_t)r->low && q[i] <= (uint64_t)r->high) r->std += (q[i] - r->avg) * (q[i] - r->avg);
		r->std = sqrt(r->std / x);
		fprintf(stderr, "[M::mem_pestat] mean and std.dev: (%.2f, %.2f)\n", r->avg, r->std);
		r->low = (int)(p25 - MAPPING_BOUND * (p75 - p25) + .499);
		r->high = (int)(p75 + MAPPING_BOUND * (p75 - p25) + .499);
		if (r->low > r->avg - MAX_STDDEV * r->std) r->low = (int)(r->avg - MAX_STDDEV * r->std + .499);
		if (r->high < r->avg + MAX_STDDEV * r->std) r->high = (int)(r->avg + MAX_STDDEV * r->std + .499);
		if (r->low < 1) r->low = 1;
		fprintf(stderr, "[M::mem_pestat] low and high boundaries for proper pairs: (%d, %d)\n", r->low, r->high);
	}
	for (d = 0, max = 0; d < 4; ++d) max = max > (int)isize[d].n ? max : (int)isize[d].n;
	for (d = 0; d < 4; ++d)
		if (pes[d].failed == 0 && isize[d].n < max * MIN_DIR_RATIO) {
			pes[d].failed = 1;
			fprintf(stderr, "[M::mem_pestat] skip orientation %c%c\n", "FR"[d >> 1 & 1], "FR"[d & 1]);
		}
	for (d = 0; d < 4; ++d) free(isize[d].a);
}

/* local SW of the mate inside the window the insert-size bounds allow; new hits are merged into ma */
static int matesw(const ssqo_opt_t *opt, const ssqo_idx_t *idx, const ssqo_pestat_t pes[4], const ssqo_alnreg_t *a, int l_ms, const uint8_t *ms, ssqo_alnreg_v *ma)
{
	const ssqo_bns_t *bns = &idx->bns;
	int64_t l_pac = bns->l_pac;
	int i, r, skip[4], n = 0, rid = -1;
	for (r = 0; r < 4; ++r) skip[r] = pes[r].failed ? 1 : 0;
	for (i = 0; i < (int)ma->n; ++i) { /* orientations that already have a consistent hit */
		int64_t dist;
		r = infer_dir(l_pac, a->rb, ma->a[i].rb, &dist);
		if (dist >= pes[r].low && dist <= pes[r].high) skip[r] = 1;
	}
	if (skip[0] + skip[1] + skip[2] + skip[3] == 4) return 0;
	for (r = 0; r < 4; ++r) {
		int is_rev, is_larger;
		uint8_t *seq, *rev = 0, *ref = 0;
		int64_t rb, re;
		if (skip[r]) continue;
		is_rev = (r >> 1 != (r & 1));
		is_larger = !(r >> 1);
		if (is_rev) {
			rev = (uint8_t*)malloc(l_ms);
			for (i = 0; i < l_ms; ++i) rev[l_ms - 1 - i] = ms[i] < 4 ? 3 - ms[i] : 4;
			seq = rev;
		} else seq = (uint8_t*)ms;
		if (!is_rev) {
			rb = is_larger ? a->rb + pes[r].low : a->rb - pes[r].high;
			re = (is_larger ? a->rb + pes[r].high : a->rb - pes[r].low) + l_ms;
		} else {
			rb = (is_larger ? a->rb + pes[r].low : a->rb - pes[r].high) - l_ms;
			re = is_larger ? a->rb + pes[r].high : a->rb - pes[r].low;
		}
		if (rb < 0) rb = 0;
		if (re > l_pac << 1) re = l_pac << 1;
		rid = -1;
		if (rb < re) ref = ssqo_fetch_seq(bns, idx->pac, &rb, (rb + re) >> 1, &re, &rid);
		if (a->rid == rid && re - rb >= opt->min_seed_len) {
			ssqo_kswr_t aln;
			ssqo_alnreg_t b;
			int tmp, xtra = SSQO_KSW_XSUBO | SSQO_KSW_XSTART | (l_ms * opt->a < 250 ? SSQO_KSW_XBYTE : 0) | (opt->min_seed_len * opt->a);
			aln = ssqo_ksw_align2(l_ms, seq, (int)(re - rb), ref, 5, opt->mat, opt->o_del, opt->e_del, opt->o_ins, opt->e_ins, xtra);
			memset(&b, 0, sizeof b);
			if (aln.score >= opt->min_seed_len && aln.qb >= 0) {
				b.rid = a->rid;
				b.is_alt = a->is_alt;
				b.qb = is_rev ? l_ms - (aln.qe + 1) : aln.qb;
				b.qe = is_rev ? l_ms - aln.qb : aln.qe + 1;
				b.rb = is_rev ? (l_pac << 1) - (rb + aln.te + 1) : rb + aln.tb;
				b.re = is_rev ? (l_pac << 1) - (rb + aln.tb) : rb + aln.te + 1;
				b.score = aln.score;
				b.csub = aln.score2;
				b.secondary = -1;
				b.seedcov = (int)((b.re - b.rb < b.qe - b.qb ? b.re - b.rb : b.qe - b.qb) >> 1);
				if (ma->n == ma->m) { ma->m = ma->m ? ma->m << 1 : 4; ma->a = (ssqo_alnreg_t*)realloc(ma->a, ma->m * sizeof(ssqo_alnreg_t)); }
				++ma->n;
				for (i = 0; i < (int)ma->n - 1; ++i) if (ma->a[i].score < b.score) break; /* keep ma sorted by score */
				tmp = i;
				for (i = (int)ma->n - 1; i > tmp; --i) ma->a[i] = ma->a[i - 1];
				ma->a[i] = b;
			}
			++n;
		}
		if (n) ma->n = ssqo_sort_dedup_patch(opt, 0, 0, (int)ma->n, ma->a);
		free(rev); free(ref);
	}
	return n;
}

static int mem_pair(const ssqo_opt_t *opt, const ssqo_idx_t *idx, const ssqo_pestat_t pes[4], ssqo_alnreg_v a[2], int64_t id, int *sub, int *n_sub, int z[2])
{
	const ssqo_bns_t *bns = &idx->bns;
	pair64_t *v, *u;
	size_t nv = 0, nu = 0, mu = 16;
	int r, i, k, y[4], ret;
	int64_t l_pac = bns->l_pac;
	v = (pair64_t*)malloc(sizeof(pair64_t) * (a[0].n + a[1].n + 1));
	u = (pair64_t*)malloc(sizeof(pair64_t) * mu);
	for (r = 0; r < 2; ++r)
		for (i = 0; i < (int)a[r].n; ++i) {
			pair64_t key;
			ssqo_alnreg_t *e = &a[r].a[i];
			key.x = e->rb < l_pac ? e->rb : (l_pac << 1) - 1 - e->rb; /* forward position */
			key.x = (uint64_t)e->rid << 32 | (key.x - bns->anns[e->rid].offset);
			key.y = (uint64_t)e->score << 32 | i << 2 | (e->rb >= l_pac) << 1 | r;
			v[nv++] = key;
		}
	ssqo_introsort_p64(nv, v);
	y[0] = y[1] = y[2] = y[3] = -1;
	for (i = 0; i < (int)nv; ++i) {
		for (r = 0; r < 2; ++r) { /* two candidate orientations for hit i */
			int dir = r << 1 | (v[i].y >> 1 & 1), which;
			if (pes[dir].failed) continue;
			which = r << 1 | ((v[i].y & 1) ^ 1);
			if (y[which] < 0) continue;
			for (k = y[which]; k >= 0; --k) {
				int64_t dist;
				int q;
				double ns;
				pair64_t *p;
				if ((int)(v[k].y & 3) != which) continue;
				dist = (int64_t)v[i].x - v[k].x;
				if (dist > pes[dir].high) break;
				if (dist < pes[dir].low) continue;
				ns = (dist - pes[dir].avg) / pes[dir].std;
				q = (int)((v[i].y >> 32) + (v[k].y >> 32) + .721 * log(2. * erfc(fabs(ns) * M_SQRT1_2)) * opt->a + .499);
				if (q < 0) q = 0;
				if (nu == mu) { mu <<= 1; u = (pair64_t*)realloc(u, sizeof(pair64_t) * mu); }
				p = &u[nu++];
				p->y = (uint64_t)k << 32 | (uint32_t)i;
				p->x = (uint64_t)q << 32 | (ssqo_hash64(p->y ^ id << 8) & 0xffffffffU);
			}
		}
		y[v[i].y & 3] = i;
	}
	if (nu) {
		int tmp = opt->a + opt->b;
		tmp = tmp > opt->o_del + opt->e_del ? tmp : opt->o_del + opt->e_del;
		tmp = tmp > opt->o_ins + opt->e_ins ? tmp : opt->o_ins + opt->e_ins;
		ssqo_introsort_p64(nu, u);
		i = (int)(u[nu - 1].y >> 32); k = (int)(u[nu - 1].y << 32 >> 32);
		z[v[i].y & 1] = (int)(v[i].y << 32 >> 34);
		z[v[k].y & 1] = (int)(v[k].y << 32 >> 34);
		ret = (int)(u[nu - 1].x >> 32);
		*sub = nu > 1 ? (int)(u[nu - 2].x >> 32) : 0;
		for (i = (int)nu - 2, *n_sub = 0; i >= 0; --i)
			if (*sub - (int)(u[i].x >> 32) <= tmp) ++*n_sub;
	} else ret = 0, *sub = 0, *n_sub = 0;
	free(u); free(v);
	return ret;
}

#define raw_mapq(diff, a) ((int)(6.02 * (diff) / (a) + .499))

static int sam_pe(const ssqo_opt_t *opt, const ssqo_idx_t *idx, const ssqo_pestat_t pes[4], uint64_t id, ssqo_read_t s[2], ssqo_alnreg_v a[2], const char *rg_id)
{
	int n = 0, i, j, z[2], o, subo, n_sub, extra_flag = 1, n_pri[2];
	ssqo_aln_t h[2];
	memset(h, 0, sizeof h);
	{ /* mate rescue from every near-best hit of either end */
		ssqo_alnreg_v b[2] = {{0, 0, 0}, {0, 0, 0}};
		for (i = 0; i < 2; ++i)
			for (j = 0; j < (int)a[i].n; ++j)
				if (a[i].a[j].score >= a[i].a[0].score - opt->pen_unpaired) {
					if (b[i].n == b[i].m) { b[i].m = b[i].m ? b[i].m << 1 : 4; b[i].a = (ssqo_alnreg_t*)realloc(b[i].a, b[i].m * sizeof(ssqo_alnreg_t)); }
					b[i].a[b[i].n++] = a[i].a[j];
				}
		for (i = 0; i < 2; ++i)
			for (j = 0; j < (int)b[i].n && j < opt->max_matesw; ++j)
				n += matesw(opt, idx, pes, &b[i].a[j], s[!i].l_seq, (uint8_t*)s[!i].seq, &a[!i]);
		free(b[0].a); free(b[1].a);
	}
	n_pri[0] = ssqo_mark_primary_se(opt, (int)a[0].n, a[0].a, id << 1 | 0);
	n_pri[1] = ssqo_mark_primary_se(opt, (int)a[1].n, a[1].a, id << 1 | 1);
	if (n_pri[0] && n_pri[1] && (o = mem_pair(opt, idx, pes, a, (int64_t)id, &subo, &n_sub, z)) > 0) {
		int is_multi[2], q_pe, score_un, q_se[2];
		char **XA[2];
		for (i = 0; i < 2; ++i) { /* a second independent hit above threshold => treat as multi-part read */
			for (j = 1; j < n_pri[i]; ++j)
				if (a[i].a[j].secondary < 0 && a[i].a[j].score >= opt->T) break;
			is_multi[i] = j < n_pri[i] ? 1 : 0;
		}
		if (is_multi[0] || is_multi[1]) goto no_pairing;
		score_un = a[0].a[0].score + a[1].a[0].score - opt->pen_unpaired;
		subo = subo > score_un ? subo : score_un;
		q_pe = raw_mapq(o - subo, opt->a);
		if (n_sub > 0) q_pe -= (int)(4.343 * log(n_sub + 1) + .499);
		if (q_pe < 0) q_pe = 0;
		if (q_pe > 60) q_pe = 60;
		q_pe = (int)(q_pe * (1. - .5 * (a[0].a[0].frac_rep + a[1].a[0].frac_rep)) + .499);
		if (o > score_un) { /* the pair beats the two best single-end hits */
			ssqo_alnreg_t *c[2];
			c[0] = &a[0].a[z[0]]; c[1] = &a[1].a[z[1]];
			for (i = 0; i < 2; ++i) {
				if (c[i]->secondary >= 0) c[i]->sub = a[i].a[c[i]->secondary].score, c[i]->secondary = -2;
				q_se[i] = ssqo_approx_mapq_se(opt, c[i]);
			}
			q_se[0] = q_se[0] > q_pe ? q_se[0] : q_pe < q_se[0] + 40 ? q_pe : q_se[0] + 40;
			q_se[1] = q_se[1] > q_pe ? q_se[1] : q_pe < q_se[1] + 40 ? q_pe : q_se[1] + 40;
			extra_flag |= 2;
			q_se[0] = q_se[0] < raw_mapq(c[0]->score - c[0]->csub, opt->a) ? q_se[0] : raw_mapq(c[0]->score - c[0]->csub, opt->a);
			q_se[1] = q_se[1] < raw_mapq(c[1]->score - c[1]->csub, opt->a) ? q_se[1] : raw_mapq(c[1]->score - c[1]->csub, opt->a);
		} else {
			z[0] = z[1] = 0;
			q_se[0] = ssqo_approx_mapq_se(opt, &a[0].a[0]);
			q_se[1] = ssqo_approx_mapq_se(opt, &a[1].a[0]);
		}
		for (i = 0; i < 2; ++i) { /* the chosen hit becomes the representative of its overlap group */
			int k = a[i].a[z[i]].secondary_all;
			if (k >= 0 && k < n_pri[i]) {
				for (j = 0; j < (int)a[i].n; ++j)
					if (a[i].a[j].secondary_all == k || j == k) a[i].a[j].secondary_all = z[i];
				a[i].a[z[i]].secondary_all = -1;
			}
		}
		for (i = 0; i < 2; ++i) XA[i] = ssqo_gen_alt(opt, idx, &a[i], s[i].l_seq, s[i].seq);
		for (i = 0; i < 2; ++i) {
			h[i] = ssqo_reg2aln(opt, idx, s[i].l_seq, s[i].seq, &a[i].a[z[i]]);
			h[i].mapq = q_se[i];
			h[i].flag |= 0x40 << i | extra_flag;
			h[i].XA = XA[i] && XA[i][z[i]] ? strdup(XA[i][z[i]]) : 0;
		}
		for (i = 0; i < 2; ++i) {
			ssqo_sb_t str = {0, 0, 0};
			ssqo_aln2sam(opt, &idx->bns, &str, &s[i], 1, &h[i], 0, &h[!i], rg_id);
			s[i].sam = str.s;
		}
		for (i = 0; i < 2; ++i) {
			ssqo_aln_free(&h[i]);
			if (XA[i]) { for (j = 0; j < (int)a[i].n; ++j) free(XA[i][j]); free(XA[i]); }
		}
		return n;
	}
no_pairing:
	for (i = 0; i < 2; ++i) {
		int which = -1;
		if (a[i].n && a[i].a[0].score >= opt->T) which = 0;
		if (which >= 0) h[i] = ssqo_reg2aln(opt, idx, s[i].l_seq, s[i].seq, &a[i].a[which]);
		else h[i] = ssqo_reg2aln(opt, idx, s[i].l_seq, s[i].seq, 0);
	}
	if (h[0].rid == h[1].rid && h[0].rid >= 0) { /* top hits happen to form a proper pair */
		int64_t dist;
		int d = infer_dir(idx->bns.l_pac, a[0].a[0].rb, a[1].a[0].rb, &dist);
		if (!pes[d].failed && dist >= pes[d].low && dist <= pes[d].high) extra_flag |= 2;
	}
	ssqo_reg2sam(opt, idx, &s[0], &a[0], 0x41 | extra_flag, &h[1], rg_id);
	ssqo_reg2sam(opt, idx, &s[1], &a[1], 0x81 | extra_flag, &h[0], rg_id);
	ssqo_aln_free(&h[0]); ssqo_aln_free(&h[1]);
	return n;
}

typedef struct {
	const ssqo_opt_t *opt; const ssqo_idx_t *idx; ssqo_read_t *reads; ssqo_alnreg_v *regs;
	const ssqo_pestat_t *pes; int64_t n_processed; const char *rg_id;
} pworker_t;

static void worker_align(void *d, long i, int tid)
{
	pworker_t *w = (pworker_t*)d; (void)tid;
	w->regs[i] = ssqo_align1(w->opt, w->idx, w->reads[i].l_seq, w->reads[i].seq);
}
static void worker_pe(void *d, long i, int tid)
{
	pworker_t *w = (pworker_t*)d; (void)tid;
	sam_pe(w->opt, w->idx, w->pes, (uint64_t)(w->n_processed >> 1) + i, &w->reads[i << 1], &w->regs[i << 1], w->rg_id);
	free(w->regs[i << 1 | 0].a); free(w->regs[i << 1 | 1].a);
}
static void worker_se(void *d, long i, int tid)
{
	pworker_t *w = (pworker_t*)d; (void)tid;
	ssqo_mark_primary_se(w->opt, (int)w->regs[i].n, w->regs[i].a, w->n_processed + i);
	ssqo_reg2sam(w->opt, w->idx, &w->reads[i], &w->regs[i], 0, 0, w->rg_id);
	free(w->regs[i].a);
}

void ssqo_process_seqs(const ssqo_opt_t *opt, const ssqo_idx_t *idx, int64_t n_processed, int n, ssqo_read_t *reads,
                       const ssqo_pestat_t *pes0, const char *rg_id)
{
	ssqo_pestat_t pes[4];
	pworker_t w;
	w.opt = opt; w.idx = idx; w.reads = reads; w.pes = pes; w.n_processed = n_processed; w.rg_id = rg_id;
	w.regs = (ssqo_alnreg_v*)calloc(n, sizeof(ssqo_alnreg_v));
	ssqo_parallel_for(opt->n_threads, n, worker_align, &w);
	if (opt->flag & SSQO_F_PE) {
		if (pes0) memcpy(pes, pes0, sizeof pes);
		else ssqo_pestat(opt, idx->bns.l_pac, n, w.regs, pes);
		ssqo_parallel_for(opt->n_threads, n >> 1, worker_pe, &w);
	} else ssqo_parallel_for(opt->n_threads, n, worker_se, &w);
	free(w.regs);
}

/* ------------------------------------------------------------ `bwa mem` ---- */
static void trim_readno(ssqo_str_t *s)
{
	if (s->l > 2 && s->s[s->l - 2] == '/' && isdigit((unsigned char)s->s[s->l - 1])) s->l -= 2, s->s[s->l] = 0;
}

static void kseq2read(const ssqo_kseq_t *ks, ssqo_read_t *r)
{
	r->name = strdup(ks->name.s);
	r->comment = ks->comment.l ? strdup(ks->comment.s) : 0;
	r->seq = (char*)malloc(ks->seq.l + 1); memcpy(r->seq, ks->seq.s, ks->seq.l + 1);
	r->qual = ks->qual.l ? strdup(ks->qual.s) : 0;
	r->l_seq = (int)ks->seq.l;
	r->sam = 0;
}

/* read until the base count reaches chunk_size AND the read count is even */
static ssqo_read_t *read_batch(int chunk_size, int *n_, ssqo_kseq_t *ks, ssqo_kseq_t *ks2)
{
	int size = 0, m = 0, n = 0;
	ssqo_read_t *seqs = 0;
	while (ssqo_kseq_read(ks) >= 0) {
		if (ks2 && ssqo_kseq_read(ks2) < 0) { fprintf(stderr, "[W::bseq_read] the 2nd file has fewer sequences.\n"); break; }
		if (n + 2 > m) { m = m ? m << 1 : 256; seqs = (ssqo_read_t*)realloc(seqs, m * sizeof(ssqo_read_t)); }
		trim_readno(&ks->name);
		kseq2read(ks, &seqs[n]); seqs[n].id = n; size += seqs[n++].l_seq;
		if (ks2) { trim_readno(&ks2->name); kseq2read(ks2, &seqs[n]); seqs[n].id = n; size += seqs[n++].l_seq; }
		if (size >= chunk_size && (n & 1) == 0) break;
	}
	if (size == 0 && ks2 && ssqo_kseq_read(ks2) >= 0) fprintf(stderr, "[W::bseq_read] the 1st file has fewer sequences.\n");
	*n_ = n;
	return seqs;
}

static char *unescape(char *s)
{
	char *p, *q;
	for (p = q = s; *p; ++p) {
		if (*p == '\\') {
			++p;
			if (*p == 't') *q++ = '\t';
			else if (*p == 'n') *q++ = '\n';
			else if (*p == 'r') *q++ = '\r';
			else if (*p == '\\') *q++ = '\\';
			else if (*p == 0) break;
		} else *q++ = *p;
	}
	*q = 0;
	return s;
}

#define SSQO_BWA_VERSION "0.7.12-r1039"
const char *ssqo_prog = "bwa";

int ssqo_main_mem(int argc, char **argv)
{
	ssqo_opt_t opt;
	ssqo_pestat_t pes[4], *pes0 = 0;
	ssqo_idx_t *idx;
	ssqo_kseq_t *ks, *ks2 = 0;
	char *rg_line = 0, rg_id[256] = {0}, *p;
	int c, i, n, copy_comment = 0, smart_pe = 0;
	int64_t n_processed = 0;
	ssqo_opt_init(&opt);
	memset(pes, 0, sizeof pes);
	pes[0].failed = pes[1].failed = pes[2].failed = pes[3].failed = 1;
	optind = 1;
	while ((c = getopt(argc, argv, "t:pR:I:Cv:")) >= 0) {
		if (c == 't') opt.n_threads = atoi(optarg) > 1 ? atoi(optarg) : 1;
		else if (c == 'p') opt.flag |= SSQO_F_PE, smart_pe = 1;
		else if (c == 'C') copy_comment = 1;
		else if (c == 'v') ;
		else if (c == 'R') {
			if (strstr(optarg, "@RG") != optarg) { fprintf(stderr, "[E::bwa_set_rg] the read group line is not started with @RG\n"); return 1; }
			rg_line = unescape(strdup(optarg));
			if ((p = strstr(rg_line, "\tID:")) == 0) { fprintf(stderr, "[E::bwa_set_rg] no ID at the read group line\n"); return 1; }
			p += 4;
			for (i = 0; p[i] && p[i] != '\t' && p[i] != '\n' && i < 255; ++i) rg_id[i] = p[i];
		} else if (c == 'I') {
			pes0 = pes;
			pes[1].failed = 0;
			pes[1].avg = strtod(optarg, &p);
			pes[1].std = pes[1].avg * .1;
			if (*p != 0 && ispunct((unsigned char)*p) && isdigit((unsigned char)p[1])) pes[1].std = strtod(p + 1, &p);
			pes[1].high = (int)(pes[1].avg + 4. * pes[1].std + .499);
			pes[1].low = (int)(pes[1].avg - 4. * pes[1].std + .499);
			if (pes[1].low < 1) pes[1].low = 1;
			if (*p != 0 && ispunct((unsigned char)*p) && isdigit((unsigned char)p[1])) pes[1].high = (int)(strtod(p + 1, &p) + .499);
			if (*p != 0 && ispunct((unsigned char)*p) && isdigit((unsigned char)p[1])) pes[1].low = (int)(strtod(p + 1, &p) + .499);
		} else return 1;
	}
	if (optind + 1 >= argc || optind + 3 < argc) {
		fprintf(stderr, "Usage: bwa mem [-t INT] [-p] [-C] [-I FLOAT[,FLOAT[,INT[,INT]]]] [-R STR] <idxbase> <in1.fq> [in2.fq]\n");
		return 1;
	}
	if (!(idx = ssqo_idx_load(argv[optind]))) return 1;
	if (!(ks = ssqo_kseq_open(argv[optind + 1]))) { fprintf(stderr, "[E::main_mem] fail to open file `%s'.\n", argv[optind + 1]); return 1; }
	if (optind + 2 < argc) {
		if (opt.flag & SSQO_F_PE) fprintf(stderr, "[W::main_mem] when '-p' is in use, the second query file is ignored.\n");
		else {
			if (!(ks2 = ssqo_kseq_open(argv[optind + 2]))) { fprintf(stderr, "[E::main_mem] fail to open file `%s'.\n", argv[optind + 2]); return 1; }
			opt.flag |= SSQO_F_PE;
		}
	}
	for (i = 0; i < idx->bns.n_seqs; ++i) printf("@SQ\tSN:%s\tLN:%d\n", idx->bns.anns[i].name, idx->bns.anns[i].len);
	if (rg_line) printf("%s\n", rg_line);
	printf("@PG\tID:bwa\tPN:bwa\tVN:%s\tCL:%s", SSQO_BWA_VERSION, ssqo_prog);
	for (i = 0; i < argc; ++i) printf(" %s", argv[i]);
	printf("\n");
	for (;;) {
		ssqo_read_t *seqs = read_batch(opt.chunk_size * opt.n_threads, &n, ks, ks2);
		if (n == 0) { free(seqs); break; }
		if (!copy_comment) for (i = 0; i < n; ++i) { free(seqs[i].comment); seqs[i].comment = 0; }
		fprintf(stderr, "[M::process] read %d sequences (%ld bp)...\n", n, ({ long t = 0; for (i = 0; i < n; ++i) t += seqs[i].l_seq; t; }));
		if (smart_pe) { /* interleaved input: adjacent equal names are pairs, the rest single-end */
			int n_se = 0, n_pe = 0, has_last;
			ssqo_read_t *se = (ssqo_read_t*)malloc(n * sizeof(ssqo_read_t)), *pe = (ssqo_read_t*)malloc(n * sizeof(ssqo_read_t));
			ssqo_opt_t tmp = opt;
			for (i = 1, has_last = 1; i < n; ++i) {
				if (has_last) {
					if (strcmp(seqs[i].name, seqs[i - 1].name) == 0) { pe[n_pe++] = seqs[i - 1]; pe[n_pe++] = seqs[i]; has_last = 0; }
					else se[n_se++] = seqs[i - 1];
				} else has_last = 1;
			}
			if (has_last) se[n_se++] = seqs[i - 1];
			fprintf(stderr, "[M::process] %d single-end sequences; %d paired-end sequences\n", n_se, n_pe);
			if (n_se) {
				tmp.flag &= ~SSQO_F_PE;
				ssqo_process_seqs(&tmp, idx, n_processed, n_se, se, 0, rg_id);
				for (i = 0; i < n_se; ++i) seqs[se[i].id].sam = se[i].sam;
			}
			if (n_pe) {
				tmp.flag |= SSQO_F_PE;
				ssqo_process_seqs(&tmp, idx, n_processed + n_se, n_pe, pe, pes0, rg_id);
				for (i = 0; i < n_pe; ++i) seqs[pe[i].id].sam = pe[i].sam;
			}
			free(se); free(pe);
		} else ssqo_process_seqs(&opt, idx, n_processed, n, seqs, pes0, rg_id);
		n_processed += n;
		for (i = 0; i < n; ++i) {
			if (seqs[i].sam) fputs(seqs[i].sam, stdout);
			free(seqs[i].name); free(seqs[i].comment); free(seqs[i].seq); free(seqs[i].qual); free(seqs[i].sam);
		}
		free(seqs);
	}
	fflush(stdout);
	ssqo_kseq_close(ks); if (ks2) ssqo_kseq_close(ks2);
	ssqo_idx_destroy(idx);
	free(rg_line);
	return 0;
}
