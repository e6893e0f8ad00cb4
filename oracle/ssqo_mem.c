/*
 * ssqo_mem.c — ORACLE (test infrastructure): single-end core of BWA-MEM.
 * SURVEY.md §8a rows a4-a9, a13-a15: seeding passes, chaining, chain filter, seed extension,
 * de-duplication/patching, primary marking, MAPQ, CIGAR/NM/MD and SAM text.
 * Reference call site: `$BWA mem -t T [-p] -R RG REF FQ` at speedseq/bin/speedseq:438,468
 * (every scoring option at its default).  Upstream names (not in tree): mem_collect_intv,
 * mem_chain, mem_chain_flt, mem_chain2aln, mem_sort_dedup_patch, mem_patch_reg,
 * mem_mark_primary_se, mem_approx_mapq_se, bwa_gen_cigar2, mem_reg2aln, mem_aln2sam, mem_gen_alt.
 * ALT-contig handling is omitted: `speedseq align` never supplies a .alt file, so is_alt == 0.
 */
#include <stdlib.h>
#include <string.h>
#include <math.h>
#include <limits.h>
#include <assert.h>
#include "ssqo.h"
#include "ssqo_kseq.h"
#include "ssqo_sort.h"
#include "ssqo_mem.h"

#define LT_INTV(a, b) ((a).info < (b).info)
SSQO_SORT_INIT(intv, ssqo_intv_t, LT_INTV)
#define LT_U64(a, b) ((a) < (b))
SSQO_SORT_INIT(u64, uint64_t, LT_U64)
#define LT_FLT(a, b) ((a).w > (b).w)
SSQO_SORT_INIT(flt, ssqo_chain_t, LT_FLT)
#define LT_ARS2(a, b) ((a).re < (b).re)
SSQO_SORT_INIT(ars2, ssqo_alnreg_t, LT_ARS2)
#define LT_ARS(a, b) ((a).score > (b).score || ((a).score == (b).score && ((a).rb < (b).rb || ((a).rb == (b).rb && (a).qb < (b).qb))))
SSQO_SORT_INIT(ars, ssqo_alnreg_t, LT_ARS)
#define LT_ARSH(a, b) ((a).score > (b).score || ((a).score == (b).score && ((a).is_alt < (b).is_alt || ((a).is_alt == (b).is_alt && (a).hash < (b).hash))))
SSQO_SORT_INIT(arsh, ssqo_alnreg_t, LT_ARSH)

void ssqo_sort_u64(size_t n, uint64_t *a) { ssqo_introsort_u64(n, a); }

void ssqo_opt_init(ssqo_opt_t *o)
{
	int i, j, k;
	memset(o, 0, sizeof(*o));
	o->a = 1; o->b = 4; o->o_del = o->o_ins = 6; o->e_del = o->e_ins = 1;
	o->w = 100; o->T = 30; o->zdrop = 100; o->pen_unpaired = 17; o->pen_clip5 = o->pen_clip3 = 5;
	o->max_mem_intv = 20; o->min_seed_len = 19; o->split_width = 10; o->max_occ = 500;
	o->max_chain_gap = 10000; o->max_ins = 10000; o->mask_level = 0.50f; o->drop_ratio = 0.50f;
	o->XA_drop_ratio = 0.80f; o->split_factor = 1.5f; o->chunk_size = 10000000; o->n_threads = 1;
	o->max_XA_hits = 5; o->max_XA_hits_alt = 200; o->max_matesw = 50; o->mask_level_redun = 0.95f;
	o->min_chain_weight = 0; o->max_chain_extend = 1 << 30;
	o->mapQ_coef_len = 50; o->mapQ_coef_fac = (int)log(o->mapQ_coef_len); /* an int field upstream: ln(50) truncates to 3 */
	for (i = k = 0; i < 4; ++i) {
		for (j = 0; j < 4; ++j) o->mat[k++] = i == j ? o->a : -o->b;
		o->mat[k++] = -1;
	}
	for (j = 0; j < 5; ++j) o->mat[k++] = -1;
}

uint64_t ssqo_hash64(uint64_t key)
{
	key += ~(key << 32); key ^= (key >> 22);
	key += ~(key << 13); key ^= (key >> 8);
	key += (key << 3);   key ^= (key >> 15);
	key += ~(key << 27); key ^= (key >> 31);
	return key;
}

/* ------------------------------------------------------------ reference ---- */
#define PAC_GET(pac, l) ((pac)[(l) >> 2] >> ((~(l) & 3) << 1) & 3)

int ssqo_pos2rid(const ssqo_bns_t *bns, int64_t pos_f)
{
	int left = 0, mid = 0, right = bns->n_seqs;
	if (pos_f >= bns->l_pac) return -1;
	while (left < right) {
		mid = (left + right) >> 1;
		if (pos_f >= bns->anns[mid].offset) {
			if (mid == bns->n_seqs - 1) break;
			if (pos_f < bns->anns[mid + 1].offset) break;
			left = mid + 1;
		} else right = mid;
	}
	return mid;
}

static inline int64_t depos(const ssqo_bns_t *bns, int64_t pos, int *is_rev)
{
	return (*is_rev = (pos >= bns->l_pac)) ? (bns->l_pac << 1) - 1 - pos : pos;
}

int ssqo_intv2rid(const ssqo_bns_t *bns, int64_t rb, int64_t re)
{
	int is_rev, rid_b, rid_e;
	if (rb < bns->l_pac && re > bns->l_pac) return -2;
	rid_b = ssqo_pos2rid(bns, depos(bns, rb, &is_rev));
	rid_e = rb < re ? ssqo_pos2rid(bns, depos(bns, re - 1, &is_rev)) : rid_b;
	return rid_b == rid_e ? rid_b : -1;
}

uint8_t *ssqo_get_seq(int64_t l_pac, const uint8_t *pac, int64_t beg, int64_t end, int64_t *len)
{
	uint8_t *seq = 0;
	if (end < beg) { int64_t t = end; end = beg; beg = t; }
	if (end > l_pac << 1) end = l_pac << 1;
	if (beg < 0) beg = 0;
	if (beg >= l_pac || end <= l_pac) {
		int64_t k, l = 0;
		*len = end - beg;
		seq = (uint8_t*)malloc(end - beg + 1);
		if (beg >= l_pac) { /* reverse strand: complement of the mirrored forward bases */
			int64_t beg_f = (l_pac << 1) - 1 - end, end_f = (l_pac << 1) - 1 - beg;
			for (k = end_f; k > beg_f; --k) seq[l++] = 3 - PAC_GET(pac, k);
		} else for (k = beg; k < end; ++k) seq[l++] = PAC_GET(pac, k);
	} else *len = 0; /* bridges the forward/reverse boundary */
	return seq;
}

uint8_t *ssqo_fetch_seq(const ssqo_bns_t *bns, const uint8_t *pac, int64_t *beg, int64_t mid, int64_t *end, int *rid)
{
	int64_t far_beg, far_end, len;
	int is_rev;
	uint8_t *seq;
	if (*end < *beg) { int64_t t = *end; *end = *beg; *beg = t; }
	assert(*beg <= mid && mid < *end);
	*rid = ssqo_pos2rid(bns, depos(bns, mid, &is_rev));
	far_beg = bns->anns[*rid].offset;
	far_end = far_beg + bns->anns[*rid].len;
	if (is_rev) { int64_t t = far_beg; far_beg = (bns->l_pac << 1) - far_end; far_end = (bns->l_pac << 1) - t; }
	*beg = *beg > far_beg ? *beg : far_beg;
	*end = *end < far_end ? *end : far_end;
	seq = ssqo_get_seq(bns->l_pac, pac, *beg, *end, &len);
	assert(seq && *end - *beg == len);
	return seq;
}

/* -------------------------------------------------------------- seeding ---- */
static inline void iv_push(ssqo_intv_v *v, const ssqo_intv_t *x)
{
	if (v->n == v->m) { v->m = v->m ? v->m << 1 : 16; v->a = (ssqo_intv_t*)realloc(v->a, v->m * sizeof(ssqo_intv_t)); }
	v->a[v->n++] = *x;
}

void ssqo_collect_intv(const ssqo_opt_t *opt, const ssqo_bwt_t *bwt, int len, const uint8_t *seq, ssqo_intv_v *out)
{
	int i, k, x = 0, old_n;
	int split_len = (int)(opt->min_seed_len * opt->split_factor + .499);
	ssqo_intv_v mem1 = {0, 0, 0}, tmp[2] = {{0, 0, 0}, {0, 0, 0}};
	out->n = 0;
	/* pass 1: all SMEMs */
	while (x < len) {
		if (seq[x] < 4) {
			x = ssqo_smem1(bwt, len, seq, x, 1, &mem1, tmp);
			for (i = 0; i < (int)mem1.n; ++i) {
				ssqo_intv_t *p = &mem1.a[i];
				int slen = (int)((uint32_t)p->info - (p->info >> 32));
				if (slen >= opt->min_seed_len) iv_push(out, p);
			}
		} else ++x;
	}
	/* pass 2: re-seed inside long, nearly unique SMEMs from their midpoint */
	old_n = (int)out->n;
	for (k = 0; k < old_n; ++k) {
		ssqo_intv_t *p = &out->a[k];
		int start = (int)(p->info >> 32), end = (int32_t)p->info;
		if (end - start < split_len || p->x[2] > (uint64_t)opt->split_width) continue;
		ssqo_smem1(bwt, len, seq, (start + end) >> 1, (int)p->x[2] + 1, &mem1, tmp);
		for (i = 0; i < (int)mem1.n; ++i)
			if ((int)((uint32_t)mem1.a[i].info - (mem1.a[i].info >> 32)) >= opt->min_seed_len) iv_push(out, &mem1.a[i]);
	}
	/* pass 3: greedy forward seeds that become rare enough */
	if (opt->max_mem_intv > 0) {
		x = 0;
		while (x < len) {
			if (seq[x] < 4) {
				ssqo_intv_t m;
				x = ssqo_seed_strategy1(bwt, len, seq, x, opt->min_seed_len, (int)opt->max_mem_intv, &m);
				if (m.x[2] > 0) iv_push(out, &m);
			} else ++x;
		}
	}
	ssqo_introsort_intv(out->n, out->a);
	free(mem1.a); free(tmp[0].a); free(tmp[1].a);
}

/* ------------------------------------------------------------- chaining ---- */
/* returns 1 if the seed was absorbed or appended, 0 if a new chain is needed */
static int test_and_merge(const ssqo_opt_t *opt, int64_t l_pac, ssqo_chain_t *c, const ssqo_seed_t *p, int seed_rid)
{
	int64_t qend, rend, x, y;
	const ssqo_seed_t *last = &c->seeds[c->n - 1];
	qend = last->qbeg + last->len;
	rend = last->rbeg + last->len;
	if (seed_rid != c->rid) return 0;
	if (p->qbeg >= c->seeds[0].qbeg && p->qbeg + p->len <= qend && p->rbeg >= c->seeds[0].rbeg && p->rbeg + p->len <= rend) return 1;
	if ((last->rbeg < l_pac || c->seeds[0].rbeg < l_pac) && p->rbeg >= l_pac) return 0;
	x = p->qbeg - last->qbeg;
	y = p->rbeg - last->rbeg;
	if (y >= 0 && x - y <= opt->w && y - x <= opt->w && x - last->len < opt->max_chain_gap && y - last->len < opt->max_chain_gap) {
		if (c->n == c->m) { c->m <<= 1; c->seeds = (ssqo_seed_t*)realloc(c->seeds, c->m * sizeof(ssqo_seed_t)); }
		c->seeds[c->n++] = *p;
		return 1;
	}
	return 0;
}

/*
 * Chains are kept in an array ordered by `pos` (= rbeg of their first seed).  Upstream keeps them
 * in a B-tree; the restatement of its two operations on one ordered sequence is:
 *   lookup(pos): the first chain whose key equals pos, else the last chain with key < pos;
 *   insert     : directly after the slot lookup() returned (at the front if none).
 */
ssqo_chain_v ssqo_mem_chain(const ssqo_opt_t *opt, const ssqo_idx_t *idx, int len, const uint8_t *seq)
{
	const ssqo_bwt_t *bwt = &idx->bwt;
	const ssqo_bns_t *bns = &idx->bns;
	int i, b, e, l_rep;
	int64_t l_pac = bns->l_pac;
	ssqo_chain_v chain = {0, 0, 0};
	ssqo_intv_v mem = {0, 0, 0};
	if (len < opt->min_seed_len) return chain;
	ssqo_collect_intv(opt, bwt, len, seq, &mem);
	for (i = 0, b = e = l_rep = 0; i < (int)mem.n; ++i) { /* query bases covered by over-frequent seeds */
		ssqo_intv_t *p = &mem.a[i];
		int sb = (int)(p->info >> 32), se = (int)(uint32_t)p->info;
		if (p->x[2] <= (uint64_t)opt->max_occ) continue;
		if (sb > e) l_rep += e - b, b = sb, e = se;
		else e = e > se ? e : se;
	}
	l_rep += e - b;
	for (i = 0; i < (int)mem.n; ++i) {
		ssqo_intv_t *p = &mem.a[i];
		int step, count, slen = (int)((uint32_t)p->info - (p->info >> 32));
		int64_t k;
		step = p->x[2] > (uint64_t)opt->max_occ ? (int)(p->x[2] / opt->max_occ) : 1;
		for (k = count = 0; k < (int64_t)p->x[2] && count < opt->max_occ; k += step, ++count) {
			ssqo_seed_t s;
			int rid, to_add = 0;
			long lo, hi, slot;
			s.rbeg = (int64_t)ssqo_sa(bwt, p->x[0] + k);
			s.qbeg = (int)(p->info >> 32);
			s.score = s.len = slen;
			rid = ssqo_intv2rid(bns, s.rbeg, s.rbeg + s.len);
			if (rid < 0) continue; /* spans two contigs or the strand boundary */
			/* lower_bound on pos */
			lo = 0; hi = (long)chain.n;
			while (lo < hi) { long mid = (lo + hi) >> 1; if (chain.a[mid].pos < s.rbeg) lo = mid + 1; else hi = mid; }
			slot = (lo < (long)chain.n && chain.a[lo].pos == s.rbeg) ? lo : lo - 1;
			if (chain.n) {
				if (slot < 0 || !test_and_merge(opt, l_pac, &chain.a[slot], &s, rid)) to_add = 1;
			} else to_add = 1;
			if (to_add) {
				ssqo_chain_t tmp;
				memset(&tmp, 0, sizeof tmp);
				tmp.n = 1; tmp.m = 4;
				tmp.seeds = (ssqo_seed_t*)calloc(tmp.m, sizeof(ssqo_seed_t));
				tmp.seeds[0] = s; tmp.rid = rid; tmp.pos = s.rbeg; tmp.is_alt = 0;
				if (chain.n == chain.m) { chain.m = chain.m ? chain.m << 1 : 8; chain.a = (ssqo_chain_t*)realloc(chain.a, chain.m * sizeof(ssqo_chain_t)); }
				memmove(&chain.a[slot + 2], &chain.a[slot + 1], (chain.n - (size_t)(slot + 1)) * sizeof(ssqo_chain_t));
				chain.a[slot + 1] = tmp;
				++chain.n;
			}
		}
	}
	for (i = 0; i < (int)chain.n; ++i) chain.a[i].frac_rep = (float)l_rep / len;
	free(mem.a);
	return chain;
}

static int chain_weight(const ssqo_chain_t *c)
{
	int64_t end;
	int j, w = 0, tmp;
	for (j = 0, end = 0; j < c->n; ++j) {
		const ssqo_seed_t *s = &c->seeds[j];
		if (s->qbeg >= end) w += s->len;
		else if (s->qbeg + s->len > end) w += (int)(s->qbeg + s->len - end);
		end = end > s->qbeg + s->len ? end : s->qbeg + s->len;
	}
	tmp = w; w = 0;
	for (j = 0, end = 0; j < c->n; ++j) {
		const ssqo_seed_t *s = &c->seeds[j];
		if (s->rbeg >= end) w += s->len;
		else if (s->rbeg + s->len > end) w += (int)(s->rbeg + s->len - end);
		end = end > s->rbeg + s->len ? end : s->rbeg + s->len;
	}
	w = w < tmp ? w : tmp;
	return w < 1 << 30 ? w : (1 << 30) - 1;
}

#define chn_beg(ch) ((ch).seeds->qbeg)
#define chn_end(ch) ((ch).seeds[(ch).n - 1].qbeg + (ch).seeds[(ch).n - 1].len)

int ssqo_chain_flt(const ssqo_opt_t *opt, int n_chn, ssqo_chain_t *a)
{
	int i, k, n_kept = 0, *kept_idx;
	if (n_chn == 0) return 0;
	for (i = k = 0; i < n_chn; ++i) {
		ssqo_chain_t *c = &a[i];
		c->first = -1; c->kept = 0;
		c->w = chain_weight(c);
		if ((int)c->w < opt->min_chain_weight) free(c->seeds);
		else a[k++] = *c;
	}
	n_chn = k;
	ssqo_introsort_flt(n_chn, a);
	kept_idx = (int*)malloc(sizeof(int) * n_chn);
	a[0].kept = 3;
	kept_idx[n_kept++] = 0;
	for (i = 1; i < n_chn; ++i) {
		int large_ovlp = 0;
		for (k = 0; k < n_kept; ++k) {
			int j = kept_idx[k];
			int b_max = chn_beg(a[j]) > chn_beg(a[i]) ? chn_beg(a[j]) : chn_beg(a[i]);
			int e_min = chn_end(a[j]) < chn_end(a[i]) ? chn_end(a[j]) : chn_end(a[i]);
			if (e_min > b_max && (!a[j].is_alt || a[i].is_alt)) {
				int li = chn_end(a[i]) - chn_beg(a[i]);
				int lj = chn_end(a[j]) - chn_beg(a[j]);
				int min_l = li < lj ? li : lj;
				if (e_min - b_max >= min_l * opt->mask_level && min_l < opt->max_chain_gap) {
					large_ovlp = 1;
					if (a[j].first < 0) a[j].first = i; /* remember the first shadowed chain */
					if (a[i].w < a[j].w * opt->drop_ratio && (int)a[j].w - (int)a[i].w >= opt->min_seed_len << 1) break;
				}
			}
		}
		if (k == n_kept) {
			kept_idx[n_kept++] = i;
			a[i].kept = large_ovlp ? 2 : 3;
		}
	}
	for (i = 0; i < n_kept; ++i) {
		ssqo_chain_t *c = &a[kept_idx[i]];
		if (c->first >= 0) a[c->first].kept = 1;
	}
	free(kept_idx);
	for (i = k = 0; i < n_chn; ++i) {
		if (a[i].kept == 0 || a[i].kept == 3) continue;
		if (++k >= opt->max_chain_extend) break;
	}
	for (; i < n_chn; ++i) if (a[i].kept < 3) a[i].kept = 0;
	for (i = k = 0; i < n_chn; ++i) {
		ssqo_chain_t *c = &a[i];
		if (c->kept == 0) free(c->seeds);
		else a[k++] = a[i];
	}
	return k;
}

/* ------------------------------------------------------------ extension ---- */
static inline int cal_max_gap(const ssqo_opt_t *opt, int qlen)
{
	int l_del = (int)((double)(qlen * opt->a - opt->o_del) / opt->e_del + 1.);
	int l_ins = (int)((double)(qlen * opt->a - opt->o_ins) / opt->e_ins + 1.);
	int l = l_del > l_ins ? l_del : l_ins;
	l = l > 1 ? l : 1;
	return l < opt->w << 1 ? l : opt->w << 1;
}

#define MAX_BAND_TRY 2

void ssqo_chain2aln(const ssqo_opt_t *opt, const ssqo_idx_t *idx, int l_query, const uint8_t *query, const ssqo_chain_t *c, ssqo_alnreg_v *av)
{
	const ssqo_bns_t *bns = &idx->bns;
	const uint8_t *pac = idx->pac;
	int i, k, rid, max_off[2], aw[2];
	int64_t l_pac = bns->l_pac, rmax[2], tmp, max = 0;
	const ssqo_seed_t *s;
	uint8_t *rseq = 0;
	uint64_t *srt;
	if (c->n == 0) return;
	rmax[0] = l_pac << 1; rmax[1] = 0;
	for (i = 0; i < c->n; ++i) {
		int64_t b, e;
		const ssqo_seed_t *t = &c->seeds[i];
		b = t->rbeg - (t->qbeg + cal_max_gap(opt, t->qbeg));
		e = t->rbeg + t->len + ((l_query - t->qbeg - t->len) + cal_max_gap(opt, l_query - t->qbeg - t->len));
		rmax[0] = rmax[0] < b ? rmax[0] : b;
		rmax[1] = rmax[1] > e ? rmax[1] : e;
		if (t->len > max) max = t->len;
	}
	rmax[0] = rmax[0] > 0 ? rmax[0] : 0;
	rmax[1] = rmax[1] < l_pac << 1 ? rmax[1] : l_pac << 1;
	if (rmax[0] < l_pac && l_pac < rmax[1]) { /* straddles the strand boundary: keep the seeds' side */
		if (c->seeds[0].rbeg < l_pac) rmax[1] = l_pac;
		else rmax[0] = l_pac;
	}
	rseq = ssqo_fetch_seq(bns, pac, &rmax[0], c->seeds[0].rbeg, &rmax[1], &rid);
	assert(c->rid == rid);
	srt = (uint64_t*)malloc(c->n * 8);
	for (i = 0; i < c->n; ++i) srt[i] = (uint64_t)c->seeds[i].score << 32 | (uint32_t)i;
	ssqo_introsort_u64(c->n, srt);
	for (k = c->n - 1; k >= 0; --k) {
		ssqo_alnreg_t *a;
		s = &c->seeds[(uint32_t)srt[k]];
		for (i = 0; i < (int)av->n; ++i) { /* is this seed already explained by an earlier hit? */
			ssqo_alnreg_t *p = &av->a[i];
			int64_t rd;
			int qd, w, max_gap;
			if (s->rbeg < p->rb || s->rbeg + s->len > p->re || s->qbeg < p->qb || s->qbeg + s->len > p->qe) continue;
			if (s->len - p->seedlen0 > .1 * l_query) continue;
			qd = s->qbeg - p->qb; rd = s->rbeg - p->rb;
			max_gap = cal_max_gap(opt, qd < rd ? qd : (int)rd);
			w = max_gap < p->w ? max_gap : p->w;
			if (qd - rd < w && rd - qd < w) break;
			qd = p->qe - (s->qbeg + s->len); rd = p->re - (s->rbeg + s->len);
			max_gap = cal_max_gap(opt, qd < rd ? qd : (int)rd);
			w = max_gap < p->w ? max_gap : p->w;
			if (qd - rd < w && rd - qd < w) break;
		}
		if (i < (int)av->n) { /* yes, unless a long overlapping seed of this chain sits on another diagonal */
			for (i = k + 1; i < c->n; ++i) {
				const ssqo_seed_t *t;
				if (srt[i] == 0) continue;
				t = &c->seeds[(uint32_t)srt[i]];
				if (t->len < s->len * .95) continue;
				if (s->qbeg <= t->qbeg && s->qbeg + s->len - t->qbeg >= s->len >> 2 && t->qbeg - s->qbeg != t->rbeg - s->rbeg) break;
				if (t->qbeg <= s->qbeg && t->qbeg + t->len - s->qbeg >= s->len >> 2 && s->qbeg - t->qbeg != s->rbeg - t->rbeg) break;
			}
			if (i == c->n) { srt[k] = 0; continue; }
		}
		if (av->n == av->m) { av->m = av->m ? av->m << 1 : 4; av->a = (ssqo_alnreg_t*)realloc(av->a, av->m * sizeof(ssqo_alnreg_t)); }
		a = &av->a[av->n++];
		memset(a, 0, sizeof(*a));
		a->w = aw[0] = aw[1] = opt->w;
		a->score = a->truesc = -1;
		a->rid = c->rid;
		if (s->qbeg) { /* left extension on reversed prefixes */
			uint8_t *rs, *qs;
			int qle, tle, gtle, gscore;
			qs = (uint8_t*)malloc(s->qbeg);
			for (i = 0; i < s->qbeg; ++i) qs[i] = query[s->qbeg - 1 - i];
			tmp = s->rbeg - rmax[0];
			rs = (uint8_t*)malloc(tmp + 1);
			for (i = 0; i < tmp; ++i) rs[i] = rseq[tmp - 1 - i];
			for (i = 0; i < MAX_BAND_TRY; ++i) {
				int prev = a->score;
				aw[0] = opt->w << i;
				a->score = ssqo_ksw_extend2(s->qbeg, qs, (int)tmp, rs, 5, opt->mat, opt->o_del, opt->e_del, opt->o_ins, opt->e_ins, aw[0], opt->pen_clip5, opt->zdrop, s->len * opt->a, &qle, &tle, &gtle, &gscore, &max_off[0]);
				if (a->score == prev || max_off[0] < (aw[0] >> 1) + (aw[0] >> 2)) break;
			}
			if (gscore <= 0 || gscore <= a->score - opt->pen_clip5) { /* local end */
				a->qb = s->qbeg - qle; a->rb = s->rbeg - tle;
				a->truesc = a->score;
			} else { /* reach the query start */
				a->qb = 0; a->rb = s->rbeg - gtle;
				a->truesc = gscore;
			}
			free(qs); free(rs);
		} else a->score = a->truesc = s->len * opt->a, a->qb = 0, a->rb = s->rbeg;
		if (s->qbeg + s->len != l_query) { /* right extension */
			int qle, tle, qe, re, gtle, gscore, sc0 = a->score;
			qe = s->qbeg + s->len;
			re = (int)(s->rbeg + s->len - rmax[0]);
			assert(re >= 0);
			for (i = 0; i < MAX_BAND_TRY; ++i) {
				int prev = a->score;
				aw[1] = opt->w << i;
				a->score = ssqo_ksw_extend2(l_query - qe, query + qe, (int)(rmax[1] - rmax[0] - re), rseq + re, 5, opt->mat, opt->o_del, opt->e_del, opt->o_ins, opt->e_ins, aw[1], opt->pen_clip3, opt->zdrop, sc0, &qle, &tle, &gtle, &gscore, &max_off[1]);
				if (a->score == prev || max_off[1] < (aw[1] >> 1) + (aw[1] >> 2)) break;
			}
			if (gscore <= 0 || gscore <= a->score - opt->pen_clip3) {
				a->qe = qe + qle; a->re = rmax[0] + re + tle;
				a->truesc += a->score - sc0;
			} else {
				a->qe = l_query; a->re = rmax[0] + re + gtle;
				a->truesc += gscore - sc0;
			}
		} else a->qe = l_query, a->re = s->rbeg + s->len;
		for (i = 0, a->seedcov = 0; i < c->n; ++i) {
			const ssqo_seed_t *t = &c->seeds[i];
			if (t->qbeg >= a->qb && t->qbeg + t->len <= a->qe && t->rbeg >= a->rb && t->rbeg + t->len <= a->re) a->seedcov += t->len;
		}
		a->w = aw[0] > aw[1] ? aw[0] : aw[1];
		a->seedlen0 = s->len;
		a->frac_rep = c->frac_rep;
	}
	free(srt); free(rseq);
}

/* ------------------------------------------------------- CIGAR / NM / MD ---- */
typedef struct { size_t l, m; char *s; } sb_t;
static inline void sb_reserve(sb_t *b, size_t add)
{
	if (b->l + add + 1 > b->m) { b->m = (b->l + add + 1) * 2; if (b->m < 64) b->m = 64; b->s = (char*)realloc(b->s, b->m); }
}
static inline void sb_putc(sb_t *b, int c) { sb_reserve(b, 1); b->s[b->l++] = (char)c; b->s[b->l] = 0; }
static inline void sb_putsn(sb_t *b, const char *s, size_t n) { sb_reserve(b, n); memcpy(b->s + b->l, s, n); b->l += n; b->s[b->l] = 0; }
static inline void sb_puts(sb_t *b, const char *s) { sb_putsn(b, s, strlen(s)); }
static inline void sb_putl(sb_t *b, long long v)
{
	char buf[32]; int i = 0; unsigned long long x = v < 0 ? -(unsigned long long)v : (unsigned long long)v;
	do { buf[i++] = (char)('0' + x % 10); x /= 10; } while (x);
	if (v < 0) buf[i++] = '-';
	sb_reserve(b, i);
	while (i > 0) b->s[b->l++] = buf[--i];
	b->s[b->l] = 0;
}

/* global alignment of query[0,l_query) to ref [rb,re); returns CIGAR; MD string (if asked) in *md (malloc'd) */
uint32_t *ssqo_gen_cigar2(const int8_t mat[25], int o_del, int e_del, int o_ins, int e_ins, int w_, int64_t l_pac, const uint8_t *pac,
                          int l_query, uint8_t *query, int64_t rb, int64_t re, int *score, int *n_cigar, int *NM, char **md)
{
	uint32_t *cigar = 0;
	uint8_t tmp, *rseq;
	int i;
	int64_t rlen;
	if (n_cigar) *n_cigar = 0;
	if (NM) *NM = -1;
	if (md) *md = 0;
	if (l_query <= 0 || rb >= re || (rb < l_pac && re > l_pac)) return 0;
	rseq = ssqo_get_seq(l_pac, pac, rb, re, &rlen);
	if (re - rb != rlen) goto done;
	if (rb >= l_pac) { /* reverse both so that gaps end up left-aligned on the forward strand */
		for (i = 0; i < l_query >> 1; ++i) tmp = query[i], query[i] = query[l_query - 1 - i], query[l_query - 1 - i] = tmp;
		for (i = 0; i < rlen >> 1; ++i) tmp = rseq[i], rseq[i] = rseq[rlen - 1 - i], rseq[rlen - 1 - i] = tmp;
	}
	if (l_query == re - rb && w_ == 0) { /* ungapped */
		if (n_cigar) { cigar = (uint32_t*)malloc(4); cigar[0] = (uint32_t)l_query << 4 | 0; *n_cigar = 1; }
		for (i = 0, *score = 0; i < l_query; ++i) *score += mat[rseq[i] * 5 + query[i]];
	} else {
		int w, max_gap, max_ins, max_del, min_w;
		max_ins = (int)((double)(((l_query + 1) >> 1) * mat[0] - o_ins) / e_ins + 1.);
		max_del = (int)((double)(((l_query + 1) >> 1) * mat[0] - o_del) / e_del + 1.);
		max_gap = max_ins > max_del ? max_ins : max_del;
		max_gap = max_gap > 1 ? max_gap : 1;
		w = (max_gap + abs((int)rlen - l_query) + 1) >> 1;
		w = w < w_ ? w : w_;
		min_w = abs((int)rlen - l_query) + 3;
		w = w > min_w ? w : min_w;
		*score = ssqo_ksw_global2(l_query, query, (int)rlen, rseq, 5, mat, o_del, e_del, o_ins, e_ins, w, n_cigar, n_cigar ? &cigar : 0);
	}
	if (NM && n_cigar) {
		int k, x, y, u, n_mm = 0, n_gap = 0;
		sb_t str = {0, 0, 0};
		const char *int2base = rb < l_pac ? "ACGTN" : "TGCAN";
		for (k = 0, x = y = u = 0; k < *n_cigar; ++k) {
			int op = cigar[k] & 0xf, len = (int)(cigar[k] >> 4);
			if (op == 0) {
				for (i = 0; i < len; ++i) {
					if (query[x + i] != rseq[y + i]) { sb_putl(&str, u); sb_putc(&str, int2base[rseq[y + i]]); ++n_mm; u = 0; }
					else ++u;
				}
				x += len; y += len;
			} else if (op == 2) {
				if (k > 0 && k < *n_cigar - 1) { /* terminal deletions are squeezed out later */
					sb_putl(&str, u); sb_putc(&str, '^');
					for (i = 0; i < len; ++i) sb_putc(&str, int2base[rseq[y + i]]);
					u = 0; n_gap += len;
				}
				y += len;
			} else if (op == 1) x += len, n_gap += len;
		}
		sb_putl(&str, u);
		*NM = n_mm + n_gap;
		if (md) *md = str.s; else free(str.s);
	}
	if (rb >= l_pac)
		for (i = 0; i < l_query >> 1; ++i) tmp = query[i], query[i] = query[l_query - 1 - i], query[l_query - 1 - i] = tmp;
done:
	free(rseq);
	return cigar;
}

/* --------------------------------------------------------- dedup / patch ---- */
#define PATCH_MAX_R_BW 0.05f
#define PATCH_MIN_SC_RATIO 0.90f

static int patch_reg(const ssqo_opt_t *opt, const ssqo_idx_t *idx, uint8_t *query, const ssqo_alnreg_t *a, const ssqo_alnreg_t *b, int *_w)
{
	int w, score, q_s, r_s;
	double r;
	if (idx == 0 || query == 0) return 0;
	assert(a->rid == b->rid && a->rb <= b->rb);
	if (a->rb < idx->bns.l_pac && b->rb >= idx->bns.l_pac) return 0;
	if (a->qb >= b->qb || a->qe >= b->qe || a->re >= b->re) return 0; /* not colinear */
	w = (int)((a->re - b->rb) - (a->qe - b->qb));
	w = w > 0 ? w : -w;
	r = (double)(a->re - b->rb) / (b->re - a->rb) - (double)(a->qe - b->qb) / (b->qe - a->qb);
	r = r > 0. ? r : -r;
	if (a->re < b->rb || a->qe < b->qb) {
		if (w > opt->w << 1 || r >= PATCH_MAX_R_BW) return 0;
	} else if (w > opt->w << 2 || r >= PATCH_MAX_R_BW * 2) return 0;
	w += a->w + b->w;
	w = w < opt->w << 2 ? w : opt->w << 2;
	ssqo_gen_cigar2(opt->mat, opt->o_del, opt->e_del, opt->o_ins, opt->e_ins, w, idx->bns.l_pac, idx->pac, b->qe - a->qb, query + a->qb, a->rb, b->re, &score, 0, 0, 0);
	q_s = (int)((double)(b->qe - a->qb) / ((b->qe - b->qb) + (a->qe - a->qb)) * (b->score + a->score) + .499);
	r_s = (int)((double)(b->re - a->rb) / ((b->re - b->rb) + (a->re - a->rb)) * (b->score + a->score) + .499);
	if ((double)score / (q_s > r_s ? q_s : r_s) < PATCH_MIN_SC_RATIO) return 0;
	*_w = w;
	return score;
}

int ssqo_sort_dedup_patch(const ssqo_opt_t *opt, const ssqo_idx_t *idx, uint8_t *query, int n, ssqo_alnreg_t *a)
{
	int m, i, j;
	if (n <= 1) return n;
	ssqo_introsort_ars2(n, a); /* by reference END */
	for (i = 0; i < n; ++i) a[i].n_comp = 1;
	for (i = 1; i < n; ++i) {
		ssqo_alnreg_t *p = &a[i];
		if (p->rid != a[i - 1].rid || p->rb >= a[i - 1].re + opt->max_chain_gap) continue;
		for (j = i - 1; j >= 0 && p->rid == a[j].rid && p->rb < a[j].re + opt->max_chain_gap; --j) {
			ssqo_alnreg_t *q = &a[j];
			int64_t or_, oq, mr, mq;
			int score, w;
			if (q->qe == q->qb) continue; /* already excluded */
			or_ = q->re - p->rb;
			oq = q->qb < p->qb ? q->qe - p->qb : p->qe - q->qb;
			mr = q->re - q->rb < p->re - p->rb ? q->re - q->rb : p->re - p->rb;
			mq = q->qe - q->qb < p->qe - p->qb ? q->qe - q->qb : p->qe - p->qb;
			if (or_ > opt->mask_level_redun * mr && oq > opt->mask_level_redun * mq) { /* one of the two is redundant */
				if (p->score < q->score) { p->qe = p->qb; break; }
				else q->qe = q->qb;
			} else if (q->rb < p->rb && (score = patch_reg(opt, idx, query, q, p, &w)) > 0) { /* merge q into p */
				p->n_comp += q->n_comp + 1;
				p->seedcov = p->seedcov > q->seedcov ? p->seedcov : q->seedcov;
				p->sub = p->sub > q->sub ? p->sub : q->sub;
				p->csub = p->csub > q->csub ? p->csub : q->csub;
				p->qb = q->qb; p->rb = q->rb;
				p->truesc = p->score = score;
				p->w = w;
				q->qb = q->qe;
			}
		}
	}
	for (i = 0, m = 0; i < n; ++i)
		if (a[i].qe > a[i].qb) { if (m != i) a[m++] = a[i]; else ++m; }
	n = m;
	ssqo_introsort_ars(n, a);
	for (i = 1; i < n; ++i)
		if (a[i].score == a[i - 1].score && a[i].rb == a[i - 1].rb && a[i].qb == a[i - 1].qb) a[i].qe = a[i].qb;
	for (i = 1, m = 1; i < n; ++i)
		if (a[i].qe > a[i].qb) { if (m != i) a[m++] = a[i]; else ++m; }
	return m;
}

ssqo_alnreg_v ssqo_align1(const ssqo_opt_t *opt, const ssqo_idx_t *idx, int l_seq, char *seq)
{
	int i;
	ssqo_chain_v chn;
	ssqo_alnreg_v regs = {0, 0, 0};
	for (i = 0; i < l_seq; ++i) seq[i] = seq[i] < 4 ? seq[i] : (char)ssqo_nt4[(uint8_t)seq[i]];
	chn = ssqo_mem_chain(opt, idx, l_seq, (uint8_t*)seq);
	chn.n = ssqo_chain_flt(opt, (int)chn.n, chn.a);
	/* mem_flt_chained_seeds is a no-op while 5.5*ln(L) > 0.05*L, i.e. for every read shorter than ~700 bp */
	for (i = 0; i < (int)chn.n; ++i) {
		ssqo_chain2aln(opt, idx, l_seq, (uint8_t*)seq, &chn.a[i], &regs);
		free(chn.a[i].seeds);
	}
	free(chn.a);
	regs.n = ssqo_sort_dedup_patch(opt, idx, (uint8_t*)seq, (int)regs.n, regs.a);
	return regs;
}

/* -------------------------------------------------- primary marking, MAPQ ---- */
int ssqo_mark_primary_se(const ssqo_opt_t *opt, int n, ssqo_alnreg_t *a, int64_t id)
{
	int i, k, tmp, n_z = 0, *z;
	if (n == 0) return 0;
	for (i = 0; i < n; ++i) {
		a[i].sub = a[i].alt_sc = 0; a[i].secondary = a[i].secondary_all = -1;
		a[i].hash = ssqo_hash64(id + i);
	}
	ssqo_introsort_arsh(n, a);
	tmp = opt->a + opt->b;
	tmp = opt->o_del + opt->e_del > tmp ? opt->o_del + opt->e_del : tmp;
	tmp = opt->o_ins + opt->e_ins > tmp ? opt->o_ins + opt->e_ins : tmp;
	z = (int*)malloc(sizeof(int) * n);
	z[n_z++] = 0;
	for (i = 1; i < n; ++i) {
		for (k = 0; k < n_z; ++k) {
			int j = z[k];
			int b_max = a[j].qb > a[i].qb ? a[j].qb : a[i].qb;
			int e_min = a[j].qe < a[i].qe ? a[j].qe : a[i].qe;
			if (e_min > b_max) {
				int min_l = a[i].qe - a[i].qb < a[j].qe - a[j].qb ? a[i].qe - a[i].qb : a[j].qe - a[j].qb;
				if (e_min - b_max >= min_l * opt->mask_level) { /* i is shadowed by j */
					if (a[j].sub == 0) a[j].sub = a[i].score;
					if (a[j].score - a[i].score <= tmp) ++a[j].sub_n;
					break;
				}
			}
		}
		if (k == n_z) z[n_z++] = i;
		else a[i].secondary = z[k];
	}
	free(z);
	for (i = 0; i < n; ++i) a[i].secondary_all = a[i].secondary;
	return n;
}

int ssqo_approx_mapq_se(const ssqo_opt_t *opt, const ssqo_alnreg_t *a)
{
	int mapq, l, sub = a->sub ? a->sub : opt->min_seed_len * opt->a;
	double identity;
	sub = a->csub > sub ? a->csub : sub;
	if (sub >= a->score) return 0;
	l = a->qe - a->qb > a->re - a->rb ? a->qe - a->qb : (int)(a->re - a->rb);
	identity = 1. - (double)(l * opt->a - a->score) / (opt->a + opt->b) / l;
	if (a->score == 0) mapq = 0;
	else {
		double tmp;
		tmp = l < opt->mapQ_coef_len ? 1. : opt->mapQ_coef_fac / log(l);
		tmp *= identity * identity;
		mapq = (int)(6.02 * (a->score - sub) / opt->a * tmp * tmp + .499);
	}
	if (a->sub_n > 0) mapq -= (int)(4.343 * log(a->sub_n + 1) + .499);
	if (mapq > 60) mapq = 60;
	if (mapq < 0) mapq = 0;
	mapq = (int)(mapq * (1. - a->frac_rep) + .499);
	return mapq;
}

/* ------------------------------------------------------------- reg -> aln ---- */
static inline int infer_bw(int l1, int l2, int score, int a, int q, int r)
{
	int w;
	if (l1 == l2 && l1 * a - score < (q + r - a) << 1) return 0; /* equal lengths need at least two gaps */
	w = (int)((double)((l1 < l2 ? l1 : l2) * a - score - q) / r + 2.);
	if (w < abs(l1 - l2)) w = abs(l1 - l2);
	return w;
}

void ssqo_aln_free(ssqo_aln_t *a) { free(a->cigar); free(a->md); free(a->XA); a->cigar = 0; a->md = 0; a->XA = 0; }

ssqo_aln_t ssqo_reg2aln(const ssqo_opt_t *opt, const ssqo_idx_t *idx, int l_query, const char *query_, const ssqo_alnreg_t *ar)
{
	const ssqo_bns_t *bns = &idx->bns;
	ssqo_aln_t a;
	int i, w2, tmp, qb, qe, NM, score, is_rev, last_sc = -(1 << 30);
	int64_t pos, rb, re;
	uint8_t *query;
	memset(&a, 0, sizeof a);
	if (ar == 0 || ar->rb < 0 || ar->re < 0) { a.rid = -1; a.pos = -1; a.flag |= 0x4; return a; }
	qb = ar->qb; qe = ar->qe; rb = ar->rb; re = ar->re;
	query = (uint8_t*)malloc(l_query);
	for (i = 0; i < l_query; ++i) query[i] = query_[i] < 5 ? query_[i] : ssqo_nt4[(uint8_t)query_[i]];
	a.mapq = ar->secondary < 0 ? ssqo_approx_mapq_se(opt, ar) : 0;
	if (ar->secondary >= 0) a.flag |= 0x100;
	tmp = infer_bw(qe - qb, (int)(re - rb), ar->truesc, opt->a, opt->o_del, opt->e_del);
	w2 = infer_bw(qe - qb, (int)(re - rb), ar->truesc, opt->a, opt->o_ins, opt->e_ins);
	w2 = w2 > tmp ? w2 : tmp;
	if (w2 > opt->w) w2 = w2 < ar->w ? w2 : ar->w;
	i = 0; a.cigar = 0; a.md = 0;
	do { /* widen the band until the global score catches up with the extension score */
		free(a.cigar); free(a.md);
		w2 = w2 < opt->w << 2 ? w2 : opt->w << 2;
		a.cigar = ssqo_gen_cigar2(opt->mat, opt->o_del, opt->e_del, opt->o_ins, opt->e_ins, w2, bns->l_pac, idx->pac, qe - qb, &query[qb], rb, re, &score, &a.n_cigar, &NM, &a.md);
		if (score == last_sc || w2 == opt->w << 2) break;
		last_sc = score;
		w2 <<= 1;
	} while (++i < 3 && score < ar->truesc - opt->a);
	a.NM = NM;
	pos = depos(bns, rb < bns->l_pac ? rb : re - 1, &is_rev);
	a.is_rev = is_rev;
	if (a.n_cigar > 0) { /* squeeze out a leading or trailing deletion */
		if ((a.cigar[0] & 0xf) == 2) {
			pos += a.cigar[0] >> 4;
			--a.n_cigar;
			memmove(a.cigar, a.cigar + 1, a.n_cigar * 4);
		} else if ((a.cigar[a.n_cigar - 1] & 0xf) == 2) --a.n_cigar;
	}
	if (qb != 0 || qe != l_query) { /* clipping */
		int clip5 = is_rev ? l_query - qe : qb, clip3 = is_rev ? qb : l_query - qe;
		a.cigar = (uint32_t*)realloc(a.cigar, 4 * (a.n_cigar + 2));
		if (clip5) { memmove(a.cigar + 1, a.cigar, a.n_cigar * 4); a.cigar[0] = (uint32_t)clip5 << 4 | 3; ++a.n_cigar; }
		if (clip3) a.cigar[a.n_cigar++] = (uint32_t)clip3 << 4 | 3;
	}
	a.rid = ssqo_pos2rid(bns, pos);
	assert(a.rid == ar->rid);
	a.pos = pos - bns->anns[a.rid].offset;
	a.score = ar->score; a.sub = ar->sub > ar->csub ? ar->sub : ar->csub;
	free(query);
	return a;
}

static inline int get_rlen(int n_cigar, const uint32_t *cigar)
{
	int k, l;
	for (k = l = 0; k < n_cigar; ++k) { int op = cigar[k] & 0xf; if (op == 0 || op == 2) l += cigar[k] >> 4; }
	return l;
}

/* one SAM line for list[which]; m_ = the mate's primary alignment (or NULL) */
void ssqo_aln2sam(const ssqo_opt_t *opt, const ssqo_bns_t *bns, ssqo_sb_t *str_, const ssqo_read_t *s, int n, const ssqo_aln_t *list, int which, const ssqo_aln_t *m_, const char *rg_id)
{
	sb_t *str = (sb_t*)str_;
	int i;
	ssqo_aln_t ptmp = list[which], *p = &ptmp, mtmp, *m = 0;
	(void)opt;
	if (m_) mtmp = *m_, m = &mtmp;
	p->flag |= m ? 0x1 : 0;
	p->flag |= p->rid < 0 ? 0x4 : 0;
	p->flag |= m && m->rid < 0 ? 0x8 : 0;
	if (p->rid < 0 && m && m->rid >= 0) p->rid = m->rid, p->pos = m->pos, p->is_rev = m->is_rev, p->n_cigar = 0; /* unmapped read sits at its mate */
	if (m && m->rid < 0 && p->rid >= 0) m->rid = p->rid, m->pos = p->pos, m->is_rev = p->is_rev, m->n_cigar = 0;
	p->flag |= p->is_rev ? 0x10 : 0;
	p->flag |= m && m->is_rev ? 0x20 : 0;
	sb_puts(str, s->name); sb_putc(str, '\t');
	sb_putl(str, (p->flag & 0xffff) | (p->flag & 0x10000 ? 0x100 : 0)); sb_putc(str, '\t');
	if (p->rid >= 0) {
		sb_puts(str, bns->anns[p->rid].name); sb_putc(str, '\t');
		sb_putl(str, p->pos + 1); sb_putc(str, '\t');
		sb_putl(str, p->mapq); sb_putc(str, '\t');
		if (p->n_cigar) {
			for (i = 0; i < p->n_cigar; ++i) {
				int c = p->cigar[i] & 0xf;
				if (c == 3 || c == 4) c = which ? 4 : 3; /* supplementary lines are hard-clipped */
				sb_putl(str, p->cigar[i] >> 4); sb_putc(str, "MIDSH"[c]);
			}
		} else sb_putc(str, '*');
	} else sb_putsn(str, "*\t0\t0\t*", 7);
	sb_putc(str, '\t');
	if (m && m->rid >= 0) {
		if (p->rid == m->rid) sb_putc(str, '='); else sb_puts(str, bns->anns[m->rid].name);
		sb_putc(str, '\t');
		sb_putl(str, m->pos + 1); sb_putc(str, '\t');
		if (p->rid == m->rid) {
			int64_t p0 = p->pos + (p->is_rev ? get_rlen(p->n_cigar, p->cigar) - 1 : 0);
			int64_t p1 = m->pos + (m->is_rev ? get_rlen(m->n_cigar, m->cigar) - 1 : 0);
			if (m->n_cigar == 0 || p->n_cigar == 0) sb_putc(str, '0');
			else sb_putl(str, -(p0 - p1 + (p0 > p1 ? 1 : p0 < p1 ? -1 : 0)));
		} else sb_putc(str, '0');
	} else sb_putsn(str, "*\t0\t0", 5);
	sb_putc(str, '\t');
	if (p->flag & 0x100) sb_putsn(str, "*\t*", 3);
	else if (!p->is_rev) {
		int qb = 0, qe = s->l_seq;
		if (p->n_cigar && which) {
			if ((p->cigar[0] & 0xf) == 4 || (p->cigar[0] & 0xf) == 3) qb += p->cigar[0] >> 4;
			if ((p->cigar[p->n_cigar - 1] & 0xf) == 4 || (p->cigar[p->n_cigar - 1] & 0xf) == 3) qe -= p->cigar[p->n_cigar - 1] >> 4;
		}
		for (i = qb; i < qe; ++i) sb_putc(str, "ACGTN"[(int)s->seq[i]]);
		sb_putc(str, '\t');
		if (s->qual) for (i = qb; i < qe; ++i) sb_putc(str, s->qual[i]);
		else sb_putc(str, '*');
	} else {
		int qb = 0, qe = s->l_seq;
		if (p->n_cigar && which) {
			if ((p->cigar[0] & 0xf) == 4 || (p->cigar[0] & 0xf) == 3) qe -= p->cigar[0] >> 4;
			if ((p->cigar[p->n_cigar - 1] & 0xf) == 4 || (p->cigar[p->n_cigar - 1] & 0xf) == 3) qb += p->cigar[p->n_cigar - 1] >> 4;
		}
		for (i = qe - 1; i >= qb; --i) sb_putc(str, "TGCAN"[(int)s->seq[i]]);
		sb_putc(str, '\t');
		if (s->qual) for (i = qe - 1; i >= qb; --i) sb_putc(str, s->qual[i]);
		else sb_putc(str, '*');
	}
	if (p->n_cigar) {
		sb_putsn(str, "\tNM:i:", 6); sb_putl(str, p->NM);
		sb_putsn(str, "\tMD:Z:", 6); sb_puts(str, p->md ? p->md : "");
	}
	if (p->score >= 0) { sb_putsn(str, "\tAS:i:", 6); sb_putl(str, p->score); }
	if (p->sub >= 0) { sb_putsn(str, "\tXS:i:", 6); sb_putl(str, p->sub); }
	if (rg_id && rg_id[0]) { sb_putsn(str, "\tRG:Z:", 6); sb_puts(str, rg_id); }
	if (!(p->flag & 0x100)) {
		for (i = 0; i < n; ++i) if (i != which && !(list[i].flag & 0x100)) break;
		if (i < n) { /* other non-secondary lines of this read */
			sb_putsn(str, "\tSA:Z:", 6);
			for (i = 0; i < n; ++i) {
				const ssqo_aln_t *r = &list[i];
				int k;
				if (i == which || (r->flag & 0x100)) continue;
				sb_puts(str, bns->anns[r->rid].name); sb_putc(str, ',');
				sb_putl(str, r->pos + 1); sb_putc(str, ',');
				sb_putc(str, "+-"[r->is_rev]); sb_putc(str, ',');
				for (k = 0; k < r->n_cigar; ++k) { sb_putl(str, r->cigar[k] >> 4); sb_putc(str, "MIDSH"[r->cigar[k] & 0xf]); }
				sb_putc(str, ','); sb_putl(str, r->mapq);
				sb_putc(str, ','); sb_putl(str, r->NM);
				sb_putc(str, ';');
			}
		}
	}
	if (p->XA) { sb_putsn(str, "\tXA:Z:", 6); sb_puts(str, p->XA); }
	if (s->comment) { sb_putc(str, '\t'); sb_puts(str, s->comment); }
	sb_putc(str, '\n');
}

/* XA strings: secondary hits scoring >= 0.8 x their primary, at most 5 per primary */
char **ssqo_gen_alt(const ssqo_opt_t *opt, const ssqo_idx_t *idx, const ssqo_alnreg_v *a, int l_query, const char *query)
{
	int i, k, r, *cnt, tot;
	sb_t *aln = 0;
	char **XA = 0;
	cnt = (int*)calloc(a->n + 1, sizeof(int));
	for (i = 0, tot = 0; i < (int)a->n; ++i) {
		k = a->a[i].secondary_all;
		r = (k >= 0 && a->a[i].score >= a->a[k].score * (double)opt->XA_drop_ratio) ? k : -1;
		if (r >= 0) ++cnt[r], ++tot;
	}
	if (tot == 0) { free(cnt); return 0; }
	aln = (sb_t*)calloc(a->n, sizeof(sb_t));
	for (i = 0; i < (int)a->n; ++i) {
		ssqo_aln_t t;
		k = a->a[i].secondary_all;
		r = (k >= 0 && a->a[i].score >= a->a[k].score * (double)opt->XA_drop_ratio) ? k : -1;
		if (r < 0) continue;
		if (cnt[r] > opt->max_XA_hits) continue;
		t = ssqo_reg2aln(opt, idx, l_query, query, &a->a[i]);
		sb_puts(&aln[r], idx->bns.anns[t.rid].name);
		sb_putc(&aln[r], ','); sb_putc(&aln[r], "+-"[t.is_rev]); sb_putl(&aln[r], t.pos + 1);
		sb_putc(&aln[r], ',');
		for (k = 0; k < t.n_cigar; ++k) { sb_putl(&aln[r], t.cigar[k] >> 4); sb_putc(&aln[r], "MIDSHN"[t.cigar[k] & 0xf]); }
		sb_putc(&aln[r], ','); sb_putl(&aln[r], t.NM);
		sb_putc(&aln[r], ';');
		ssqo_aln_free(&t);
	}
	XA = (char**)calloc(a->n, sizeof(char*));
	for (k = 0; k < (int)a->n; ++k) XA[k] = aln[k].s;
	free(cnt); free(aln);
	return XA;
}

/* all SAM lines of one read that is NOT written through the paired branch */
void ssqo_reg2sam(const ssqo_opt_t *opt, const ssqo_idx_t *idx, ssqo_read_t *s, ssqo_alnreg_v *a, int extra_flag, const ssqo_aln_t *m, const char *rg_id)
{
	sb_t str = {0, 0, 0};
	ssqo_aln_t *aa = (ssqo_aln_t*)calloc(a->n + 1, sizeof(ssqo_aln_t));
	int k, l, n_aa = 0;
	char **XA = ssqo_gen_alt(opt, idx, a, s->l_seq, s->seq);
	for (k = l = 0; k < (int)a->n; ++k) {
		ssqo_alnreg_t *p = &a->a[k];
		ssqo_aln_t *q;
		if (p->score < opt->T) continue;
		if (p->secondary >= 0) continue; /* no -a: secondaries only appear in XA */
		q = &aa[n_aa++];
		*q = ssqo_reg2aln(opt, idx, s->l_seq, s->seq, p);
		assert(q->rid >= 0);
		q->XA = XA && XA[k] ? strdup(XA[k]) : 0;
		q->flag |= extra_flag;
		if (l) q->flag |= 0x800; /* supplementary (no -M at speedseq:438) */
		if (l && q->mapq > aa[0].mapq) q->mapq = aa[0].mapq;
		++l;
	}
	if (n_aa == 0) {
		ssqo_aln_t t = ssqo_reg2aln(opt, idx, s->l_seq, s->seq, 0);
		t.flag |= extra_flag;
		ssqo_aln2sam(opt, &idx->bns, (ssqo_sb_t*)&str, s, 1, &t, 0, m, rg_id);
	} else {
		for (k = 0; k < n_aa; ++k) ssqo_aln2sam(opt, &idx->bns, (ssqo_sb_t*)&str, s, n_aa, aa, k, m, rg_id);
		for (k = 0; k < n_aa; ++k) ssqo_aln_free(&aa[k]);
	}
	free(aa);
	s->sam = str.s;
	if (XA) { for (k = 0; k < (int)a->n; ++k) free(XA[k]); free(XA); }
}
