/*
 * ssqo_bwt.c — ORACLE (test infrastructure): FM-index occ / bidirectional extension / SMEM search /
 * SA lookup.  SURVEY.md §8a rows a4, a5; called from inside `$BWA mem`
 * (speedseq/bin/speedseq:438,468).  Upstream names (not in tree): bwt_occ4, bwt_2occ4,
 * bwt_extend, bwt_smem1a, bwt_seed_strategy1, bwt_invPsi, bwt_sa.  Layout of the occ-interleaved
 * BWT is the one verified against the reference goldens (SURVEY.md §8c).
 */
#include <stdlib.h>
#include <string.h>
#include "ssqo.h"

__thread ssqo_counters_t ssqo_cnt;

/* one 64-byte block = u64 occ[4] + u32 w[8] (16 symbols per word, MSB first) */
static inline const uint32_t *blk(const ssqo_bwt_t *b, uint64_t k) { return b->bwt + ((k >> 7) << 4); }

static inline int bwt_sym(const ssqo_bwt_t *b, uint64_t k) /* k in the '$'-less coordinate */
{
	const uint32_t *p = blk(b, k) + 8;
	return p[(k & 0x7f) >> 4] >> ((~k & 0xf) << 1) & 3;
}

/* number of each symbol in rows [0,k] of the (n+1)-row matrix, '$' not counted */
void ssqo_occ4(const ssqo_bwt_t *b, uint64_t k, uint64_t cnt[4])
{
	const uint32_t *p;
	uint64_t kk, r, i;
	if (k == (uint64_t)-1) { memset(cnt, 0, 32); return; }
	kk = k - (k >= b->primary);
	p = blk(b, kk);
	++ssqo_cnt.n_occblk;
	memcpy(cnt, p, 32);
	p += 8;
	r = kk & 0x7f; /* count symbols at in-block offsets 0..r */
	for (i = 0; i <= r; ++i) ++cnt[p[i >> 4] >> ((~i & 0xf) << 1) & 3];
}

uint64_t ssqo_occ(const ssqo_bwt_t *b, uint64_t k, int c)
{
	uint64_t cnt[4];
	if (k == b->seq_len) return b->L2[c + 1] - b->L2[c];
	ssqo_occ4(b, k, cnt);
	return cnt[c];
}

void ssqo_extend(const ssqo_bwt_t *b, const ssqo_intv_t *ik, ssqo_intv_t ok[4], int is_back)
{
	uint64_t tk[4], tl[4];
	int i, f = !is_back;
	++ssqo_cnt.n_extend;
	ssqo_occ4(b, ik->x[f] - 1, tk);
	ssqo_occ4(b, ik->x[f] - 1 + ik->x[2], tl);
	for (i = 0; i < 4; ++i) {
		ok[i].x[f] = b->L2[i] + 1 + tk[i];
		ok[i].x[2] = tl[i] - tk[i];
	}
	ok[3].x[is_back] = ik->x[is_back] + (ik->x[f] <= b->primary && ik->x[f] + ik->x[2] - 1 >= b->primary);
	ok[2].x[is_back] = ok[3].x[is_back] + ok[3].x[2];
	ok[1].x[is_back] = ok[2].x[is_back] + ok[2].x[2];
	ok[0].x[is_back] = ok[1].x[is_back] + ok[1].x[2];
}

static inline void set_intv(const ssqo_bwt_t *b, int c, ssqo_intv_t *ik)
{
	ik->x[0] = b->L2[c] + 1; ik->x[2] = b->L2[c + 1] - b->L2[c]; ik->x[1] = b->L2[3 - c] + 1; ik->info = 0;
}

static inline void v_push(ssqo_intv_v *v, const ssqo_intv_t *x)
{
	if (v->n == v->m) { v->m = v->m ? v->m << 1 : 16; v->a = (ssqo_intv_t*)realloc(v->a, v->m * sizeof(ssqo_intv_t)); }
	v->a[v->n++] = *x;
}

static void v_reverse(ssqo_intv_v *v)
{
	size_t i;
	for (i = 0; i < v->n >> 1; ++i) { ssqo_intv_t t = v->a[i]; v->a[i] = v->a[v->n - 1 - i]; v->a[v->n - 1 - i] = t; }
}

/* all super-maximal exact matches covering query position x; returns where the next search starts */
int ssqo_smem1(const ssqo_bwt_t *b, int len, const uint8_t *q, int x, int min_intv, ssqo_intv_v *mem, ssqo_intv_v tmp[2])
{
	int i, j, c, ret;
	ssqo_intv_t ik, ok[4];
	ssqo_intv_v *prev = &tmp[0], *curr = &tmp[1], *swap;
	mem->n = 0;
	if (q[x] > 3) return x + 1;
	if (min_intv < 1) min_intv = 1;
	set_intv(b, q[x], &ik);
	ik.info = x + 1;
	for (i = x + 1, curr->n = 0; i < len; ++i) { /* forward extension, remember every size change */
		if (q[i] < 4) {
			c = 3 - q[i];
			ssqo_extend(b, &ik, ok, 0);
			if (ok[c].x[2] != ik.x[2]) {
				v_push(curr, &ik);
				if (ok[c].x[2] < (uint64_t)min_intv) break;
			}
			ik = ok[c]; ik.info = i + 1;
		} else { v_push(curr, &ik); break; }
	}
	if (i == len) v_push(curr, &ik);
	v_reverse(curr); /* longest match first */
	ret = (int)curr->a[0].info;
	swap = curr; curr = prev; prev = swap;
	for (i = x - 1; i >= -1; --i) { /* backward extension of the whole set */
		c = i < 0 ? -1 : q[i] < 4 ? q[i] : -1;
		for (j = 0, curr->n = 0; j < (int)prev->n; ++j) {
			ssqo_intv_t *p = &prev->a[j];
			if (c >= 0) ssqo_extend(b, p, ok, 1);
			if (c < 0 || ok[c].x[2] < (uint64_t)min_intv) {
				if (curr->n == 0) { /* no longer match survives: p is maximal on the left */
					if (mem->n == 0 || (uint64_t)(i + 1) < mem->a[mem->n - 1].info >> 32) {
						ik = *p; ik.info |= (uint64_t)(i + 1) << 32;
						v_push(mem, &ik);
					}
				}
			} else if (curr->n == 0 || ok[c].x[2] != curr->a[curr->n - 1].x[2]) {
				ok[c].info = p->info;
				v_push(curr, &ok[c]);
			}
		}
		if (curr->n == 0) break;
		swap = curr; curr = prev; prev = swap;
	}
	v_reverse(mem); /* sorted by start */
	return ret;
}

int ssqo_seed_strategy1(const ssqo_bwt_t *b, int len, const uint8_t *q, int x, int min_len, int max_intv, ssqo_intv_t *mem)
{
	int i, c;
	ssqo_intv_t ik, ok[4];
	memset(mem, 0, sizeof(*mem));
	if (q[x] > 3) return x + 1;
	set_intv(b, q[x], &ik);
	for (i = x + 1; i < len; ++i) {
		if (q[i] < 4) {
			c = 3 - q[i];
			ssqo_extend(b, &ik, ok, 0);
			if (ok[c].x[2] < (uint64_t)max_intv && i - x >= min_len) {
				*mem = ok[c];
				mem->info = (uint64_t)x << 32 | (uint32_t)(i + 1);
				return i + 1;
			}
			ik = ok[c];
		} else return i + 1;
	}
	return len;
}

static inline uint64_t inv_psi(const ssqo_bwt_t *b, uint64_t k)
{
	uint64_t x = k - (k > b->primary);
	int c = bwt_sym(b, x);
	x = b->L2[c] + ssqo_occ(b, k, c);
	return k == b->primary ? 0 : x;
}

uint64_t ssqo_sa(const ssqo_bwt_t *b, uint64_t k)
{
	uint64_t sa = 0, mask = b->sa_intv - 1;
	++ssqo_cnt.n_sa;
	while (k & mask) { ++sa; ++ssqo_cnt.n_sa_steps; k = inv_psi(b, k); }
	return sa + b->sa[k / b->sa_intv];
}
