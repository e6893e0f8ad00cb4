/* ssqo_bai.c — CPU restatement of `sambamba index` (0.5.9) for coordinate-sorted BAM: TEST INFRASTRUCTURE only, never linked by
 * the product.  It reads the file the way a sequential indexer does — BGZF members one after the other with zlib, records one after
 * the other with the virtual offsets a reader reports — and keeps sambamba's builder state: the previous record, the start of the
 * current chunk (the end of the record before it), one chunk list per bin in a chained hash table with druntime's growth and
 * iteration order, the linear index with C's truncating division, and the per-reference metadata.  Every rule is pinned by the
 * fixtures tests/golden/bai_*.bam(.bai), which the reference's sambamba indexed (tests/golden/make_bai_golden.py).
 * Input the device builder refuses is refused here too (a non-zero return and a message): see the head of
 * speedseq_b200/csrc/ssq_bai.cuh.
 *   int ssqo_bai(const void *bam, size_t n, void **out, size_t *out_len, char *err, size_t err_cap);   free(*out) */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <zlib.h>

typedef struct { uint64_t beg, end; } chunk_t;
typedef struct ent { uint32_t bin; chunk_t *c; int n, m; struct ent *next; } ent_t;
typedef struct { ent_t **b; size_t nb, nodes; } aa_t;                 /* druntime's chained table (uint keys hash to themselves) */

static const size_t PRIMES[] = {31, 97, 389, 1543, 6151, 24593, 98317, 393241, 1572869};

static void aa_init(aa_t *a) { a->nb = 4; a->nodes = 0; a->b = (ent_t**)calloc(4, sizeof(ent_t*)); }
static void aa_append(ent_t **b, size_t nb, ent_t *e) { ent_t **p = &b[e->bin % nb]; while (*p) p = &(*p)->next; e->next = 0; *p = e; }
static ent_t *aa_get(aa_t *a, uint32_t bin)
{
	ent_t *e;
	for (e = a->b[bin % a->nb]; e; e = e->next) if (e->bin == bin) return e;
	e = (ent_t*)calloc(1, sizeof(ent_t)); e->bin = bin;
	aa_append(a->b, a->nb, e);
	if (++a->nodes > a->nb * 4) { /* rehash: the old entries are moved last to first */
		size_t p = 0, k = 0, i, nb;
		ent_t **all = (ent_t**)malloc(a->nodes * sizeof(ent_t*)), **b2, *x;
		while (p + 1 < sizeof PRIMES / sizeof *PRIMES && a->nodes > PRIMES[p]) ++p;
		nb = PRIMES[p];
		for (i = 0; i < a->nb; ++i) for (x = a->b[i]; x; x = x->next) all[k++] = x;
		b2 = (ent_t**)calloc(nb, sizeof(ent_t*));
		while (k) aa_append(b2, nb, all[--k]);
		free(all); free(a->b); a->b = b2; a->nb = nb;
	}
	return e;
}
static void aa_free(aa_t *a) { size_t i; for (i = 0; i < a->nb; ++i) { ent_t *e = a->b[i]; while (e) { ent_t *n = e->next; free(e->c); free(e); e = n; } } free(a->b); a->b = 0; }

typedef struct { char *p; size_t n, cap; } buf_t;
static void put(buf_t *b, const void *p, size_t n) { if (b->n + n > b->cap) { b->cap = (b->n + n) * 2 + 64; b->p = (char*)realloc(b->p, b->cap); } memcpy(b->p + b->n, p, n); b->n += n; }
static void put32(buf_t *b, uint32_t v) { put(b, &v, 4); }
static void put64(buf_t *b, uint64_t v) { put(b, &v, 8); }
static uint32_t rd32(const uint8_t *p) { return p[0] | p[1] << 8 | p[2] << 16 | (uint32_t)p[3] << 24; }

typedef struct {                       /* the builder's state for the current reference */
	aa_t bins;
	uint64_t *lin; size_t lin_n, lin_cap;  /* lin_n: windows written (the largest last window + 1) */
	uint64_t beg_vo, end_vo, mapped, unmapped;
	int have;
} ref_t;

static void lin_touch(ref_t *r, long long w0, long long w1, uint64_t vo) /* windows [w0, w1] */
{
	long long w;
	if (w1 < 0) return;
	if ((size_t)w1 + 1 > r->lin_cap) { size_t c = ((size_t)w1 + 1) * 2; r->lin = (uint64_t*)realloc(r->lin, c * 8); memset(r->lin + r->lin_cap, 0, (c - r->lin_cap) * 8); r->lin_cap = c; }
	for (w = w0; w <= w1; ++w) if (!r->lin[w]) r->lin[w] = vo;
	if ((size_t)w1 + 1 > r->lin_n) r->lin_n = (size_t)w1 + 1;
}
static void add_chunk(ref_t *r, uint32_t bin, uint64_t beg, uint64_t end)
{
	ent_t *e = aa_get(&r->bins, bin);
	if (e->n && (e->c[e->n - 1].end >> 16) == (beg >> 16)) { e->c[e->n - 1].end = end; return; }
	if (e->n == e->m) { e->m = e->m ? e->m * 2 : 4; e->c = (chunk_t*)realloc(e->c, e->m * sizeof(chunk_t)); }
	e->c[e->n].beg = beg; e->c[e->n].end = end; ++e->n;
}
static void dump_ref(buf_t *o, ref_t *r)
{
	size_t i, w;
	uint64_t prev = 0;
	if (!r->have) { put32(o, 0); put32(o, 0); return; }
	put32(o, (uint32_t)(r->bins.nodes + 1));
	for (i = 0; i < r->bins.nb; ++i) {
		const ent_t *e;
		for (e = r->bins.b[i]; e; e = e->next) { int k; put32(o, e->bin); put32(o, (uint32_t)e->n); for (k = 0; k < e->n; ++k) { put64(o, e->c[k].beg); put64(o, e->c[k].end); } }
	}
	put32(o, 37450); put32(o, 2); put64(o, r->beg_vo); put64(o, r->end_vo); put64(o, r->mapped); put64(o, r->unmapped);
	put32(o, (uint32_t)r->lin_n);
	for (w = 0; w < r->lin_n; ++w) { if (!r->lin[w]) r->lin[w] = prev; prev = r->lin[w]; put64(o, r->lin[w]); }
}
static void ref_reset(ref_t *r) { aa_free(&r->bins); aa_init(&r->bins); if (r->lin) memset(r->lin, 0, r->lin_cap * 8); r->lin_n = 0; r->mapped = r->unmapped = 0; r->have = 0; }

#define FAIL(...) do { snprintf(err, err_cap, __VA_ARGS__); rc = 1; goto done; } while (0)

int ssqo_bai(const void *bam, size_t n, void **out, size_t *out_len, char *err, size_t err_cap)
{
	const uint8_t *z = (const uint8_t*)bam;
	uint8_t *text = 0;
	uint64_t *mco = 0, *mto = 0;        /* per member: compressed offset, text offset */
	size_t nm = 0, mcap = 0, tn = 0, c = 0, at, k;
	buf_t o = {0, 0, 0};
	ref_t R;
	int rc = 0, n_ref, cur = -1, i, first = 1, seen_nocoor = 0;
	uint64_t no_coor = 0, chunk_beg = 0, prev_end = 0; /* prev_end: the end of the last record with a reference */
	int32_t prev_pos = 0;
	uint32_t run_bin = 0;
	memset(&R, 0, sizeof R); aa_init(&R.bins);
	*out = 0; *out_len = 0; err[0] = 0;
	/* BGZF, member by member */
	while (c < n) {
		uint32_t xlen, bsize = 0, isize, x; int have = 0; z_stream s; uint8_t *t2;
		if (c + 12 > n || z[c] != 0x1f || z[c + 1] != 0x8b || z[c + 2] != 8 || !(z[c + 3] & 4)) FAIL("not BGZF at compressed byte %zu", c);
		xlen = z[c + 10] | z[c + 11] << 8;
		for (x = 0; x + 4 <= xlen && c + 12 + x + 6 <= n; x += 4 + (z[c + 14 + x] | z[c + 15 + x] << 8))
			if (z[c + 12 + x] == 'B' && z[c + 13 + x] == 'C' && (z[c + 14 + x] | z[c + 15 + x] << 8) == 2) { bsize = z[c + 16 + x] | z[c + 17 + x] << 8; have = 1; break; }
		if (!have || c + bsize + 1 > n || bsize + 1 < 12 + xlen + 8) FAIL("not BGZF (BSIZE) at compressed byte %zu", c);
		isize = rd32(z + c + bsize + 1 - 4);
		if (isize > 65536) FAIL("a member of more than 64 KB at compressed byte %zu", c);
		t2 = (uint8_t*)realloc(text, tn + isize + 1); if (!t2) FAIL("out of memory"); text = t2;
		memset(&s, 0, sizeof s);
		inflateInit2(&s, -15);
		s.next_in = (Bytef*)(z + c + 12 + xlen); s.avail_in = bsize + 1 - 12 - xlen - 8;
		s.next_out = text + tn; s.avail_out = isize + 1;
		x = inflate(&s, Z_FINISH) == Z_STREAM_END && s.total_out == isize && crc32(0, text + tn, isize) == rd32(z + c + bsize + 1 - 8);
		inflateEnd(&s);
		if (!x) FAIL("corrupt BGZF member at compressed byte %zu", c);
		if (nm == mcap) { mcap = mcap ? mcap * 2 : 1024; mco = (uint64_t*)realloc(mco, mcap * 8); mto = (uint64_t*)realloc(mto, mcap * 8); }
		mco[nm] = c; mto[nm] = tn; ++nm;
		tn += isize; c += bsize + 1;
	}
	for (k = 0; k + 1 < nm; ++k) if (mto[k + 1] == mto[k]) FAIL("an empty BGZF member before the last one");
	/* header */
	if (tn < 12 || memcmp(text, "BAM\1", 4)) FAIL("not a BAM file");
	at = 8 + (size_t)rd32(text + 4);
	if (at + 4 > tn) FAIL("truncated header");
	n_ref = (int)rd32(text + at); at += 4;
	for (i = 0; i < n_ref; ++i) { if (at + 4 > tn) FAIL("truncated header"); at += 8 + rd32(text + at); if (at > tn) FAIL("truncated header"); }
	put(&o, "BAI\1", 4); put32(&o, (uint32_t)n_ref);
	/* records */
	k = 0; /* member of the reader */
	while (at < tn) {
		uint32_t bs, bin, flag, ncig, lrn, q; int32_t ref, pos, rlen = 0; uint64_t vb, ve; size_t e;
		if (at + 36 > tn || (bs = rd32(text + at)) < 32 || at + 4 + bs > tn) FAIL("truncated record at text byte %zu", at);
		ref = (int32_t)rd32(text + at + 4); pos = (int32_t)rd32(text + at + 8); lrn = text[at + 12];
		bin = text[at + 14] | text[at + 15] << 8; ncig = text[at + 16] | text[at + 17] << 8; flag = text[at + 18] | text[at + 19] << 8;
		if (36 + lrn + 4 * ncig > 4 + bs) FAIL("malformed record at text byte %zu", at);
		for (q = 0; q < ncig; ++q) { uint32_t v = rd32(text + at + 36 + lrn + 4 * q), op = v & 15; if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) rlen += (int32_t)(v >> 4); }
		e = at + 4 + bs;
		while (k + 1 < nm && mto[k + 1] <= at) ++k; /* the member holding the record's first byte */
		vb = mco[k] << 16 | (at - mto[k]);
		{ size_t j = k; while (j + 1 < nm && mto[j + 1] < e) ++j;  /* and its end: the next member's start at a member border */
		  ve = e - mto[j] < (j + 1 < nm ? mto[j + 1] - mto[j] : tn - mto[j]) ? (mco[j] << 16 | (e - mto[j])) : (j + 1 < nm ? mco[j + 1] : n) << 16; }
		at = e;
		if (ref < -1 || ref >= n_ref) FAIL("refID %d is not a reference of the header", ref);
		if (ref < 0) { ++no_coor; seen_nocoor = 1; if (cur >= 0) R.end_vo = ve; continue; } /* the last reference ends with the file */
		if (seen_nocoor) FAIL("a record without a reference before one with a reference");
		if (pos < 0) FAIL("a record with a reference and no position");
		if ((long long)pos + ((flag & 4) || !rlen ? 1 : rlen) > (1ll << 29)) FAIL("a record past 2^29");
		if (ref < cur || (ref == cur && pos < prev_pos)) FAIL("not coordinate-sorted");
		if (ref != cur) {
			if (cur >= 0) { add_chunk(&R, run_bin, chunk_beg, prev_end); dump_ref(&o, &R); ref_reset(&R); }
			for (i = cur + 1; i < ref; ++i) { put32(&o, 0); put32(&o, 0); }
			cur = ref;
			chunk_beg = first ? vb : prev_end;
			R.have = 1; R.beg_vo = vb; run_bin = bin;
		} else if (bin != run_bin) { add_chunk(&R, run_bin, chunk_beg, prev_end); chunk_beg = prev_end; run_bin = bin; }
		first = 0;
		if (flag & 4) { ++R.unmapped; lin_touch(&R, pos / 16384, pos / 16384, vb); }
		else { ++R.mapped; lin_touch(&R, pos / 16384, ((long long)pos + rlen - 1) / 16384, vb); } /* C division: truncates toward zero */
		R.end_vo = ve; prev_end = ve; prev_pos = pos;
	}
	if (cur >= 0) { add_chunk(&R, run_bin, chunk_beg, prev_end); dump_ref(&o, &R); }
	for (i = cur + 1; i < n_ref; ++i) { put32(&o, 0); put32(&o, 0); }
	put64(&o, no_coor);
done:
	if (rc) free(o.p); else { *out = o.p; *out_len = o.n; }
	aa_free(&R.bins); free(R.lin); free(text); free(mco); free(mto);
	return rc;
}
