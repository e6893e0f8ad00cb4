/* ssqo_merge.c — the checker's sequential restatement of `sambamba merge` (0.5.9) for coordinate-sorted BAM files: each input is
 * read whole with zlib, the merged header is built by sambamba's rules and the records are merged by its heap (D's NWayUnion over
 * a BinaryHeap; the rules are written out at the head of speedseq_b200/csrc/ssq_merge.cuh).  Independent of the device code:
 * plain arrays, its own header parser, hash table and heap.  Refuses what the device refuses.
 *   int ssqo_merge(paths, n, &body, &len, err, err_cap): 0 and the uncompressed merged file (malloc'd), or -1 and a message. */
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <zlib.h>

typedef struct { uint8_t *d; size_t n, r0, nrec; size_t *off; uint64_t *key; size_t next; char *text; size_t lt, refs_at; } in_t;
typedef struct { char **id, **line; uint64_t *h; int n; } tab_t;

static char *g_err; static size_t g_cap;
#define FAIL(...) do { snprintf(g_err, g_cap, __VA_ARGS__); goto fail; } while (0)
static uint32_t u32(const uint8_t *p) { return p[0] | p[1] << 8 | p[2] << 16 | (uint32_t)p[3] << 24; }
static uint64_t key_of(const uint8_t *r)
{
	const int32_t ref = (int32_t)u32(r + 4), pos = (int32_t)u32(r + 8);
	return ref < 0 ? ~0ull : ((uint64_t)(uint32_t)ref << 34 | (uint64_t)(uint32_t)(pos + 1) << 1 | ((r[18] >> 4) & 1));
}
/* sambamba's tag order of an @SQ / @RG / @PG line (no newline) into out */
static void reorder(const char *l, size_t n, char *out)
{
	static const char *sq[] = {"SN", "LN", "AS", "M5", "SP", "UR", 0}, *rg[] = {"ID", "CN", "DS", "DT", "FO", "KS", "LB", "PG", "PI", "PL", "PU", "SM", 0}, *pg[] = {"ID", "PN", "CL", "PP", "VN", 0};
	const char **ord = !strncmp(l, "@SQ", 3) ? sq : !strncmp(l, "@RG", 3) ? rg : pg;
	const char *f[256] = {0}; size_t fl[256] = {0}; int nf = 0, used[256] = {0}, k, i;
	size_t at = 0;
	for (const char *p = l; p < l + n && nf < 256;) { const char *e = memchr(p, '\t', (size_t)(l + n - p)); if (!e) e = l + n; f[nf] = p; fl[nf++] = (size_t)(e - p); p = e + 1; }
	memcpy(out, f[0], fl[0]); at = fl[0];
	for (k = 0; ord[k]; ++k) for (i = 1; i < nf; ++i) if (!used[i] && fl[i] >= 3 && f[i][2] == ':' && !strncmp(f[i], ord[k], 2)) { out[at++] = '\t'; memcpy(out + at, f[i], fl[i]); at += fl[i]; used[i] = 1; }
	for (i = 1; i < nf; ++i) if (!used[i]) { out[at++] = '\t'; memcpy(out + at, f[i], fl[i]); at += fl[i]; }
	out[at] = 0;
}
/* druntime's associative array iteration order over the hashes h[0, n) (4 buckets, > 4 keys per bucket -> the next prime, old
 * keys moved last to first, new keys at their bucket's tail) */
static void aa_order(const uint64_t *h, int n, int *order)
{
	static const size_t primes[] = {4, 31, 97, 389, 1543, 6151, 24593, 98317};
	int *nxt = malloc(sizeof(int) * (n + 1)), *head = 0, *tail = 0, i, k = 0;
	size_t nb = 4, b, p = 0;
	head = malloc(sizeof(int) * 98317); tail = malloc(sizeof(int) * 98317);
	for (b = 0; b < nb; ++b) head[b] = tail[b] = -1;
	for (i = 0; i < n; ++i) {
		b = h[i] % nb; nxt[i] = -1;
		if (tail[b] < 0) head[b] = i; else nxt[tail[b]] = i;
		tail[b] = i;
		if ((size_t)i + 1 > nb * 4) { /* rehash: old buckets last to first, each bucket's keys last to first */
			int *all = malloc(sizeof(int) * (i + 1)), na = 0, j;
			for (b = nb; b--;) { int c = 0, x; for (x = head[b]; x >= 0; x = nxt[x]) ++c; { int *tmp = malloc(sizeof(int) * (c + 1)), t = 0; for (x = head[b]; x >= 0; x = nxt[x]) tmp[t++] = x; while (t--) all[na++] = tmp[t]; free(tmp); } }
			while (p + 1 < sizeof primes / sizeof *primes && (size_t)i + 1 > primes[p]) ++p;
			nb = primes[p];
			for (b = 0; b < nb; ++b) head[b] = tail[b] = -1;
			for (j = 0; j < na; ++j) { const int x = all[j]; b = h[x] % nb; nxt[x] = -1; if (tail[b] < 0) head[b] = x; else nxt[tail[b]] = x; tail[b] = x; }
			free(all);
		}
	}
	for (b = 0; b < nb; ++b) for (i = head[b]; i >= 0; i = nxt[i]) order[k++] = i;
	free(nxt); free(head); free(tail);
}
static in_t *g_in;
static int less_front(int a, int b) { return g_in[b].key[g_in[b].next] < g_in[a].key[g_in[a].next]; } /* comp(a, b) */
static void down(int *h, int n, int i)
{
	for (;;) {
		const int l = 2 * i + 1, r = l + 1; int g, t;
		if (r == n) { if (less_front(h[i], h[l])) { t = h[i]; h[i] = h[l]; h[l] = t; } return; }
		if (r > n) return;
		g = less_front(h[i], h[l]) ? (less_front(h[l], h[r]) ? r : l) : (less_front(h[i], h[r]) ? r : i);
		if (g == i) return;
		t = h[i]; h[i] = h[g]; h[g] = t; i = g;
	}
}

int ssqo_merge(const char **paths, int n, void **body, size_t *len, char *err, size_t err_cap)
{
	in_t *in = calloc((size_t)n + 1, sizeof(in_t));
	tab_t tab[2] = {{0}, {0}};
	char *out = 0, *hd0 = 0, *sq0 = 0, *co = 0, *line = 0;
	size_t olen = 0, ocap = 0, i, colen = 0;
	int k, *h = 0, nh = 0, rc = -1;
	g_err = err; g_cap = err_cap; err[0] = 0; g_in = in;
	if (n < 2) FAIL("merge needs at least two inputs");
	co = calloc(1, 1);
	for (k = 0; k < n; ++k) { /* read, header, records */
		in_t *I = &in[k];
		size_t cap = 1 << 20, at, q;
		uint8_t magic[4] = {0};
		FILE *fp = fopen(paths[k], "rb");
		gzFile z;
		int nr, got;
		char *hd = calloc(1, 1), *sq = calloc(1, 1);
		if (!fp) FAIL("cannot open %s", paths[k]);
		if (fread(magic, 1, 4, fp) != 4 || magic[0] != 0x1f || magic[1] != 0x8b || !(magic[3] & 4)) { fclose(fp); FAIL("%s is not BGZF", paths[k]); }
		fclose(fp);
		z = gzopen(paths[k], "rb");
		I->d = malloc(cap);
		while ((got = gzread(z, I->d + I->n, (unsigned)(cap - I->n))) > 0) { I->n += (size_t)got; if (I->n == cap) I->d = realloc(I->d, cap *= 2); }
		if (got < 0) { gzclose(z); FAIL("%s is not BGZF: corrupt", paths[k]); }
		gzclose(z);
		if (I->n < 12 || memcmp(I->d, "BAM\1", 4)) FAIL("%s: not a BAM file", paths[k]);
		I->lt = u32(I->d + 4); I->text = (char*)I->d + 8; I->refs_at = 8 + I->lt;
		nr = (int)u32(I->d + I->refs_at);
		for (at = I->refs_at + 4, q = 0; q < (size_t)nr; ++q) at += 8 + u32(I->d + at);
		I->r0 = at;
		for (at = I->r0; at + 4 <= I->n; at += 4 + u32(I->d + at)) {
			if (at + 4 + u32(I->d + at) > I->n) break;
			if (u32(I->d + at) < 32) FAIL("%s: record %zu is not a BAM record", paths[k], I->nrec);
			I->off = realloc(I->off, sizeof(size_t) * (I->nrec + 1)); I->key = realloc(I->key, 8 * (I->nrec + 1));
			I->off[I->nrec] = at; I->key[I->nrec] = key_of(I->d + at);
			{ const int32_t ref = (int32_t)u32(I->d + at + 4); if (ref < -1 || ref >= nr) FAIL("%s: record %zu: refID outside the header", paths[k], I->nrec); }
			if (I->nrec && I->key[I->nrec - 1] >> 1 > I->key[I->nrec] >> 1) FAIL("%s: record %zu is not coordinate-sorted", paths[k], I->nrec);
			++I->nrec;
		}
		if (at != I->n) FAIL("%s: a record runs past the end of the file", paths[k]);
		/* header lines */
		for (const char *p = I->text; p < I->text + I->lt && *p;) {
			const char *e = memchr(p, '\n', (size_t)(I->text + I->lt - p));
			const size_t l = e ? (size_t)(e - p) : strnlen(p, (size_t)(I->text + I->lt - p));
			line = realloc(line, 2 * l + 16);
			if (!l) { p += 1; continue; }
			if (!strncmp(p, "@HD", 3)) { hd = realloc(hd, strlen(hd) + l + 2); strncat(hd, p, l); strcat(hd, "\n"); }
			else if (!strncmp(p, "@CO", 3)) { co = realloc(co, colen + l + 2); memcpy(co + colen, p, l); colen += l; co[colen++] = '\n'; co[colen] = 0; }
			else if (!strncmp(p, "@SQ", 3)) { reorder(p, l, line); sq = realloc(sq, strlen(sq) + strlen(line) + 2); strcat(sq, line); strcat(sq, "\n"); }
			else if (!strncmp(p, "@RG", 3) || !strncmp(p, "@PG", 3)) {
				tab_t *T = &tab[p[1] == 'P'];
				const char *id, *ie; int j; uint64_t hv = 0;
				reorder(p, l, line);
				if (!(id = strstr(line, "\tID:"))) FAIL("%s: a line without ID", paths[k]);
				id += 4; ie = strchr(id, '\t'); if (!ie) ie = id + strlen(id);
				for (j = 0; j < T->n; ++j) if (strlen(T->id[j]) == (size_t)(ie - id) && !strncmp(T->id[j], id, (size_t)(ie - id))) break;
				if (j < T->n) { if (strcmp(T->line[j], line)) FAIL("%s: an ID carried by two different lines", paths[k]); }
				else {
					const char *c;
					for (c = id; c < ie; ++c) hv = hv * 11 + (unsigned char)*c;
					T->id = realloc(T->id, sizeof(char*) * (T->n + 1)); T->line = realloc(T->line, sizeof(char*) * (T->n + 1)); T->h = realloc(T->h, 8 * (T->n + 1));
					T->id[T->n] = strndup(id, (size_t)(ie - id)); T->line[T->n] = strdup(line); T->h[T->n++] = hv;
				}
			} else FAIL("%s: a header line that is not merged", paths[k]);
			p += l + (e ? 1 : 0);
		}
		if (!strstr(hd, "\tSO:coordinate")) FAIL("%s: not SO:coordinate", paths[k]);
		if (!k) { hd0 = hd; sq0 = sq; continue; }
		if (strcmp(hd, hd0)) FAIL("the @HD lines differ");
		if (strcmp(sq, sq0) || I->r0 - I->refs_at != in[0].r0 - in[0].refs_at || memcmp(I->d + I->refs_at, in[0].d + in[0].refs_at, I->r0 - I->refs_at)) FAIL("the @SQ dictionaries differ");
		free(hd); free(sq);
	}
	{ /* the header */
		size_t tl = 64 + strlen(sq0) + colen; int t, j, *ord;
		char *txt;
		uint32_t l32;
		for (t = 0; t < 2; ++t) for (j = 0; j < tab[t].n; ++j) tl += strlen(tab[t].line[j]) + 1;
		txt = malloc(tl); strcpy(txt, "@HD\tVN:1.3\tSO:coordinate\n"); strcat(txt, sq0);
		for (t = 0; t < 2; ++t) { ord = malloc(sizeof(int) * (tab[t].n + 1)); aa_order(tab[t].h, tab[t].n, ord); for (j = 0; j < tab[t].n; ++j) { strcat(txt, tab[t].line[ord[j]]); strcat(txt, "\n"); } free(ord); }
		strcat(txt, co);
		l32 = (uint32_t)strlen(txt);
		ocap = 16 + l32 + in[0].r0;
		for (k = 0; k < n; ++k) ocap += in[k].n;
		out = malloc(ocap);
		memcpy(out, "BAM\1", 4); memcpy(out + 4, &l32, 4); memcpy(out + 8, txt, l32); olen = 8 + l32;
		memcpy(out + olen, in[0].d + in[0].refs_at, in[0].r0 - in[0].refs_at); olen += in[0].r0 - in[0].refs_at;
		free(txt);
	}
	/* the heap: empty inputs removed unstably, built by down(i) for i = n/2-1 .. 0 */
	h = malloc(sizeof(int) * (size_t)n);
	for (k = 0; k < n; ++k) h[nh++] = k;
	for (i = 0; i < (size_t)nh;) {
		if (in[h[i]].nrec) { ++i; continue; }
		while (nh && !in[h[nh - 1]].nrec) --nh;
		if (i >= (size_t)nh) break;
		h[i] = h[--nh]; ++i;
	}
	for (k = nh / 2 - 1; k >= 0; --k) down(h, nh, k);
	while (nh) {
		in_t *I = &in[h[0]];
		const size_t at = I->off[I->next], l = 4 + u32(I->d + at);
		int t, x;
		memcpy(out + olen, I->d + at, l); olen += l;
		t = h[0]; h[0] = h[nh - 1]; h[nh - 1] = t; --nh;
		down(h, nh, 0);
		x = h[nh];
		if (++in[x].next < in[x].nrec) { int c = nh++; while (c > 0 && less_front(h[(c - 1) / 2], h[c])) { t = h[c]; h[c] = h[(c - 1) / 2]; h[(c - 1) / 2] = t; c = (c - 1) / 2; } }
	}
	*body = out; *len = olen; out = 0; rc = 0;
fail:
	free(out); free(h); free(line); free(co);
	for (k = 0; k < n; ++k) { free(in[k].d); free(in[k].off); free(in[k].key); }
	free(in);
	return rc;
}
