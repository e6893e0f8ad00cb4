/*
 * ssqo_index.c — ORACLE (test infrastructure): `bwa index` restatement and index loader.
 *
 * Follows: call site speedseq/bin/speedseq:386-391 (`$BWA index $REF` must create
 * REF.{amb,ann,pac,bwt,sa}); on-disk format verified against the goldens
 * speedseq/example/data/human_g1k_v37_20_42220611-42542245.fasta.{amb,ann,pac,bwt,sa}
 * (SURVEY.md §8c "Verified on-disk index format").  Upstream names (not in tree): bns_fasta2bntseq,
 * bwt_pac2bwt, bwt_bwtupdate_core, bwt_cal_sa, bwa_idx_load.
 */
#define _GNU_SOURCE
#include <stdlib.h>
#include <string.h>
#include <ctype.h>
#include <zlib.h>
#include "ssqo.h"
#include "ssqo_kseq.h"

const uint8_t ssqo_nt4[256] = {
#define R16 4,4,4,4,4,4,4,4,4,4,4,4,4,4,4,4
	R16, R16, R16, R16,
	4,0,4,1,4,4,4,2,4,4,4,4,4,4,4,4, 4,4,4,4,3,4,4,4,4,4,4,4,4,4,4,4,
	4,0,4,1,4,4,4,2,4,4,4,4,4,4,4,4, 4,4,4,4,3,4,4,4,4,4,4,4,4,4,4,4,
	R16, R16, R16, R16, R16, R16, R16, R16
#undef R16
};

/* ---------------------------------------------------------------- SA-IS ---- */
/* Induced-sorting suffix array construction (Nong, Zhang & Chan 2009), written for this oracle. */
#define T_S 1
#define T_L 0
static inline int is_lms(const uint8_t *t, int32_t i) { return i > 0 && t[i] == T_S && t[i - 1] == T_L; }

static void bucket_bounds(const int32_t *s, int32_t *bkt, int32_t n, int32_t K, int want_end)
{
	int32_t i, sum = 0;
	memset(bkt, 0, sizeof(int32_t) * (size_t)K);
	for (i = 0; i < n; ++i) ++bkt[s[i]];
	for (i = 0; i < K; ++i) {
		sum += bkt[i];
		bkt[i] = want_end ? sum : sum - bkt[i];
	}
}

static void induce(const int32_t *s, int32_t *sa, const uint8_t *t, int32_t *bkt, int32_t n, int32_t K)
{
	int32_t i, j;
	bucket_bounds(s, bkt, n, K, 0);
	for (i = 0; i < n; ++i) { /* L-type, left to right */
		j = sa[i] - 1;
		if (sa[i] > 0 && t[j] == T_L) sa[bkt[s[j]]++] = j;
	}
	bucket_bounds(s, bkt, n, K, 1);
	for (i = n - 1; i >= 0; --i) { /* S-type, right to left */
		j = sa[i] - 1;
		if (sa[i] > 0 && t[j] == T_S) sa[--bkt[s[j]]] = j;
	}
}

void ssqo_sais(const int32_t *s, int32_t *sa, int32_t n, int32_t K)
{
	int32_t i, j, n1 = 0, name = 0, prev = -1;
	uint8_t *t = (uint8_t*)malloc((size_t)n);
	int32_t *bkt = (int32_t*)malloc(sizeof(int32_t) * (size_t)K);
	int32_t *s1, *sa1;
	if (n == 1) { sa[0] = 0; free(t); free(bkt); return; }
	t[n - 1] = T_S;
	for (i = n - 2; i >= 0; --i)
		t[i] = (s[i] < s[i + 1] || (s[i] == s[i + 1] && t[i + 1] == T_S)) ? T_S : T_L;
	/* stage 1: sort LMS substrings */
	bucket_bounds(s, bkt, n, K, 1);
	for (i = 0; i < n; ++i) sa[i] = -1;
	for (i = 1; i < n; ++i) if (is_lms(t, i)) sa[--bkt[s[i]]] = i;
	induce(s, sa, t, bkt, n, K);
	for (i = 0; i < n; ++i) if (is_lms(t, sa[i])) sa[n1++] = sa[i];
	for (i = n1; i < n; ++i) sa[i] = -1;
	for (i = 0; i < n1; ++i) {
		int32_t pos = sa[i], d, diff = 0;
		if (prev < 0) diff = 1;
		else for (d = 0; ; ++d) {
			if (s[pos + d] != s[prev + d] || t[pos + d] != t[prev + d]) { diff = 1; break; }
			if (d > 0 && (is_lms(t, pos + d) || is_lms(t, prev + d))) break;
		}
		if (diff) { ++name; prev = pos; }
		sa[n1 + (pos >> 1)] = name - 1;
	}
	for (i = n - 1, j = n - 1; i >= n1; --i) if (sa[i] >= 0) sa[j--] = sa[i];
	/* stage 2: recurse on the reduced string */
	sa1 = sa; s1 = sa + n - n1;
	if (name < n1) ssqo_sais(s1, sa1, n1, name);
	else for (i = 0; i < n1; ++i) sa1[s1[i]] = i;
	/* stage 3: induce the full SA from sorted LMS suffixes */
	bucket_bounds(s, bkt, n, K, 1);
	for (i = 1, j = 0; i < n; ++i) if (is_lms(t, i)) s1[j++] = i;
	for (i = 0; i < n1; ++i) sa1[i] = s1[sa1[i]];
	for (i = n1; i < n; ++i) sa[i] = -1;
	for (i = n1 - 1; i >= 0; --i) { j = sa[i]; sa[i] = -1; sa[--bkt[s[j]]] = j; }
	induce(s, sa, t, bkt, n, K);
	free(t); free(bkt);
}

/* ------------------------------------------------------------ pac/ann/amb ---- */
#define PAC_SET(pac, l, c) ((pac)[(l) >> 2] |= (c) << ((~(l) & 3) << 1))
#define PAC_GET(pac, l) ((pac)[(l) >> 2] >> ((~(l) & 3) << 1) & 3)

typedef struct { ssqo_bns_t bns; uint8_t *pac; int64_t m_pac; int m_seqs, m_holes; } packer_t;

/* one FASTA record -> bns + pac; ambiguous bases become lrand48()&3 after srand48(11), holes logged */
static void pack_one(packer_t *pk, const ssqo_kseq_t *ks)
{
	ssqo_bns_t *b = &pk->bns;
	ssqo_ann_t *p;
	ssqo_hole_t *q = 0;
	int i, lasts = 0;
	if (b->n_seqs == pk->m_seqs) {
		pk->m_seqs = pk->m_seqs ? pk->m_seqs << 1 : 8;
		b->anns = (ssqo_ann_t*)realloc(b->anns, sizeof(ssqo_ann_t) * pk->m_seqs);
	}
	p = &b->anns[b->n_seqs];
	p->name = strdup(ks->name.s);
	p->anno = ks->comment.l > 0 ? strdup(ks->comment.s) : strdup("(null)");
	p->gi = 0; p->len = (int32_t)ks->seq.l;
	p->offset = b->n_seqs == 0 ? 0 : (p - 1)->offset + (p - 1)->len;
	p->n_ambs = 0;
	for (i = 0; i < (int)ks->seq.l; ++i) {
		int c = ssqo_nt4[(uint8_t)ks->seq.s[i]];
		if (c >= 4) {
			if (lasts == ks->seq.s[i]) ++q->len;
			else {
				if (b->n_holes == pk->m_holes) {
					pk->m_holes = pk->m_holes ? pk->m_holes << 1 : 8;
					b->holes = (ssqo_hole_t*)realloc(b->holes, sizeof(ssqo_hole_t) * pk->m_holes);
				}
				q = &b->holes[b->n_holes++];
				q->len = 1; q->offset = b->l_pac; q->amb = ks->seq.s[i];
				++p->n_ambs;
			}
		}
		lasts = ks->seq.s[i];
		if (c >= 4) c = (int)(lrand48() & 3);
		if (b->l_pac == pk->m_pac) {
			int64_t old = pk->m_pac;
			pk->m_pac = pk->m_pac ? pk->m_pac << 1 : 0x10000;
			pk->pac = (uint8_t*)realloc(pk->pac, pk->m_pac / 4);
			memset(pk->pac + old / 4, 0, (pk->m_pac - old) / 4);
		}
		PAC_SET(pk->pac, b->l_pac, c);
		++b->l_pac;
	}
	++b->n_seqs;
}

static int write_bns_text(const ssqo_bns_t *b, const char *prefix)
{
	char fn[4096];
	FILE *fp;
	int i;
	snprintf(fn, sizeof fn, "%s.ann", prefix);
	if (!(fp = fopen(fn, "w"))) return -1;
	fprintf(fp, "%lld %d %u\n", (long long)b->l_pac, b->n_seqs, b->seed);
	for (i = 0; i < b->n_seqs; ++i) {
		const ssqo_ann_t *p = &b->anns[i];
		fprintf(fp, "%d %s", p->gi, p->name);
		if (p->anno[0]) fprintf(fp, " %s\n", p->anno); else fprintf(fp, "\n");
		fprintf(fp, "%lld %d %d\n", (long long)p->offset, p->len, p->n_ambs);
	}
	fclose(fp);
	snprintf(fn, sizeof fn, "%s.amb", prefix);
	if (!(fp = fopen(fn, "w"))) return -1;
	fprintf(fp, "%lld %d %u\n", (long long)b->l_pac, b->n_seqs, b->n_holes);
	for (i = 0; i < b->n_holes; ++i)
		fprintf(fp, "%lld %d %c\n", (long long)b->holes[i].offset, b->holes[i].len, b->holes[i].amb);
	fclose(fp);
	return 0;
}

static int write_pac(const uint8_t *pac, int64_t l_pac, const char *prefix)
{
	char fn[4096];
	FILE *fp;
	uint8_t ct;
	snprintf(fn, sizeof fn, "%s.pac", prefix);
	if (!(fp = fopen(fn, "wb"))) return -1;
	fwrite(pac, 1, (l_pac >> 2) + ((l_pac & 3) == 0 ? 0 : 1), fp);
	if (l_pac % 4 == 0) { ct = 0; fwrite(&ct, 1, 1, fp); }
	ct = l_pac % 4;
	fwrite(&ct, 1, 1, fp);
	fclose(fp);
	return 0;
}

int ssqo_index_build(const char *fasta, const char *prefix)
{
	packer_t pk;
	ssqo_kseq_t *ks;
	int64_t l_pac, n, i;
	int32_t *s, *sa;
	uint64_t primary = 0, L2[5], c4[4];
	uint32_t *raw, *buf;
	uint64_t raw_words, n_occ, bwt_size, k;
	char fn[4096];
	FILE *fp;

	memset(&pk, 0, sizeof pk);
	pk.bns.seed = 11;
	srand48(11);
	if (!(ks = ssqo_kseq_open(fasta))) return -1;
	while (ssqo_kseq_read(ks) >= 0) pack_one(&pk, ks);
	ssqo_kseq_close(ks);
	l_pac = pk.bns.l_pac;
	if (l_pac == 0) return -2;
	if (2 * l_pac + 1 >= 0x7fffffffLL) { fprintf(stderr, "[ssqo_index] reference too large for the 32-bit oracle SA-IS\n"); return -3; }
	if (write_bns_text(&pk.bns, prefix) || write_pac(pk.pac, l_pac, prefix)) return -4;

	/* T = forward + reverse complement (+ sentinel 0; bases shifted to 1..4) */
	n = 2 * l_pac;
	s = (int32_t*)malloc(sizeof(int32_t) * (n + 1));
	sa = (int32_t*)malloc(sizeof(int32_t) * (n + 1));
	for (i = 0; i < l_pac; ++i) {
		int c = PAC_GET(pk.pac, i);
		s[i] = c + 1;
		s[n - 1 - i] = (3 - c) + 1;
	}
	s[n] = 0;
	ssqo_sais(s, sa, (int32_t)(n + 1), 5);

	/* BWT (the '$' row is dropped from the symbol stream; primary = its row) */
	raw_words = (n + 15) / 16;
	raw = (uint32_t*)calloc(raw_words, 4);
	memset(L2, 0, sizeof L2);
	for (i = 0, k = 0; i <= n; ++i) {
		if (sa[i] == 0) { primary = i; continue; }
		{
			uint32_t c = (uint32_t)(s[sa[i] - 1] - 1);
			raw[k >> 4] |= c << ((~k & 15) << 1);
			++L2[c + 1];
			++k;
		}
	}
	for (i = 2; i <= 4; ++i) L2[i] += L2[i - 1];
	/* interleave occ checkpoints every 128 symbols */
	n_occ = (n + 127) / 128 + 1;
	bwt_size = raw_words + n_occ * 8;
	buf = (uint32_t*)calloc(bwt_size, 4);
	memset(c4, 0, sizeof c4);
	for (i = 0, k = 0; i < n; ++i) {
		if (i % 128 == 0) { memcpy(buf + k, c4, 32); k += 8; }
		if (i % 16 == 0) buf[k++] = raw[i / 16];
		++c4[raw[i >> 4] >> ((~i & 15) << 1) & 3];
	}
	memcpy(buf + k, c4, 32);
	if (k + 8 != bwt_size) { fprintf(stderr, "[ssqo_index] inconsistent bwt_size\n"); return -5; }
	snprintf(fn, sizeof fn, "%s.bwt", prefix);
	if (!(fp = fopen(fn, "wb"))) return -4;
	fwrite(&primary, 8, 1, fp);
	fwrite(L2 + 1, 8, 4, fp);
	fwrite(buf, 4, bwt_size, fp);
	fclose(fp);
	/* sampled SA, every 32 rows, row 0 implicit */
	{
		uint64_t sa_intv = 32, seq_len = n, n_sa = (n + 32) / 32, v;
		snprintf(fn, sizeof fn, "%s.sa", prefix);
		if (!(fp = fopen(fn, "wb"))) return -4;
		fwrite(&primary, 8, 1, fp);
		fwrite(L2 + 1, 8, 4, fp);
		fwrite(&sa_intv, 8, 1, fp);
		fwrite(&seq_len, 8, 1, fp);
		for (k = 1; k < n_sa; ++k) { v = (uint64_t)sa[k * 32]; fwrite(&v, 8, 1, fp); }
		fclose(fp);
	}
	free(s); free(sa); free(raw); free(buf); free(pk.pac);
	for (i = 0; i < pk.bns.n_seqs; ++i) { free(pk.bns.anns[i].name); free(pk.bns.anns[i].anno); }
	free(pk.bns.anns); free(pk.bns.holes);
	return 0;
}

/* ----------------------------------------------------------------- loader ---- */
static void *slurp(const char *fn, size_t skip, size_t *len)
{
	FILE *fp = fopen(fn, "rb");
	long sz;
	void *p;
	if (!fp) return 0;
	fseek(fp, 0, SEEK_END); sz = ftell(fp); fseek(fp, (long)skip, SEEK_SET);
	*len = (size_t)sz - skip;
	p = malloc(*len + 8);
	if (fread(p, 1, *len, fp) != *len) { free(p); p = 0; }
	fclose(fp);
	return p;
}

ssqo_idx_t *ssqo_idx_load(const char *prefix)
{
	ssqo_idx_t *idx = (ssqo_idx_t*)calloc(1, sizeof(ssqo_idx_t));
	char fn[4096], str[8192];
	FILE *fp;
	size_t len;
	uint64_t hdr[7];
	int i;
	long long ll;
	/* .bwt */
	snprintf(fn, sizeof fn, "%s.bwt", prefix);
	if (!(fp = fopen(fn, "rb"))) goto fail;
	if (fread(hdr, 8, 5, fp) != 5) { fclose(fp); goto fail; }
	fclose(fp);
	idx->bwt.primary = hdr[0];
	idx->bwt.L2[0] = 0; memcpy(idx->bwt.L2 + 1, hdr + 1, 32);
	idx->bwt.seq_len = idx->bwt.L2[4];
	idx->bwt.bwt = (uint32_t*)slurp(fn, 40, &len);
	if (!idx->bwt.bwt) goto fail;
	idx->bwt.bwt_size = len / 4;
	/* .sa */
	snprintf(fn, sizeof fn, "%s.sa", prefix);
	if (!(fp = fopen(fn, "rb"))) goto fail;
	if (fread(hdr, 8, 7, fp) != 7) { fclose(fp); goto fail; }
	if (hdr[0] != idx->bwt.primary || hdr[6] != idx->bwt.seq_len) { fclose(fp); goto fail; }
	idx->bwt.sa_intv = (int)hdr[5];
	idx->bwt.n_sa = (idx->bwt.seq_len + idx->bwt.sa_intv) / idx->bwt.sa_intv;
	idx->bwt.sa = (uint64_t*)calloc(idx->bwt.n_sa, 8);
	idx->bwt.sa[0] = (uint64_t)-1;
	if (fread(idx->bwt.sa + 1, 8, idx->bwt.n_sa - 1, fp) != idx->bwt.n_sa - 1) { fclose(fp); goto fail; }
	fclose(fp);
	/* .ann */
	snprintf(fn, sizeof fn, "%s.ann", prefix);
	if (!(fp = fopen(fn, "r"))) goto fail;
	if (fscanf(fp, "%lld%d%u", &ll, &idx->bns.n_seqs, &idx->bns.seed) != 3) { fclose(fp); goto fail; }
	idx->bns.l_pac = ll;
	idx->bns.anns = (ssqo_ann_t*)calloc(idx->bns.n_seqs, sizeof(ssqo_ann_t));
	for (i = 0; i < idx->bns.n_seqs; ++i) {
		ssqo_ann_t *p = &idx->bns.anns[i];
		char *q = str;
		int c;
		if (fscanf(fp, "%u%8191s", &p->gi, str) != 2) { fclose(fp); goto fail; }
		p->name = strdup(str);
		while (q - str < (long)sizeof(str) - 1 && (c = fgetc(fp)) != '\n' && c != EOF) *q++ = (char)c;
		*q = 0;
		p->anno = (q - str > 1 && strcmp(str, " (null)") != 0) ? strdup(str + 1) : strdup("");
		if (fscanf(fp, "%lld%d%d", &ll, &p->len, &p->n_ambs) != 3) { fclose(fp); goto fail; }
		p->offset = ll;
	}
	fclose(fp);
	/* .amb */
	snprintf(fn, sizeof fn, "%s.amb", prefix);
	if (!(fp = fopen(fn, "r"))) goto fail;
	{
		int ns; unsigned nh;
		if (fscanf(fp, "%lld%d%u", &ll, &ns, &nh) != 3) { fclose(fp); goto fail; }
		idx->bns.n_holes = (int)nh;
		idx->bns.holes = (ssqo_hole_t*)calloc(nh ? nh : 1, sizeof(ssqo_hole_t));
		for (i = 0; i < (int)nh; ++i) {
			ssqo_hole_t *h = &idx->bns.holes[i];
			if (fscanf(fp, "%lld%d%8191s", &ll, &h->len, str) != 3) { fclose(fp); goto fail; }
			h->offset = ll; h->amb = str[0];
		}
	}
	fclose(fp);
	/* .pac */
	snprintf(fn, sizeof fn, "%s.pac", prefix);
	idx->pac = (uint8_t*)slurp(fn, 0, &len);
	if (!idx->pac) goto fail;
	if ((int64_t)len < idx->bns.l_pac / 4 + 1) goto fail;
	return idx;
fail:
	fprintf(stderr, "[ssqo_idx_load] failed to load index '%s'\n", prefix);
	ssqo_idx_destroy(idx);
	return 0;
}

void ssqo_idx_destroy(ssqo_idx_t *idx)
{
	int i;
	if (!idx) return;
	free(idx->bwt.bwt); free(idx->bwt.sa); free(idx->pac);
	for (i = 0; i < idx->bns.n_seqs && idx->bns.anns; ++i) { free(idx->bns.anns[i].name); free(idx->bns.anns[i].anno); }
	free(idx->bns.anns); free(idx->bns.holes);
	free(idx);
}

int ssqo_main_index(int argc, char **argv)
{
	const char *prefix = 0;
	int i, j = 0;
	const char *pos[2] = {0, 0};
	for (i = 1; i < argc; ++i) {
		if (!strcmp(argv[i], "-p") && i + 1 < argc) prefix = argv[++i];
		else if (!strcmp(argv[i], "-a") && i + 1 < argc) ++i; /* algorithm choice does not change the output */
		else if (argv[i][0] != '-' && j < 2) pos[j++] = argv[i];
	}
	if (!pos[0]) { fprintf(stderr, "Usage: bwa index [-p prefix] <in.fasta>\n"); return 1; }
	return ssqo_index_build(pos[0], prefix ? prefix : pos[0]) ? 1 : 0;
}
