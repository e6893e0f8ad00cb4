/*
 * samblaster — drop-in for the `$SAMBLASTER` entry of speedseq.config (speedseq/bin/speedseq.config:14), a C shim
 * over libssq.so.  Argv/stdio contract of the reference's call sites (speedseq/bin/speedseq:439,469,1963):
 *     $SAMBLASTER [--excludeDups] --addMateTags --maxSplitCount C --minNonOverlap M --splitterFile FIFO --discordantFile FIFO
 * stdin = name-grouped SAM from `bwa mem`; stdout = the same records with 0x400 on duplicates and MC/MQ appended; the two
 * side files (FIFOs in speedseq, opened up front and streamed) receive the header plus discordant pairs / split reads.
 *
 * Duplicate detection — "the first pair seen with a signature is kept" over the WHOLE stream — is the data-parallel part
 * and runs on the GPU: the shim turns every QNAME block into one ssq_dupsig_t and hands blocks of them to
 * ssq_dupset_mark() (radix sort + adjacent-equal mark within the chunk, binary search against the device-resident sorted
 * set of earlier signatures, SURVEY.md §8a a17).  Parsing, MC/MQ tags and the discordant / splitter predicates are text
 * bookkeeping done here.  Behaviour restated from samblaster 0.1.2x (not vendored in the reference tree; SURVEY Appendix B).
 * Built with SSQ_SB_DEVICE_TEXT (the Makefile's ../bin/samblaster) the records after the header go through ssq_sbtext_run
 * instead — parsing, decisions, marking and the three streams' text on the device — and this host code only takes over the runs
 * of blocks the device refuses, marking against the same dup-set.
 */
#define _GNU_SOURCE
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <stdint.h>
#include "ssq.h"
#include "ssq_fuse.h"

#define SB_VERSION "0.1.22"
#define PAD 500           /* keeps 5' coordinates left of a contig start non-negative */
#define CHUNK_BLOCKS_MAX (1 << 20) /* QNAME blocks per ssq_dupset_mark call; SSQ_SB_CHUNK lowers it (tests, latency) */

typedef struct {
	char *text;       /* the line, tabs replaced by NULs */
	char **f; int nf;
	int flag, cigar_done, raLen, qaLen, sclip, eclip, SQO, EQO, discordant, splitter;
	long long rapos, pos;
	char *extra;
} line_t;

typedef struct { line_t *lines; int n, m; int first, second; } block_t; /* indices of the primary lines, -1 if absent */

typedef struct { char **name; long long *off; int n, m; } contigs_t;

static int contig_id(const contigs_t *c, const char *name)
{
	int i;
	for (i = 0; i < c->n; ++i) if (!strcmp(c->name[i], name)) return i;
	fprintf(stderr, "samblaster: RNAME '%s' is not in the @SQ header\n", name);
	exit(1);
}

static void parse_line(line_t *l, char *text)
{
	char *p;
	int m = 16;
	size_t n = strlen(text);
	memset(l, 0, sizeof *l);
	if (n && text[n - 1] == '\n') text[--n] = 0;
	l->text = text;
	l->f = (char**)malloc(sizeof(char*) * m);
	for (p = text;;) {
		if (l->nf == m) { m *= 2; l->f = (char**)realloc(l->f, sizeof(char*) * m); }
		l->f[l->nf++] = p;
		if (!(p = strchr(p, '\t'))) break;
		*p++ = 0;
	}
	l->flag = l->nf > 1 ? atoi(l->f[1]) : 0;
}

/* clip lengths, aligned lengths on reference/query, 5' unclipped coordinate, query offsets of the aligned part */
static void cigar_geometry(line_t *l)
{
	const char *c;
	int first = 1;
	if (l->cigar_done) return;
	for (c = l->f[5]; *c && *c != '*';) {
		char *e;
		const int len = (int)strtol(c, &e, 10);
		const char op = *e;
		c = e + 1;
		if (op == 'M' || op == '=' || op == 'X') { l->raLen += len; l->qaLen += len; first = 0; }
		else if (op == 'S' || op == 'H') { if (first) l->sclip += len; else l->eclip += len; }
		else if (op == 'D' || op == 'N') l->raLen += len;
		else if (op == 'I') l->qaLen += len;
	}
	l->rapos = atoll(l->f[3]);
	if (!(l->flag & 0x10)) { l->pos = l->rapos - l->sclip; l->SQO = l->sclip; l->EQO = l->sclip + l->qaLen - 1; }
	else { l->pos = l->rapos + l->raLen + l->eclip - 1; l->SQO = l->eclip; l->EQO = l->eclip + l->qaLen - 1; }
	l->pos += PAD;
	l->cigar_done = 1;
}

static int has_tag(const line_t *l, const char *tag) { int i; for (i = 11; i < l->nf; ++i) if (!strncmp(l->f[i], tag, 5)) return 1; return 0; }
static void add_tag(line_t *l, const char *hdr, const char *val)
{
	const size_t a = l->extra ? strlen(l->extra) : 0;
	l->extra = (char*)realloc(l->extra, a + strlen(hdr) + strlen(val) + 2);
	sprintf(l->extra + a, "\t%s%s", hdr, val);
}

static void write_line(const line_t *l, FILE *fp, const char *suffix)
{
	int i;
	for (i = 0; i < l->nf; ++i) {
		if (i) fputc('\t', fp);
		if (i == 1) fprintf(fp, "%d", l->flag);
		else { fputs(l->f[i], fp); if (i == 0 && suffix) fputs(suffix, fp); }
	}
	if (l->extra) fputs(l->extra, fp);
	fputc('\n', fp);
}

typedef struct {
	int excludeDups, addMateTags, maxSplitCount, minNonOverlap, minIndelSize, maxUnmappedBases, removeDups;
	FILE *out, *disc, *split;
	contigs_t ctg;
	unsigned long long n_ids, n_dup, n_disc, n_split;
} opt_t;

/* picks the primary lines, appends MC/MQ, computes the pair's signature; returns 1 when the block can be a duplicate */
static int block_signature(block_t *b, const opt_t *o, ssq_dupsig_t *sig, int *orphan_out, int *has_pair, int *disc_out)
{
	int i, orphan = 0;
	line_t *first = 0, *second = 0;
	memset(sig, 0, sizeof *sig);
	b->first = b->second = -1;
	*has_pair = 0; *orphan_out = 0; *disc_out = 0;
	for (i = 0; i < b->n; ++i) {
		line_t *l = &b->lines[i];
		if (l->flag & 0x900) continue; /* secondary / supplementary lines never define the pair */
		if (!(l->flag & 0x1)) b->second = i;
		else if (l->flag & 0x40) b->first = i;
		else if (l->flag & 0x80) b->second = i;
	}
	if (b->first < 0 && b->second < 0) return 0;
	if (b->first < 0 || b->second < 0) { /* lone record */
		line_t *only = &b->lines[b->first >= 0 ? b->first : b->second];
		if ((only->flag & 0x1) && ((only->flag & 0x4) || !(only->flag & 0x8))) return 0;
		if (only->flag & 0x4) return 0;
		cigar_geometry(only);
		sig->pos1 = 0;
		sig->pos2 = (uint64_t)(o->ctg.off[contig_id(&o->ctg, only->f[2])] + only->pos) + 1;
		sig->strand1 = 0; sig->strand2 = (only->flag & 0x10) ? 1 : 0; /* the absent mate counts as forward */
		sig->valid = 1;
		*orphan_out = 1;
		return 1;
	}
	first = &b->lines[b->first]; second = &b->lines[b->second];
	*has_pair = 1;
	if (o->addMateTags) {
		for (i = 0; i < b->n; ++i) {
			line_t *l = &b->lines[i], *mate;
			if ((l->flag & 0xC0) == 0x40) mate = second; else if ((l->flag & 0xC0) == 0x80) mate = first; else continue;
			if (!has_tag(l, "MC:Z:")) add_tag(l, "MC:Z:", mate->f[5]);
			if (!has_tag(l, "MQ:i:")) add_tag(l, "MQ:i:", mate->f[4]);
		}
	}
	if ((first->flag & 0x4) && (second->flag & 0x4)) return 0;
	orphan = (first->flag & 0x4) || (second->flag & 0x4);
	*orphan_out = orphan;
	if (orphan) { /* keyed on the mapped end alone; the unmapped mate carries the same strand bit */
		line_t *mapped = (first->flag & 0x4) ? second : first, *unm = (first->flag & 0x4) ? first : second;
		cigar_geometry(mapped);
		sig->pos1 = 0;
		sig->pos2 = (uint64_t)(o->ctg.off[contig_id(&o->ctg, mapped->f[2])] + mapped->pos) + 1;
		sig->strand1 = (unm->flag & 0x10) ? 1 : 0; sig->strand2 = (mapped->flag & 0x10) ? 1 : 0;
	} else {
		line_t *a = first, *c = second;
		int ia, ic, swap = 0;
		cigar_geometry(a); cigar_geometry(c);
		ia = contig_id(&o->ctg, a->f[2]); ic = contig_id(&o->ctg, c->f[2]);
		/* canonical order: smaller 5' coordinate, then smaller contig, then forward before reverse */
		if (a->pos > c->pos) swap = 1;
		else if (a->pos == c->pos) {
			if (ia > ic) swap = 1;
			else if (ia == ic && (a->flag & 0x10) && !(c->flag & 0x10)) swap = 1;
		}
		if (swap) { line_t *t = a; a = c; c = t; i = ia; ia = ic; ic = i; }
		*disc_out = !(a->flag & 0x2); /* the test looks at the canonically first end (bwa sets 0x2 on both or neither) */
		sig->pos1 = (uint64_t)(o->ctg.off[ia] + a->pos) + 1;
		sig->pos2 = (uint64_t)(o->ctg.off[ic] + c->pos) + 1;
		sig->strand1 = (a->flag & 0x10) ? 1 : 0; sig->strand2 = (c->flag & 0x10) ? 1 : 0;
	}
	sig->valid = 1;
	return 1;
}

static int cmp_sqo(const void *a, const void *b) { return (*(line_t* const*)a)->SQO - (*(line_t* const*)b)->SQO; }

static void mark_splitters(block_t *b, const opt_t *o, int mask)
{
	line_t *arr[64], *left, *right;
	int count = 0, i;
	for (i = 0; i < b->n; ++i) {
		line_t *l = &b->lines[i];
		if ((l->flag & 0xC0) == mask && !(l->flag & 0x100) && !(l->flag & 0x4)) {
			if (count >= 64 || count > o->maxSplitCount) return;
			arr[count++] = l;
		}
	}
	if (count < 2 || count > o->maxSplitCount) return;
	for (i = 0; i < count; ++i) cigar_geometry(arr[i]);
	qsort(arr, count, sizeof(line_t*), cmp_sqo);
	for (i = 1, left = arr[0]; i < count; ++i, left = right) {
		int overlap, alen1, alen2, mno;
		right = arr[i];
		overlap = 1 + (left->EQO < right->EQO ? left->EQO : right->EQO) - (left->SQO > right->SQO ? left->SQO : right->SQO);
		if (overlap < 0) overlap = 0;
		alen1 = 1 + left->EQO - left->SQO; alen2 = 1 + right->EQO - right->SQO;
		mno = alen1 - overlap < alen2 - overlap ? alen1 - overlap : alen2 - overlap;
		if (mno < o->minNonOverlap) continue;
		if (!strcmp(left->f[2], right->f[2]) && (left->flag & 0x10) == (right->flag & 0x10)) { /* same contig and strand: must look like a real SV */
			const int sd_l = (int)(left->rapos - left->sclip), ed_l = (int)((left->rapos + left->raLen) - (left->sclip + left->qaLen));
			const int sd_r = (int)(right->rapos - right->sclip), ed_r = (int)((right->rapos + right->raLen) - (right->sclip + right->qaLen));
			const int ins = (left->flag & 0x10) ? ed_r - sd_l : ed_l - sd_r;
			const int desert = right->SQO - left->EQO - 1;
			if (abs(ins) < o->minIndelSize || (desert > 0 && desert - (ins > 0 ? ins : 0) > o->maxUnmappedBases)) continue;
		}
		left->splitter = right->splitter = 1;
	}
}

static void emit_block(block_t *b, opt_t *o, int is_dup, int has_pair, int orphan, int disc)
{
	int i;
	++o->n_ids;
	if (is_dup) { ++o->n_dup; for (i = 0; i < b->n; ++i) b->lines[i].flag |= 0x400; }
	if (has_pair && !orphan && disc) /* both ends mapped and not flagged proper (a pair with both ends unmapped never gets here: disc stays 0) */
		b->lines[b->first].discordant = b->lines[b->second].discordant = 1;
	if (o->split) { mark_splitters(b, o, 0x40); mark_splitters(b, o, 0x80); }
	for (i = 0; i < b->n; ++i) {
		line_t *l = &b->lines[i];
		const int dup = l->flag & 0x400;
		if (!(o->removeDups && dup)) write_line(l, o->out, 0);
		if (o->disc && l->discordant && !(o->excludeDups && dup)) { write_line(l, o->disc, 0); ++o->n_disc; }
		if (o->split && l->splitter && !(o->excludeDups && dup)) { write_line(l, o->split, (l->flag & 0x1) ? ((l->flag & 0x40) ? "_1" : "_2") : 0); ++o->n_split; }
	}
}

static void free_block(block_t *b)
{
	int i;
	for (i = 0; i < b->n; ++i) { free(b->lines[i].text); free(b->lines[i].f); free(b->lines[i].extra); }
	free(b->lines);
}

int main(int argc, char **argv)
{
	opt_t o;
	const char *splitfn = 0, *discfn = 0;
	char *line = 0, cl[4096];
	size_t cap = 0;
	ssize_t len;
	long long total = 0;
	int i, hdr_done = 0, rc, device = getenv("SSQ_DEVICE") ? atoi(getenv("SSQ_DEVICE")) : 0;
	const int CHUNK_BLOCKS = getenv("SSQ_SB_CHUNK") && atoi(getenv("SSQ_SB_CHUNK")) > 0 && atoi(getenv("SSQ_SB_CHUNK")) < CHUNK_BLOCKS_MAX ? atoi(getenv("SSQ_SB_CHUNK")) : CHUNK_BLOCKS_MAX;
	block_t *blocks = (block_t*)calloc(CHUNK_BLOCKS, sizeof(block_t)), cur;
	ssq_dupsig_t *sigs = (ssq_dupsig_t*)malloc(sizeof(ssq_dupsig_t) * CHUNK_BLOCKS);
	uint8_t *dups = (uint8_t*)malloc(CHUNK_BLOCKS), *meta = (uint8_t*)malloc(CHUNK_BLOCKS);
	int n_blocks = 0;
	ssq_dupset_t *set = 0;
#ifdef SSQ_SB_DEVICE_TEXT
	char *hdr = 0;
	size_t hdr_len = 0, hdr_cap = 0;
#endif
	memset(&o, 0, sizeof o); memset(&cur, 0, sizeof cur);
	o.maxSplitCount = 2; o.minNonOverlap = 20; o.minIndelSize = 50; o.maxUnmappedBases = 50; o.out = stdout;
	for (i = 1; i < argc; ++i) {
		if (!strcmp(argv[i], "--excludeDups") || !strcmp(argv[i], "-e")) o.excludeDups = 1;
		else if (!strcmp(argv[i], "--addMateTags")) o.addMateTags = 1;
		else if (!strcmp(argv[i], "--removeDups") || !strcmp(argv[i], "-r")) o.removeDups = 1;
		else if (!strcmp(argv[i], "--maxSplitCount") && i + 1 < argc) o.maxSplitCount = atoi(argv[++i]);
		else if (!strcmp(argv[i], "--minNonOverlap") && i + 1 < argc) o.minNonOverlap = atoi(argv[++i]);
		else if (!strcmp(argv[i], "--minIndelSize") && i + 1 < argc) o.minIndelSize = atoi(argv[++i]);
		else if (!strcmp(argv[i], "--maxUnmappedBases") && i + 1 < argc) o.maxUnmappedBases = atoi(argv[++i]);
		else if ((!strcmp(argv[i], "--splitterFile") || !strcmp(argv[i], "-s")) && i + 1 < argc) splitfn = argv[++i];
		else if ((!strcmp(argv[i], "--discordantFile") || !strcmp(argv[i], "-d")) && i + 1 < argc) discfn = argv[++i];
		else if ((!strcmp(argv[i], "-i") || !strcmp(argv[i], "--input")) && i + 1 < argc) { if (!freopen(argv[++i], "r", stdin)) return 1; }
		else if ((!strcmp(argv[i], "-o") || !strcmp(argv[i], "--output")) && i + 1 < argc) { if (!(o.out = fopen(argv[++i], "w"))) return 1; }
		else { fprintf(stderr, "samblaster: Unrecognized option: %s\n", argv[i]); return 1; }
	}
	fprintf(stderr, "samblaster: Version %s (GPU shim over libssq)\n", SB_VERSION);
	if (discfn && !(o.disc = fopen(discfn, "w"))) { fprintf(stderr, "samblaster: Unable to open %s\n", discfn); return 1; }
	if (splitfn && !(o.split = fopen(splitfn, "w"))) { fprintf(stderr, "samblaster: Unable to open %s\n", splitfn); return 1; }
	strcpy(cl, "samblaster -i stdin -o stdout");
	if (o.excludeDups) strcat(cl, " --excludeDups");
	if (o.addMateTags) strcat(cl, " --addMateTags");
	if (discfn) { strcat(cl, " -d "); strncat(cl, discfn, 1500); }
	if (splitfn) { strcat(cl, " -s "); strncat(cl, splitfn, 1500); }
	if (splitfn) sprintf(cl + strlen(cl), " --maxSplitCount %d --maxUnmappedBases %d --minIndelSize %d --minNonOverlap %d", o.maxSplitCount, o.maxUnmappedBases, o.minIndelSize, o.minNonOverlap);
#define FLUSH_CHUNK() do { \
		if (n_blocks) { \
			if (!set && (rc = ssq_dupset_create(device, &set))) { fprintf(stderr, "samblaster: %s\n", ssq_last_error()); return 1; } /* the GPU is only touched when there is work for it (not in fused mode) */ \
			if ((rc = ssq_dupset_mark(set, (uint64_t)n_blocks, sigs, dups))) { fprintf(stderr, "samblaster: ssq_dupset_mark failed (%d): %s\n", rc, ssq_last_error()); return 1; } \
			for (i = 0; i < n_blocks; ++i) { emit_block(&blocks[i], &o, dups[i], meta[i] & 1, (meta[i] >> 1) & 1, (meta[i] >> 2) & 1); free_block(&blocks[i]); } \
			n_blocks = 0; \
		} } while (0)
#define CLOSE_BLOCK() do { \
		if (cur.n) { int orphan_, pair_, disc_; block_signature(&cur, &o, &sigs[n_blocks], &orphan_, &pair_, &disc_); meta[n_blocks] = (uint8_t)(pair_ | orphan_ << 1 | disc_ << 2); \
			blocks[n_blocks++] = cur; memset(&cur, 0, sizeof cur); if (n_blocks == CHUNK_BLOCKS) FLUSH_CHUNK(); } } while (0)
	while ((len = getline(&line, &cap, stdin)) > 0) {
		line_t l;
		if (line[0] == '@' && !hdr_done && !strncmp(line, SSQ_FUSE_MARKER, strlen(SSQ_FUSE_MARKER))) {
			/* fused mode: `bwa` already ran this program's stage on the device under the options described on the marker line */
			char mine[1024];
			FILE *fps[3] = {o.out, o.split, o.disc};
			ssq_frame_hdr_t h;
			char *buf = 0; size_t bcap = 0;
			unsigned long long n_rec[3] = {0, 0, 0};
			int bam = 0;
			ssq_fuse_describe(mine, sizeof mine, o.excludeDups, o.addMateTags, o.removeDups, o.maxSplitCount, o.minNonOverlap, o.minIndelSize, o.maxUnmappedBases);
			if (len && line[len - 1] == '\n') line[--len] = 0;
			if (len >= 4 && !strcmp(line + len - 4, "\tbam")) { bam = 1; line[len - 4] = 0; } /* main records arrive as sorted BAM runs (ssq_fuse.h) */
			if (strcmp(line + strlen(SSQ_FUSE_MARKER), mine) != 0) {
				fprintf(stderr, "samblaster: the fused stream was produced under other options (SSQ_FUSE_SAMBLASTER: %s; this command line: %s)\n", line + strlen(SSQ_FUSE_MARKER), mine);
				return 1;
			}
			for (i = 0; i < 3; ++i) if (fps[i]) fprintf(fps[i], "@PG\tID:SAMBLASTER\tVN:%s\tCL:%s\n", SB_VERSION, cl);
			if (bam) fputs(SSQ_BAM_RUNS_MARKER, o.out);
			hdr_done = 1;
			while (fread(&h, sizeof h, 1, stdin) == 1) {
				size_t k;
				if (memcmp(h.magic, SSQ_FRAME_MAGIC, 8) != 0 || h.stream > 3 || (h.stream == SSQ_STREAM_BAM_RUN) != (bam && h.stream != 1 && h.stream != 2)) { fprintf(stderr, "samblaster: corrupt fused stream\n"); return 1; }
				if (h.len > bcap) { bcap = h.len + h.len / 4; buf = (char*)realloc(buf, bcap); }
				if (fread(buf, 1, h.len, stdin) != h.len) { fprintf(stderr, "samblaster: truncated fused stream\n"); return 1; }
				if (h.stream == SSQ_STREAM_BAM_RUN) { /* passed on as it is, frame header included; records counted by their length fields */
					fwrite(&h, sizeof h, 1, o.out); fwrite(buf, 1, h.len, o.out);
					for (k = 0; k + 4 <= h.len; ++n_rec[0]) { uint32_t bs; memcpy(&bs, buf + k, 4); k += 4 + (size_t)bs; }
					continue;
				}
				if (fps[h.stream]) fwrite(buf, 1, h.len, fps[h.stream]);
				for (k = 0; k < h.len; ++k) n_rec[h.stream] += buf[k] == '\n';
			}
			free(buf);
			fflush(o.out);
			if (o.disc) fclose(o.disc);
			if (o.split) fclose(o.split);
			if (discfn) fprintf(stderr, "samblaster: Output %llu discordant read pairs to %s\n", n_rec[2] / 2, discfn);
			if (splitfn) fprintf(stderr, "samblaster: Output %llu split reads to %s\n", n_rec[1] / 2, splitfn);
			fprintf(stderr, "samblaster: routed %llu records marked on the device by `bwa mem` (fused mode).\n", n_rec[0]);
			return 0;
		}
		if (line[0] == '@' && !hdr_done) {
			if (!strncmp(line, "@SQ\t", 4)) {
				char name[1024] = "";
				const char *p = strstr(line, "\tSN:"), *q = strstr(line, "\tLN:");
				if (p && q) {
					sscanf(p + 4, "%1023[^\t\n]", name);
					if (o.ctg.n == o.ctg.m) { o.ctg.m = o.ctg.m ? o.ctg.m * 2 : 64; o.ctg.name = (char**)realloc(o.ctg.name, sizeof(char*) * o.ctg.m); o.ctg.off = (long long*)realloc(o.ctg.off, sizeof(long long) * o.ctg.m); }
					o.ctg.name[o.ctg.n] = strdup(name); o.ctg.off[o.ctg.n++] = total;
					total += atoll(q + 4) + 2 * PAD + 1;
				}
			}
			fputs(line, o.out); if (o.disc) fputs(line, o.disc); if (o.split) fputs(line, o.split);
#ifdef SSQ_SB_DEVICE_TEXT
			if (hdr_len + (size_t)len > hdr_cap) { hdr_cap = (hdr_len + (size_t)len) * 2; hdr = (char*)realloc(hdr, hdr_cap); }
			memcpy(hdr + hdr_len, line, (size_t)len); hdr_len += (size_t)len;
#endif
			continue;
		}
		if (!hdr_done) {
			FILE *fps[3] = {o.out, o.disc, o.split};
			for (i = 0; i < 3; ++i) if (fps[i]) fprintf(fps[i], "@PG\tID:SAMBLASTER\tVN:%s\tCL:%s\n", SB_VERSION, cl);
			hdr_done = 1;
		}
#ifdef SSQ_SB_DEVICE_TEXT
		{	/* the records from this line on: samblaster's stage on the device (ssq_sbtext_run) over large chunks of stdin.  A chunk
			 * with lines the device does not take goes through the host code below, marking against the same dup-set, so "first
			 * seen wins" spans both; the next chunk goes back to the device. */
			ssq_sb_opts_t so;
			ssq_sbtext_t *sbt = 0;
			ssq_sbtext_out_t so_out;
			size_t cap = 64 << 20, n = 0, at = 0, used;
			char *buf;
			int eof = 0, need = 0;
			unsigned long long n_host = 0, n_host_blocks = 0;
			char host_why[600] = "";
			so.enabled = 1; so.exclude_dups = o.excludeDups; so.add_mate_tags = o.addMateTags; so.max_split_count = o.maxSplitCount; so.min_non_overlap = o.minNonOverlap;
			so.min_indel_size = o.minIndelSize; so.max_unmapped_bases = o.maxUnmappedBases; so.remove_dups = o.removeDups; so.want_split = o.split != 0; so.want_disc = o.disc != 0;
			if ((rc = ssq_sbtext_create(device, &so, hdr, hdr_len, &sbt))) { fprintf(stderr, "samblaster: %s\n", ssq_last_error()); return 1; }
			set = ssq_sbtext_dupset(sbt);
			while ((size_t)len > cap) cap *= 2;
			if (!(buf = (char*)ssq_host_alloc(cap))) { fprintf(stderr, "samblaster: out of pinned host memory\n"); return 1; }
			memcpy(buf, line, (size_t)len); n = (size_t)len;
			for (;;) {
				if (!eof && (need || n - at < cap / 2)) {
					if (need && at == 0 && n == cap) { /* one block does not fit: a larger buffer */
						char *b2 = (char*)ssq_host_alloc(cap * 2);
						if (!b2) { fprintf(stderr, "samblaster: out of pinned host memory\n"); return 1; }
						memcpy(b2, buf, n); ssq_host_free(buf); buf = b2; cap *= 2;
					}
					if (at) { memmove(buf, buf + at, n - at); n -= at; at = 0; }
					n += fread(buf + n, 1, cap - n, stdin);
					if (n < cap) eof = 1;
					need = 0;
				}
				if (at == n && eof) break;
				rc = ssq_sbtext_run(sbt, buf + at, n - at, eof, (uint64_t)CHUNK_BLOCKS, &used, &so_out);
				if (rc == SSQ_OK) {
					FILE *fps[3] = {o.out, o.split, o.disc};
					for (i = 0; i < 3; ++i) if (fps[i] && so_out.len[i] && fwrite(so_out.text[i], 1, so_out.len[i], fps[i]) != so_out.len[i]) { fprintf(stderr, "samblaster: write failed\n"); return 1; }
					o.n_ids += so_out.n_ids; o.n_dup += so_out.n_dup; o.n_disc += so_out.n_disc_lines; o.n_split += so_out.n_split_lines;
					at += used;
					if (!used) need = 1;
				} else if (rc == SSQ_EFORMAT) { /* the blocks this run would have taken go through the host code; an unfinished last block waits */
					size_t p = at, cur_at = at;
					long long closed = 0;
					const unsigned long long ids0 = o.n_ids;
					if (!n_host++) snprintf(host_why, sizeof host_why, "%s", ssq_last_error());
					while (p < n) {
						const char *e = (const char*)memchr(buf + p, '\n', n - p);
						const size_t q = e ? (size_t)(e - buf) + 1 : n;
						char *s;
						line_t l;
						if (!e && !eof) break;
						s = (char*)malloc(q - p + 1); memcpy(s, buf + p, q - p); s[q - p] = 0;
						parse_line(&l, s);
						if (cur.n && strcmp(cur.lines[0].f[0], l.f[0]) != 0) {
							CLOSE_BLOCK();
							if (++closed == CHUNK_BLOCKS) { free(l.text); free(l.f); break; }
						}
						if (!cur.n) cur_at = p;
						if (cur.n == cur.m) { cur.m = cur.m ? cur.m * 2 : 4; cur.lines = (line_t*)realloc(cur.lines, sizeof(line_t) * cur.m); }
						cur.lines[cur.n++] = l;
						p = q;
					}
					if (closed == CHUNK_BLOCKS) at = p;
					else if (eof) { CLOSE_BLOCK(); at = n; }
					else { free_block(&cur); memset(&cur, 0, sizeof cur); at = cur_at; }
					FLUSH_CHUNK();
					n_host_blocks += o.n_ids - ids0;
				} else { fprintf(stderr, "samblaster: ssq_sbtext_run failed (%d): %s\n", rc, ssq_last_error()); return 1; }
			}
			if (n_host) fprintf(stderr, "samblaster: %llu QNAME blocks went through the host code (%llu chunks; the first: %s)\n", n_host_blocks, n_host, host_why);
			ssq_host_free(buf);
			ssq_sbtext_free(sbt); /* frees the dup-set too */
			set = 0;
			break;
		}
#endif
		parse_line(&l, strdup(line));
		if (cur.n && strcmp(cur.lines[0].f[0], l.f[0]) != 0) CLOSE_BLOCK();
		if (cur.n == cur.m) { cur.m = cur.m ? cur.m * 2 : 4; cur.lines = (line_t*)realloc(cur.lines, sizeof(line_t) * cur.m); }
		cur.lines[cur.n++] = l;
	}
	if (!hdr_done) { FILE *fps[3] = {o.out, o.disc, o.split}; for (i = 0; i < 3; ++i) if (fps[i]) fprintf(fps[i], "@PG\tID:SAMBLASTER\tVN:%s\tCL:%s\n", SB_VERSION, cl); }
	CLOSE_BLOCK();
	FLUSH_CHUNK();
	fflush(o.out);
	if (o.disc) fclose(o.disc);
	if (o.split) fclose(o.split);
	if (discfn) fprintf(stderr, "samblaster: Output %llu discordant read pairs to %s\n", o.n_disc / 2, discfn);
	if (splitfn) fprintf(stderr, "samblaster: Output %llu split reads to %s\n", o.n_split / 2, splitfn);
	fprintf(stderr, "samblaster: Marked %llu of %llu (%.2f%%) read ids as duplicates.\n", o.n_dup, o.n_ids, o.n_ids ? 100.0 * o.n_dup / o.n_ids : 0.0);
	if (set) ssq_dupset_free(set);
#ifdef SSQ_SB_DEVICE_TEXT
	free(hdr);
#endif
	free(line); free(blocks); free(sigs); free(dups); free(meta);
	return 0;
}
