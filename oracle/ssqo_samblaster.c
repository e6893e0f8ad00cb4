/*
 * ssqo_samblaster.c — ORACLE (test infrastructure): SAMBLASTER restatement.
 * SURVEY.md §8a rows a16-a19 and Appendix B.  Reference call site:
 *   $SAMBLASTER [--excludeDups] --addMateTags --maxSplitCount C --minNonOverlap M
 *               --splitterFile FIFO --discordantFile FIFO      (speedseq/bin/speedseq:439,469)
 * stdin = name-grouped SAM from `bwa mem`, stdout = SAM with 0x400 set on duplicates (first-seen pair
 * per signature is kept), MC/MQ appended, side streams = discordant pairs and split reads.
 * The signature of a pair is (contig, 5'-unclipped position, strand) of both primary lines, ends
 * ordered canonically; orphans (mate unmapped) are keyed on the mapped end alone.
 * Upstream (not in tree): GregoryFaust/samblaster@b6426391 samblaster.cpp.
 */
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include "ssqo.h"

#define SB_VERSION "0.1.22"

/* ---- batch form: first-seen-wins over explicit signatures (parity target of the GPU dup-mark kernel) ---- */
typedef struct { uint64_t a, b; uint32_t c; } sigkey_t;
typedef struct { sigkey_t *keys; uint8_t *used; size_t cap, n; } sigset_t_;

static inline uint64_t mix64(uint64_t x) { x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33; return x; }

static void sigset_grow(sigset_t_ *s);
/* returns 1 if newly inserted, 0 if already present */
static int sigset_insert(sigset_t_ *s, sigkey_t k)
{
	size_t i;
	if ((s->n + 1) * 2 > s->cap) sigset_grow(s);
	i = (size_t)(mix64(k.a * 0x9e3779b97f4a7c15ULL ^ mix64(k.b) ^ k.c) & (s->cap - 1));
	while (s->used[i]) {
		if (s->keys[i].a == k.a && s->keys[i].b == k.b && s->keys[i].c == k.c) return 0;
		i = (i + 1) & (s->cap - 1);
	}
	s->used[i] = 1; s->keys[i] = k; ++s->n;
	return 1;
}
static void sigset_grow(sigset_t_ *s)
{
	sigset_t_ t;
	size_t i;
	t.cap = s->cap ? s->cap << 1 : 1024; t.n = 0;
	t.keys = (sigkey_t*)malloc(t.cap * sizeof(sigkey_t));
	t.used = (uint8_t*)calloc(t.cap, 1);
	for (i = 0; i < s->cap; ++i) if (s->used[i]) sigset_insert(&t, s->keys[i]);
	free(s->keys); free(s->used);
	*s = t;
}

void ssqo_dupmark(size_t n, const ssqo_dupsig_t *sig, uint8_t *is_dup)
{
	sigset_t_ set = {0, 0, 0, 0};
	size_t i;
	for (i = 0; i < n; ++i) {
		sigkey_t k;
		is_dup[i] = 0;
		if (!sig[i].valid) continue;
		k.a = sig[i].pos1; k.b = sig[i].pos2; k.c = (uint32_t)sig[i].strand1 << 1 | sig[i].strand2;
		if (!sigset_insert(&set, k)) is_dup[i] = 1;
	}
	free(set.keys); free(set.used);
}

/* ----------------------------------------------------------------- streaming tool ---- */
typedef struct line_s {
	char *buf;            /* the raw line, fields NUL-separated after split */
	char **f; int nf;     /* field pointers */
	int flag, flag_dirty;
	int64_t pos, rapos;   /* 5' unclipped position (padded), POS */
	int raLen, qaLen, sclip, eclip, SQO, EQO;
	int cigar_done, seqnum;
	int discordant, splitter;
	char *extra;          /* appended tags */
	char *newname;
	struct line_s *next;
} line_t;

typedef struct {
	char **names; int64_t *offs; int n_seq, m_seq;
	sigset_t_ sigs;
	int excludeDups, addMateTags, maxSplitCount, minNonOverlap, minIndelSize, maxUnmappedBases, removeDups, acceptDups;
	FILE *out, *disc, *split;
	uint64_t n_ids, n_dup, n_disc, n_split;
} sb_state_t;

#define PAD 500 /* positions are padded so that 5' coordinates left of a contig start stay non-negative */

static int seq_lookup(sb_state_t *st, const char *name)
{
	int i;
	for (i = 0; i < st->n_seq; ++i) if (strcmp(st->names[i], name) == 0) return i;
	return -1;
}

static void seq_add(sb_state_t *st, const char *name, int64_t len, int64_t *total)
{
	if (st->n_seq == st->m_seq) {
		st->m_seq = st->m_seq ? st->m_seq << 1 : 64;
		st->names = (char**)realloc(st->names, sizeof(char*) * st->m_seq);
		st->offs = (int64_t*)realloc(st->offs, sizeof(int64_t) * st->m_seq);
	}
	st->names[st->n_seq] = strdup(name);
	st->offs[st->n_seq] = *total;
	*total += len + 2 * PAD + 1;
	++st->n_seq;
}

static line_t *line_parse(char *raw)
{
	line_t *l = (line_t*)calloc(1, sizeof(line_t));
	char *p;
	int m = 16;
	size_t n = strlen(raw);
	if (n && raw[n - 1] == '\n') raw[--n] = 0;
	l->buf = raw;
	l->f = (char**)malloc(sizeof(char*) * m);
	for (p = raw; ; ) {
		if (l->nf == m) { m <<= 1; l->f = (char**)realloc(l->f, sizeof(char*) * m); }
		l->f[l->nf++] = p;
		p = strchr(p, '\t');
		if (!p) break;
		*p++ = 0;
	}
	l->flag = l->nf > 1 ? atoi(l->f[1]) : 0;
	return l;
}

static void line_free(line_t *l) { free(l->buf); free(l->f); free(l->extra); free(l->newname); free(l); }

static void calc_offsets(line_t *l)
{
	const char *c;
	int first = 1;
	if (l->cigar_done) return;
	l->raLen = l->qaLen = l->sclip = l->eclip = 0;
	for (c = l->f[5]; *c && *c != '*'; ) {
		int len = (int)strtol(c, (char**)&c, 10);
		char op = *c++;
		if (op == 'M' || op == '=' || op == 'X') { l->raLen += len; l->qaLen += len; first = 0; }
		else if (op == 'S' || op == 'H') { if (first) l->sclip += len; else l->eclip += len; }
		else if (op == 'D' || op == 'N') l->raLen += len;
		else if (op == 'I') l->qaLen += len;
	}
	l->rapos = atoll(l->f[3]);
	if (!(l->flag & 0x10)) {
		l->pos = l->rapos - l->sclip;
		l->SQO = l->sclip; l->EQO = l->sclip + l->qaLen - 1;
	} else {
		l->pos = l->rapos + l->raLen + l->eclip - 1;
		l->SQO = l->eclip; l->EQO = l->eclip + l->qaLen - 1;
	}
	l->pos += PAD;
	l->cigar_done = 1;
}

static int has_tag(const line_t *l, const char *tag)
{
	int i;
	for (i = 11; i < l->nf; ++i) if (strncmp(l->f[i], tag, 5) == 0) return 1;
	return 0;
}

static void add_tag(line_t *l, const char *hdr, const char *val)
{
	size_t a = l->extra ? strlen(l->extra) : 0, b = strlen(hdr) + strlen(val) + 2;
	l->extra = (char*)realloc(l->extra, a + b);
	sprintf(l->extra + a, "\t%s%s", hdr, val);
}

static void write_line(const line_t *l, FILE *fp, int rename)
{
	int i;
	for (i = 0; i < l->nf; ++i) {
		if (i) fputc('\t', fp);
		if (i == 0 && rename && l->newname) fputs(l->newname, fp);
		else if (i == 1) fprintf(fp, "%d", l->flag);
		else fputs(l->f[i], fp);
	}
	if (l->extra) fputs(l->extra, fp);
	fputc('\n', fp);
}

static int need_swap(const line_t *a, const line_t *b)
{
	if (a->pos > b->pos) return 1;
	if (a->pos < b->pos) return 0;
	if (a->seqnum > b->seqnum) return 1;
	if (a->seqnum < b->seqnum) return 0;
	if ((a->flag & 0x10) == (b->flag & 0x10)) return 0;
	return (a->flag & 0x10) && !(b->flag & 0x10);
}

static void mark_dups_discordants(line_t *block, sb_state_t *st)
{
	line_t *first = 0, *second = 0, *l, dummy;
	int orphan = 0, dummy_first = 0;
	for (l = block; l; l = l->next) {
		if (l->flag & 0x900) continue; /* only primary lines define a pair */
		if (!(l->flag & 0x1)) second = l;
		else if (l->flag & 0x40) first = l;
		else if (l->flag & 0x80) second = l;
	}
	if (!first && !second) return;
	if (!first || !second) {
		if (!second) { second = first; first = 0; }
		if ((second->flag & 0x1) && ((second->flag & 0x4) || !(second->flag & 0x8))) return;
		if (second->flag & 0x4) return;
		memset(&dummy, 0, sizeof dummy);
		dummy.flag = (second->flag & 0x10) ? 0x25 : 0x5;
		first = &dummy;
		orphan = 1; dummy_first = 1;
	} else {
		if (st->addMateTags) {
			for (l = block; l; l = l->next) {
				line_t *mate;
				if ((l->flag & 0xC0) == 0x40) mate = second;
				else if ((l->flag & 0xC0) == 0x80) mate = first;
				else continue;
				if (!has_tag(l, "MC:Z:")) add_tag(l, "MC:Z:", mate->f[5]);
				if (!has_tag(l, "MQ:i:")) add_tag(l, "MQ:i:", mate->f[4]);
			}
		}
		if ((first->flag & 0x4) && (second->flag & 0x4)) return;
		orphan = (first->flag & 0x4) || (second->flag & 0x4);
		if (!(first->flag & 0x4) && (second->flag & 0x4)) { line_t *t = first; first = second; second = t; } /* unmapped end goes first */
	}
	if (!st->acceptDups) {
		sigkey_t k;
		int s1, s2;
		calc_offsets(second);
		second->seqnum = seq_lookup(st, second->f[2]);
		if (orphan) { first->pos = 0; first->seqnum = -1; }
		else { calc_offsets(first); first->seqnum = seq_lookup(st, first->f[2]); }
		if (!orphan && need_swap(first, second)) { line_t *t = first; first = second; second = t; }
		k.a = orphan ? 0 : (uint64_t)(st->offs[first->seqnum] + first->pos) + 1;
		k.b = (uint64_t)(st->offs[second->seqnum] + second->pos) + 1;
		s1 = (first->flag & 0x10) ? 1 : 0; s2 = (second->flag & 0x10) ? 1 : 0;
		k.c = (uint32_t)(s1 << 1 | s2);
		if (!sigset_insert(&st->sigs, k)) {
			++st->n_dup;
			for (l = block; l; l = l->next) l->flag |= 0x400; /* all lines of the block, or none */
		}
	}
	if (dummy_first) return;
	if (!orphan && !(first->flag & 0x2)) { first->discordant = 1; second->discordant = 1; }
}

static int cmp_sqo(const void *a, const void *b)
{
	const line_t *x = *(line_t* const*)a, *y = *(line_t* const*)b;
	return x->SQO - y->SQO;
}

static void mark_splitters(line_t *block, sb_state_t *st, int mask)
{
	line_t *arr[64], *left, *right;
	int count = 0, i;
	for (left = block; left; left = left->next)
		if ((left->flag & 0xC0) == mask && !(left->flag & 0x100) && !(left->flag & 0x4)) {
			if (count >= 64 || count > st->maxSplitCount) return;
			arr[count++] = left;
		}
	if (count < 2 || count > st->maxSplitCount) return;
	for (i = 0; i < count; ++i) calc_offsets(arr[i]);
	qsort(arr, count, sizeof(line_t*), cmp_sqo);
	left = arr[0];
	for (i = 1; i < count; ++i, left = right) {
		int overlap, alen1, alen2, mno;
		right = arr[i];
		overlap = 1 + (left->EQO < right->EQO ? left->EQO : right->EQO) - (left->SQO > right->SQO ? left->SQO : right->SQO);
		if (overlap < 0) overlap = 0;
		alen1 = 1 + left->EQO - left->SQO; alen2 = 1 + right->EQO - right->SQO;
		mno = alen1 - overlap < alen2 - overlap ? alen1 - overlap : alen2 - overlap;
		if (mno < st->minNonOverlap) continue;
		if (strcmp(left->f[2], right->f[2]) == 0 && (left->flag & 0x10) == (right->flag & 0x10)) {
			int leftDiag, rightDiag, insSize, desert;
			#define START_DIAG(l) ((int)((l)->rapos - (l)->sclip))
			#define END_DIAG(l) ((int)(((l)->rapos + (l)->raLen) - ((l)->sclip + (l)->qaLen)))
			if (left->flag & 0x10) { leftDiag = START_DIAG(left); rightDiag = END_DIAG(right); insSize = rightDiag - leftDiag; }
			else { leftDiag = END_DIAG(left); rightDiag = START_DIAG(right); insSize = leftDiag - rightDiag; }
			desert = right->SQO - left->EQO - 1;
			if (abs(insSize) < st->minIndelSize || (desert > 0 && desert - (insSize > 0 ? insSize : 0) > st->maxUnmappedBases)) continue;
		}
		left->splitter = 1; right->splitter = 1;
	}
}

static void process_block(line_t *block, sb_state_t *st)
{
	line_t *l;
	++st->n_ids;
	mark_dups_discordants(block, st);
	if (st->split) { mark_splitters(block, st, 0x40); mark_splitters(block, st, 0x80); }
	for (l = block; l; l = l->next) {
		if (!(st->removeDups && (l->flag & 0x400))) write_line(l, st->out, 0);
		if (st->disc && l->discordant && !(st->excludeDups && (l->flag & 0x400))) { write_line(l, st->disc, 0); ++st->n_disc; }
		if (st->split && l->splitter && !(st->excludeDups && (l->flag & 0x400))) {
			if (l->flag & 0x1) {
				l->newname = (char*)malloc(strlen(l->f[0]) + 3);
				sprintf(l->newname, "%s_%c", l->f[0], (l->flag & 0x40) ? '1' : '2');
			}
			write_line(l, st->split, 1); ++st->n_split;
		}
	}
}

int ssqo_main_samblaster(int argc, char **argv)
{
	sb_state_t st;
	char *line = 0, *cl;
	size_t cap = 0;
	ssize_t len;
	int i, hdr_done = 0;
	const char *splitfn = 0, *discfn = 0;
	int64_t total = 0;
	line_t *block = 0, *tail = 0;
	memset(&st, 0, sizeof st);
	st.maxSplitCount = 2; st.minNonOverlap = 20; st.minIndelSize = 50; st.maxUnmappedBases = 50;
	st.out = stdout;
	for (i = 1; i < argc; ++i) {
		if (!strcmp(argv[i], "--excludeDups") || !strcmp(argv[i], "-e")) st.excludeDups = 1;
		else if (!strcmp(argv[i], "--addMateTags")) st.addMateTags = 1;
		else if (!strcmp(argv[i], "--removeDups") || !strcmp(argv[i], "-r")) st.removeDups = 1;
		else if (!strcmp(argv[i], "--acceptDupMarks") || !strcmp(argv[i], "-a")) st.acceptDups = 1;
		else if (!strcmp(argv[i], "--maxSplitCount") && i + 1 < argc) st.maxSplitCount = atoi(argv[++i]);
		else if (!strcmp(argv[i], "--minNonOverlap") && i + 1 < argc) st.minNonOverlap = atoi(argv[++i]);
		else if (!strcmp(argv[i], "--minIndelSize") && i + 1 < argc) st.minIndelSize = atoi(argv[++i]);
		else if (!strcmp(argv[i], "--maxUnmappedBases") && i + 1 < argc) st.maxUnmappedBases = atoi(argv[++i]);
		else if ((!strcmp(argv[i], "--splitterFile") || !strcmp(argv[i], "-s")) && i + 1 < argc) splitfn = argv[++i];
		else if ((!strcmp(argv[i], "--discordantFile") || !strcmp(argv[i], "-d")) && i + 1 < argc) discfn = argv[++i];
		else if ((!strcmp(argv[i], "-i") || !strcmp(argv[i], "--input")) && i + 1 < argc) { if (!freopen(argv[++i], "r", stdin)) return 1; }
		else if ((!strcmp(argv[i], "-o") || !strcmp(argv[i], "--output")) && i + 1 < argc) { if (!(st.out = fopen(argv[++i], "w"))) return 1; }
		else if (!strcmp(argv[i], "samblaster")) continue;
		else { fprintf(stderr, "samblaster: Unrecognized option: %s\n", argv[i]); return 1; }
	}
	fprintf(stderr, "samblaster: Version %s\n", SB_VERSION);
	/* both side files are FIFOs in speedseq (bin/speedseq:408-416): open them up front, stream into them */
	if (discfn && !(st.disc = fopen(discfn, "w"))) { fprintf(stderr, "samblaster: Unable to open %s\n", discfn); return 1; }
	if (splitfn && !(st.split = fopen(splitfn, "w"))) { fprintf(stderr, "samblaster: Unable to open %s\n", splitfn); return 1; }
	cl = (char*)malloc(4096); strcpy(cl, "samblaster -i stdin -o stdout");
	if (st.excludeDups) strcat(cl, " --excludeDups");
	if (st.addMateTags) strcat(cl, " --addMateTags");
	if (discfn) { strcat(cl, " -d "); strncat(cl, discfn, 1500); }
	if (splitfn) { strcat(cl, " -s "); strncat(cl, splitfn, 1500); }
	if (splitfn) sprintf(cl + strlen(cl), " --maxSplitCount %d --maxUnmappedBases %d --minIndelSize %d --minNonOverlap %d", st.maxSplitCount, st.maxUnmappedBases, st.minIndelSize, st.minNonOverlap);
	while ((len = getline(&line, &cap, stdin)) > 0) {
		if (line[0] == '@' && !hdr_done) {
			if (strncmp(line, "@SQ\t", 4) == 0) {
				char name[1024] = "", *p = strstr(line, "\tSN:"), *q = strstr(line, "\tLN:");
				if (p && q) { sscanf(p + 4, "%1023[^\t\n]", name); seq_add(&st, name, atoll(q + 4), &total); }
			}
			fputs(line, st.out);
			if (st.disc) fputs(line, st.disc);
			if (st.split) fputs(line, st.split);
			continue;
		}
		if (!hdr_done) {
			FILE *fps[3] = {st.out, st.disc, st.split};
			for (i = 0; i < 3; ++i) if (fps[i]) fprintf(fps[i], "@PG\tID:SAMBLASTER\tVN:%s\tCL:%s\n", SB_VERSION, cl);
			hdr_done = 1;
		}
		{
			line_t *l = line_parse(strdup(line));
			if (block && strcmp(block->f[0], l->f[0]) != 0) {
				line_t *n;
				process_block(block, &st);
				for (; block; block = n) { n = block->next; line_free(block); }
				tail = 0;
			}
			if (!block) block = tail = l; else { tail->next = l; tail = l; }
		}
	}
	if (!hdr_done) {
		FILE *fps[3] = {st.out, st.disc, st.split};
		for (i = 0; i < 3; ++i) if (fps[i]) fprintf(fps[i], "@PG\tID:SAMBLASTER\tVN:%s\tCL:%s\n", SB_VERSION, cl);
	}
	if (block) {
		line_t *n;
		process_block(block, &st);
		for (; block; block = n) { n = block->next; line_free(block); }
	}
	fflush(st.out);
	if (st.disc) fclose(st.disc);
	if (st.split) fclose(st.split);
	if (st.disc) fprintf(stderr, "samblaster: Output %lu discordant read pairs to %s\n", (unsigned long)(st.n_disc / 2), discfn);
	if (st.split) fprintf(stderr, "samblaster: Output %lu split reads to %s\n", (unsigned long)(st.n_split / 2), splitfn);
	fprintf(stderr, "samblaster: Marked %lu of %lu (%.2f%%) read ids as duplicates.\n", (unsigned long)st.n_dup, (unsigned long)st.n_ids, st.n_ids ? 100.0 * st.n_dup / st.n_ids : 0.0);
	free(line); free(cl);
	for (i = 0; i < st.n_seq; ++i) free(st.names[i]);
	free(st.names); free(st.offs); free(st.sigs.keys); free(st.sigs.used);
	return 0;
}
