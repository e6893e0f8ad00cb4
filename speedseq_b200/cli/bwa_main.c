/*
 * bwa — drop-in for the `$BWA` entry of speedseq.config (speedseq/bin/speedseq.config:13), a thin C shim over
 * libssq.so.  Honours the argv/stdio contract of the reference's call sites:
 *     $BWA index REF                                              speedseq/bin/speedseq:389
 *     $BWA mem -t T [-p] [-C] [-I f[,f[,i[,i]]]] -R '@RG\tID:..' REF FQ1 [FQ2]   speedseq:438,468,1961
 * stdout = SAM (header, then records name-grouped in input order).  All base-level work AND the SAM text come from the GPU
 * (ssq_index_build, ssq_aligner_run: include/ssq.h); this file parses argv, tokenises FASTQ straight into the concatenated
 * layout the aligner takes, forms batches the way the reference's `bwa mem` does (bases >= 10 M x T and an even read count), and
 * writes what comes back.
 * FASTQ tokenisation follows the reference's in-tree parser speedseq/src/samtools-1.3.1/htslib-1.3.1/htslib/kseq.h:189-231.
 *
 * Fused mode.  speedseq pipes `$BWA mem | $SAMBLASTER ...` (speedseq:438-439).  When the environment variable
 * SSQ_FUSE_SAMBLASTER holds samblaster's option string (speedseq.config can export it from speedseq's own variables, see
 * INTEGRATION.md), this program also runs samblaster's stage on the device — duplicate marking, MC/MQ tags, discordant and
 * splitter selection — and writes the three record streams as length-prefixed frames behind a marker line; the `samblaster` shim
 * recognises the marker, checks that its own argv asks for the same options, and only routes the frames to stdout and to the two
 * side files.  Without the variable the output is plain `bwa mem` SAM and `samblaster` does its own work.
 */
#include <ctype.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <pthread.h>
#include <unistd.h>
#include <zlib.h>
#include "ssq.h"
#include "ssq_fuse.h"

#define SHIM_VERSION "0.7.12-r1039" /* the bwa release whose behaviour libssq reproduces (DESIGN.md §3) */

/* ---------------------------------------------------------------- FASTQ/FASTA reader ---- */
typedef struct { gzFile fp; unsigned char *buf; int beg, end, eof, last; } fq_t;
typedef struct { char *s; size_t l, m; } str_t;
typedef struct { str_t name, comment, seq, qual; } rec_t;

/* raw text of an input for the device tokeniser (ssq_aligner_upload_fastq): page-locked, refilled from the (possibly gzipped) file */
typedef struct { gzFile fp; char *buf; size_t len, cap; int eof; } raw_t;
static int raw_open(raw_t *r, const char *fn)
{
	memset(r, 0, sizeof *r);
	r->fp = strcmp(fn, "-") ? gzopen(fn, "r") : gzdopen(0, "r");
	if (!r->fp) return -1;
	gzbuffer(r->fp, 1 << 20);
	return 0;
}
static void raw_fill(raw_t *r, size_t want)
{
	while (!r->eof && r->len < want) {
		int n;
		if (r->cap < want) {
			const size_t ncap = want + want / 4;
			char *nb = (char*)ssq_host_alloc(ncap);
			if (!nb) { fprintf(stderr, "[E::bwa] cannot allocate %zu bytes of page-locked memory\n", ncap); exit(1); }
			if (r->len) memcpy(nb, r->buf, r->len);
			ssq_host_free(r->buf); r->buf = nb; r->cap = ncap;
		}
		n = gzread(r->fp, r->buf + r->len, (unsigned)((r->cap - r->len) < (1u << 30) ? (r->cap - r->len) : (1u << 30)));
		if (n <= 0) r->eof = 1; else r->len += (size_t)n;
	}
}
/* hand the rest of a raw reader (its unconsumed bytes, then the file) to the host tokeniser */
static fq_t *fq_from_raw(raw_t *r)
{
	fq_t *f = (fq_t*)calloc(1, sizeof(fq_t));
	const size_t cap = r->len > (1u << 18) ? r->len : (1u << 18);
	f->fp = r->fp; f->buf = (unsigned char*)malloc(cap);
	if (r->len) memcpy(f->buf, r->buf, r->len);
	f->beg = 0; f->end = (int)r->len; f->eof = 0; /* a further gzread reports the end again */
	ssq_host_free(r->buf); r->buf = 0; r->len = r->cap = 0;
	return f;
}
static inline int fq_getc(fq_t *f)
{
	if (f->beg >= f->end) {
		if (f->eof) return -1;
		f->beg = 0; f->end = gzread(f->fp, f->buf, 1 << 18);
		if (f->end <= 0) { f->eof = 1; f->end = 0; return -1; }
	}
	return f->buf[f->beg++];
}
static inline void s_reserve(str_t *s, size_t add) { if (s->l + add + 1 > s->m) { s->m = (s->l + add + 1) * 2; s->s = (char*)realloc(s->s, s->m); } }
static inline void s_push(str_t *s, int c) { s_reserve(s, 1); s->s[s->l++] = (char)c; s->s[s->l] = 0; }
static inline void s_clear(str_t *s) { s->l = 0; if (!s->s) { s->m = 256; s->s = (char*)malloc(s->m); } s->s[0] = 0; }
static int fq_line(fq_t *f, str_t *s) /* appends the rest of the current line, returns -1 at EOF with nothing read */
{
	int got = 0;
	for (;;) {
		unsigned char *p, *e;
		if (f->beg >= f->end) { int c = fq_getc(f); if (c < 0) break; --f->beg; }
		got = 1;
		p = f->buf + f->beg; e = (unsigned char*)memchr(p, '\n', (size_t)(f->end - f->beg));
		if (e) { s_reserve(s, (size_t)(e - p)); memcpy(s->s + s->l, p, (size_t)(e - p)); s->l += (size_t)(e - p); s->s[s->l] = 0; f->beg += (int)(e - p) + 1; break; }
		s_reserve(s, (size_t)(f->end - f->beg)); memcpy(s->s + s->l, p, (size_t)(f->end - f->beg)); s->l += (size_t)(f->end - f->beg); s->s[s->l] = 0; f->beg = f->end;
	}
	if (s->l && s->s[s->l - 1] == '\r') s->s[--s->l] = 0;
	return got ? 0 : -1;
}
/* >= 0: sequence length; -1: end of file; -2: truncated quality */
static int fq_read(fq_t *f, rec_t *r)
{
	int c;
	if (f->last == 0) {
		while ((c = fq_getc(f)) >= 0 && c != '>' && c != '@');
		if (c < 0) return -1;
		f->last = c;
	}
	s_clear(&r->name); s_clear(&r->comment); s_clear(&r->seq); s_clear(&r->qual);
	while ((c = fq_getc(f)) >= 0 && !isspace(c)) s_push(&r->name, c);
	if (c < 0 && r->name.l == 0) return -1;
	if (c >= 0 && c != '\n') fq_line(f, &r->comment);
	while ((c = fq_getc(f)) >= 0 && c != '>' && c != '+' && c != '@') {
		if (c == '\n') continue;
		s_push(&r->seq, c);
		fq_line(f, &r->seq);
	}
	if (c == '>' || c == '@') f->last = c;
	if (c != '+') { if (c < 0) f->last = 0; return (int)r->seq.l; }
	while ((c = fq_getc(f)) >= 0 && c != '\n');
	if (c < 0) return -2;
	while (r->qual.l < r->seq.l && fq_line(f, &r->qual) == 0);
	f->last = 0;
	return r->seq.l == r->qual.l ? (int)r->seq.l : -2;
}

/* --------------------------------------------------------------------------- batches ---- */
/* one batch in the aligner's layout: concatenated fields + offsets (ssq_reads_t) */
typedef struct {
	str_t seq, qual, name, cmt;
	uint64_t *seq_off; uint32_t *name_off, *cmt_off;
	int n, m, all_qual, any_cmt;
} blob_t;

static void blob_clear(blob_t *b) { b->seq.l = b->qual.l = b->name.l = b->cmt.l = 0; b->n = 0; b->all_qual = 1; b->any_cmt = 0; }
static void trim_readno(str_t *s) { if (s->l > 2 && s->s[s->l - 2] == '/' && isdigit((unsigned char)s->s[s->l - 1])) { s->l -= 2; s->s[s->l] = 0; } }
static void blob_push(blob_t *b, const char *name, size_t ln, const char *seq, size_t ls, const char *qual, size_t lq, const char *cmt, size_t lc)
{
	if (b->n + 2 > b->m) {
		b->m = b->m ? b->m * 2 : 1 << 16;
		b->seq_off = (uint64_t*)realloc(b->seq_off, sizeof(uint64_t) * (b->m + 1)); b->name_off = (uint32_t*)realloc(b->name_off, 4 * (b->m + 1)); b->cmt_off = (uint32_t*)realloc(b->cmt_off, 4 * (b->m + 1));
	}
	if (b->n == 0) { b->seq_off[0] = 0; b->name_off[0] = 0; b->cmt_off[0] = 0; }
	s_reserve(&b->seq, ls); memcpy(b->seq.s + b->seq.l, seq, ls); b->seq.l += ls;
	s_reserve(&b->qual, ls);
	if (lq == ls && ls) memcpy(b->qual.s + b->qual.l, qual, ls); else { memset(b->qual.s + b->qual.l, '*', ls); if (ls) b->all_qual = 0; }
	b->qual.l += ls;
	s_reserve(&b->name, ln); memcpy(b->name.s + b->name.l, name, ln); b->name.l += ln;
	if (lc) { s_reserve(&b->cmt, lc); memcpy(b->cmt.s + b->cmt.l, cmt, lc); b->cmt.l += lc; b->any_cmt = 1; }
	++b->n;
	b->seq_off[b->n] = b->seq.l; b->name_off[b->n] = (uint32_t)b->name.l; b->cmt_off[b->n] = (uint32_t)b->cmt.l;
}
static void blob_push_rec(blob_t *b, const rec_t *r, int keep_comment)
{
	blob_push(b, r->name.s, r->name.l, r->seq.s, r->seq.l, r->qual.s, r->qual.l, r->comment.s, keep_comment ? r->comment.l : 0);
}
static void blob_push_from(blob_t *b, const blob_t *src, int i)
{
	const size_t ls = (size_t)(src->seq_off[i + 1] - src->seq_off[i]);
	if (!src->all_qual) b->all_qual = 0; /* mixed inputs: a read without qualities makes the sub-batch quality-less, like the parent */
	blob_push(b, src->name.s + src->name_off[i], src->name_off[i + 1] - src->name_off[i], src->seq.s + src->seq_off[i], ls, src->qual.s + src->seq_off[i], ls,
	          src->cmt.s + src->cmt_off[i], src->cmt_off[i + 1] - src->cmt_off[i]);
}

/* one batch: until the base count reaches chunk and the read count is even */
static long read_batch(long chunk, fq_t *f1, fq_t *f2, rec_t *r1, rec_t *r2, blob_t *v, int keep_comment)
{
	long size = 0;
	blob_clear(v);
	while (fq_read(f1, r1) >= 0) {
		if (f2 && fq_read(f2, r2) < 0) { fprintf(stderr, "[W::bseq_read] the 2nd file has fewer sequences.\n"); break; }
		trim_readno(&r1->name); blob_push_rec(v, r1, keep_comment); size += (long)r1->seq.l;
		if (f2) { trim_readno(&r2->name); blob_push_rec(v, r2, keep_comment); size += (long)r2->seq.l; }
		if (size >= chunk && (v->n & 1) == 0) break;
	}
	if (size == 0 && f2 && fq_read(f2, r2) >= 0) fprintf(stderr, "[W::bseq_read] the 1st file has fewer sequences.\n");
	return size;
}

static void die(const char *what, int rc) { fprintf(stderr, "[E::bwa] %s failed (%d): %s\n", what, rc, ssq_last_error()); exit(1); }
static int same_name(const blob_t *v, int i, int j)
{
	const uint32_t li = v->name_off[i + 1] - v->name_off[i], lj = v->name_off[j + 1] - v->name_off[j];
	return li == lj && memcmp(v->name.s + v->name_off[i], v->name.s + v->name_off[j], li) == 0;
}
static void fill_reads(ssq_reads_t *rd, const blob_t *b, int paired, long long n_processed)
{
	memset(rd, 0, sizeof *rd);
	rd->n_reads = b->n; rd->paired = paired; rd->seq = b->seq.s; rd->seq_off = b->seq_off; rd->qual = b->all_qual && b->n ? b->qual.s : 0;
	rd->name = b->name.s; rd->name_off = b->name_off; rd->comment = b->any_cmt ? b->cmt.s : 0; rd->comment_off = b->any_cmt ? b->cmt_off : 0; rd->n_processed = n_processed;
}
static void check_pair_names(const blob_t *b)
{
	int i;
	for (i = 0; i + 1 < b->n; i += 2)
		if (!same_name(b, i, i + 1)) {
			fprintf(stderr, "[E::mem_sam_pe] paired reads have different names: \"%.*s\", \"%.*s\"\n", (int)(b->name_off[i + 1] - b->name_off[i]), b->name.s + b->name_off[i],
			        (int)(b->name_off[i + 2] - b->name_off[i + 1]), b->name.s + b->name_off[i + 1]);
			exit(1);
		}
}

static char *unescape(char *s)
{
	char *p, *q;
	for (p = q = s; *p; ++p) {
		if (*p == '\\') {
			++p;
			if (*p == 't') *q++ = '\t'; else if (*p == 'n') *q++ = '\n'; else if (*p == 'r') *q++ = '\r'; else if (*p == '\\') *q++ = '\\'; else if (*p == 0) break;
		} else *q++ = *p;
	}
	*q = 0;
	return s;
}

static int g_bam; /* SSQ_FUSE_BAM: the main records leave as coordinate-sorted BAM runs (ssq_fuse.h) */

static void put_frame(int stream, const char *p, size_t len)
{
	ssq_frame_hdr_t h;
	if (!len) return;
	memcpy(h.magic, SSQ_FRAME_MAGIC, 8); h.stream = (uint64_t)stream; h.len = (uint64_t)len;
	fwrite(&h, sizeof h, 1, stdout); fwrite(p, 1, len, stdout);
}

/* BAM mode: out->text[0] / len[0] = the batch's main records as one sorted BAM run, text[1..2] = the side streams as SAM text */
static int fetch_bam_mode(ssq_aligner_t *al, ssq_sam_t *out)
{
	const void *b = 0; size_t bl = 0; int rc, k;
	memset(out, 0, sizeof *out);
	if ((rc = ssq_aligner_fetch_bam(al, 0, &b, &bl))) return rc;
	out->text[0] = (const char*)b; out->len[0] = bl;
	for (k = 1; k < 3; ++k) { const char *t = 0; size_t l = 0; if ((rc = ssq_aligner_fetch_text(al, k, &t, &l))) return rc; out->text[k] = t; out->len[k] = l; }
	return 0;
}

/* ------------------------------------------------------------------- stream lanes ----
 * Device-ingest mode runs SSQ_LANES (default 2) lanes, each a host thread with its own aligner object (own CUDA stream and
 * buffers): while one lane's batch is on the GPU, the other reads and uploads the next text and writes the previous records —
 * the read / compute / write overlap of upstream bwa's three-stage pipeline.  Batches are cut one after the other under a lock
 * (where a batch ends is only known once the device has parsed the text), records are written strictly in batch order (tickets),
 * and in fused mode the lanes share one dup-set whose turn counter keeps "first seen wins" in input order. */
typedef struct {
	raw_t *R1, *R2; int two_files, smart_pe, paired, keep_comment, fused; long chunk; const ssq_pestat_t *pes0;
	size_t raw_target; long long n_processed, next_ticket, write_turn;
	int stop, fallback, failed, shared_set;
	pthread_mutex_t rd_mu, wr_mu; pthread_cond_t wr_cv;
} lanes_t;
typedef struct { lanes_t *S; ssq_aligner_t *al; } lane_arg_t;

static void *lane_main(void *arg_)
{
	lane_arg_t *arg = (lane_arg_t*)arg_;
	lanes_t *S = arg->S;
	ssq_aligner_t *al = arg->al;
	for (;;) {
		size_t u1 = 0, u2 = 0;
		int n = 0, more = 0, rc;
		long long ticket;
		ssq_sam_t out;
		pthread_mutex_lock(&S->rd_mu);
		if (S->stop) { pthread_mutex_unlock(&S->rd_mu); break; }
		raw_fill(S->R1, S->raw_target);
		if (S->two_files) raw_fill(S->R2, S->raw_target);
		rc = ssq_aligner_upload_fastq(al, S->R1->buf ? S->R1->buf : "", S->R1->len, S->R1->eof, S->two_files ? (S->R2->buf ? S->R2->buf : "") : 0, S->two_files ? S->R2->len : 0,
		                              S->two_files ? S->R2->eof : 1, S->smart_pe, S->keep_comment, S->chunk, S->n_processed, &u1, &u2, &n, &more);
		if (rc == SSQ_EFORMAT) { /* every other legal input: multi-line records, FASTA, unpaired reads among the pairs, ... */
			if (getenv("SSQ_VERBOSE_INGEST")) fprintf(stderr, "[M::bwa] host tokeniser takes over: %s\n", ssq_last_error());
			S->fallback = 1; S->stop = 1; pthread_mutex_unlock(&S->rd_mu); break;
		}
		if (rc) { fprintf(stderr, "[E::bwa] ssq_aligner_upload_fastq failed (%d): %s\n", rc, ssq_last_error()); S->failed = 1; S->stop = 1; pthread_mutex_unlock(&S->rd_mu); break; }
		if (more) { S->raw_target += S->raw_target / 2; pthread_mutex_unlock(&S->rd_mu); continue; }
		if (n == 0) { S->stop = 1; pthread_mutex_unlock(&S->rd_mu); break; }
		ticket = S->next_ticket++;
		S->n_processed += n;
		memmove(S->R1->buf, S->R1->buf + u1, S->R1->len - u1); S->R1->len -= u1;
		if (S->two_files) { memmove(S->R2->buf, S->R2->buf + u2, S->R2->len - u2); S->R2->len -= u2; }
		fprintf(stderr, "[M::process] read %d sequences (%ld bp)...\n", n, (long)ssq_aligner_counter(al, 109));
		if (S->smart_pe) fprintf(stderr, "[M::process] 0 single-end sequences; %d paired-end sequences\n", n);
		pthread_mutex_unlock(&S->rd_mu);
		ssq_aligner_set_turn(al, S->shared_set ? ticket : -1);
		rc = ssq_aligner_compute(al, S->paired ? S->pes0 : 0, 1);
		if (!rc && g_bam) rc = fetch_bam_mode(al, &out);
		else if (!rc) rc = ssq_aligner_fetch(al, &out);
		pthread_mutex_lock(&S->wr_mu);
		while (S->write_turn != ticket) pthread_cond_wait(&S->wr_cv, &S->wr_mu);
		if (rc) { fprintf(stderr, "[E::bwa] batch %lld failed (%d): %s\n", ticket, rc, ssq_last_error()); S->failed = 1; }
		else if (!S->failed) {
			if (S->fused) { put_frame(g_bam ? SSQ_STREAM_BAM_RUN : 0, out.text[0], out.len[0]); put_frame(1, out.text[1], out.len[1]); put_frame(2, out.text[2], out.len[2]); }
			else fwrite(out.text[0], 1, out.len[0], stdout);
		}
		++S->write_turn;
		pthread_cond_broadcast(&S->wr_cv);
		pthread_mutex_unlock(&S->wr_mu);
		if (rc) { pthread_mutex_lock(&S->rd_mu); S->stop = 1; pthread_mutex_unlock(&S->rd_mu); break; }
	}
	return 0;
}

static int main_mem(int argc, char **argv, const char *prog)
{
	ssq_opts_t opt;
	ssq_sb_opts_t sb;
	ssq_pestat_t pes[4], *pes0 = 0;
	ssq_index_t *idx = 0;
	ssq_aligner_t *al = 0;
	fq_t *f1 = 0, *f2 = 0;
	raw_t R1, R2;
	rec_t r1, r2;
	int dev_ingest = 0, two_files = 0;
	size_t raw_target;
	blob_t v, se, pe;
	char *rg_line = 0, rg_id[256] = "", *p, fuse_opts[1024] = "";
	int c, i, n_threads = 1, smart_pe = 0, paired = 0, keep_comment = 0, device = getenv("SSQ_DEVICE") ? atoi(getenv("SSQ_DEVICE")) : 0, rc, fused = 0;
	long long n_processed = 0;
	const long chunk_size = 10000000;
	memset(&r1, 0, sizeof r1); memset(&r2, 0, sizeof r2); memset(pes, 0, sizeof pes); memset(&v, 0, sizeof v); memset(&se, 0, sizeof se); memset(&pe, 0, sizeof pe);
	pes[0].failed = pes[1].failed = pes[2].failed = pes[3].failed = 1;
	ssq_opts_default(&opt);
	ssq_sb_opts_default(&sb);
	while ((c = getopt(argc, argv, "t:pR:I:Cv:")) >= 0) {
		if (c == 't') n_threads = atoi(optarg) > 1 ? atoi(optarg) : 1;
		else if (c == 'p') smart_pe = paired = 1;
		else if (c == 'C') keep_comment = 1;
		else if (c == 'v') ;
		else if (c == 'R') {
			if (strstr(optarg, "@RG") != optarg) { fprintf(stderr, "[E::bwa_set_rg] the read group line is not started with @RG\n"); return 1; }
			rg_line = unescape(strdup(optarg));
			if (!(p = strstr(rg_line, "\tID:"))) { fprintf(stderr, "[E::bwa_set_rg] no ID at the read group line\n"); return 1; }
			for (p += 4, i = 0; p[i] && p[i] != '\t' && p[i] != '\n' && i < 255; ++i) rg_id[i] = p[i];
			rg_id[i] = 0;
		} else if (c == 'I') { /* mean[,std[,max[,min]]] for the FR orientation */
			pes0 = pes; pes[1].failed = 0;
			pes[1].avg = strtod(optarg, &p); pes[1].std = pes[1].avg * .1;
			if (*p && ispunct((unsigned char)*p) && isdigit((unsigned char)p[1])) pes[1].std = strtod(p + 1, &p);
			pes[1].high = (int)(pes[1].avg + 4. * pes[1].std + .499);
			pes[1].low = (int)(pes[1].avg - 4. * pes[1].std + .499);
			if (pes[1].low < 1) pes[1].low = 1;
			if (*p && ispunct((unsigned char)*p) && isdigit((unsigned char)p[1])) pes[1].high = (int)(strtod(p + 1, &p) + .499);
			if (*p && ispunct((unsigned char)*p) && isdigit((unsigned char)p[1])) pes[1].low = (int)(strtod(p + 1, &p) + .499);
		} else return 1;
	}
	opt.n_threads = n_threads;
	if (optind + 1 >= argc || optind + 3 < argc) { fprintf(stderr, "Usage: bwa mem [-t INT] [-p] [-C] [-I FLOAT[,FLOAT[,INT[,INT]]]] [-R STR] <idxbase> <in1.fq> [in2.fq]\n"); return 1; }
	if (getenv("SSQ_FUSE_SAMBLASTER") && getenv("SSQ_FUSE_SAMBLASTER")[0]) { /* samblaster's options: its stage runs here, on the device */
		char tmp[1024], *tok;
		snprintf(tmp, sizeof tmp, "%s", getenv("SSQ_FUSE_SAMBLASTER"));
		fused = 1; sb.enabled = 1; sb.want_split = sb.want_disc = 1;
		for (tok = strtok(tmp, " \t"); tok; tok = strtok(0, " \t")) {
			if (!strcmp(tok, "--excludeDups") || !strcmp(tok, "-e")) sb.exclude_dups = 1;
			else if (!strcmp(tok, "--addMateTags")) sb.add_mate_tags = 1;
			else if (!strcmp(tok, "--removeDups") || !strcmp(tok, "-r")) sb.remove_dups = 1;
			else if (!strcmp(tok, "--maxSplitCount")) { if ((tok = strtok(0, " \t"))) sb.max_split_count = atoi(tok); }
			else if (!strcmp(tok, "--minNonOverlap")) { if ((tok = strtok(0, " \t"))) sb.min_non_overlap = atoi(tok); }
			else if (!strcmp(tok, "--minIndelSize")) { if ((tok = strtok(0, " \t"))) sb.min_indel_size = atoi(tok); }
			else if (!strcmp(tok, "--maxUnmappedBases")) { if ((tok = strtok(0, " \t"))) sb.max_unmapped_bases = atoi(tok); }
			else { fprintf(stderr, "[E::bwa] SSQ_FUSE_SAMBLASTER: option '%s' is not one the fused stage implements\n", tok); return 1; }
		}
		ssq_fuse_describe(fuse_opts, sizeof fuse_opts, sb.exclude_dups, sb.add_mate_tags, sb.remove_dups, sb.max_split_count, sb.min_non_overlap, sb.min_indel_size, sb.max_unmapped_bases);
		g_bam = getenv("SSQ_FUSE_BAM") && atoi(getenv("SSQ_FUSE_BAM"));
	} else if (getenv("SSQ_FUSE_BAM") && atoi(getenv("SSQ_FUSE_BAM"))) { fprintf(stderr, "[E::bwa] SSQ_FUSE_BAM needs the fused samblaster stage (SSQ_FUSE_SAMBLASTER)\n"); return 1; }
	if ((rc = ssq_index_load(argv[optind], device, &idx))) die("ssq_index_load", rc);
	if ((rc = ssq_aligner_create(idx, &opt, fused ? &sb : 0, rg_id, &al))) die("ssq_aligner_create", rc);
	if (g_bam && (rc = ssq_aligner_set_bam(al, 1, 1))) die("ssq_aligner_set_bam", rc);
	if (raw_open(&R1, argv[optind + 1])) { fprintf(stderr, "[E::main_mem] fail to open file `%s'.\n", argv[optind + 1]); return 1; }
	if (optind + 2 < argc) {
		if (smart_pe) fprintf(stderr, "[W::main_mem] when '-p' is in use, the second query file is ignored.\n");
		else { if (raw_open(&R2, argv[optind + 2])) { fprintf(stderr, "[E::main_mem] fail to open file `%s'.\n", argv[optind + 2]); return 1; } paired = 1; two_files = 1; }
	}
	dev_ingest = !(getenv("SSQ_HOST_FASTQ") && atoi(getenv("SSQ_HOST_FASTQ"))); /* the device tokenises; the host tokeniser takes over when the text is not four-line FASTQ */
	if (!dev_ingest) { f1 = fq_from_raw(&R1); if (two_files) f2 = fq_from_raw(&R2); }
	{ /* header: @SQ from the index, @RG as given, @PG with the command line */
		const int ns = (int)ssq_index_info(idx, 3);
		static char obuf[1 << 22];
		setvbuf(stdout, obuf, _IOFBF, sizeof obuf);
		for (i = 0; i < ns; ++i) { int64_t len; const char *nm = ssq_index_contig(idx, i, &len); printf("@SQ\tSN:%s\tLN:%lld\n", nm, (long long)len); }
		if (rg_line) printf("%s\n", rg_line);
		printf("@PG\tID:bwa\tPN:bwa\tVN:%s\tCL:%s", SHIM_VERSION, prog);
		for (i = 0; i < argc; ++i) printf(" %s", argv[i]);
		printf("\n");
		if (fused) printf("%s%s%s\n", SSQ_FUSE_MARKER, fuse_opts, g_bam ? "\tbam" : "");
	}
	if (!two_files) memset(&R2, 0, sizeof R2);
	raw_target = (size_t)((double)chunk_size * n_threads * 2.7 / (two_files ? 2 : 1)) + (1u << 20); /* bytes of text one batch is expected to span */
	for (;;) {
		long size;
		ssq_reads_t rd;
		ssq_sam_t out;
		int n_se = 0, n_pe = 0, mixed = 0;
		if (dev_ingest) { /* FASTQ text -> device -> records, in lanes (see lane_main) */
			lanes_t S;
			lane_arg_t la[4];
			pthread_t th[4];
			ssq_dupset_t *dset = 0;
			int n_lanes = getenv("SSQ_LANES") ? atoi(getenv("SSQ_LANES")) : 2, k;
			if (n_lanes < 1) n_lanes = 1;
			if (n_lanes > 4) n_lanes = 4;
			memset(&S, 0, sizeof S);
			S.R1 = &R1; S.R2 = &R2; S.two_files = two_files; S.smart_pe = smart_pe; S.paired = paired; S.keep_comment = keep_comment; S.fused = fused; S.chunk = chunk_size * n_threads;
			S.pes0 = pes0; S.raw_target = raw_target; S.n_processed = n_processed;
			pthread_mutex_init(&S.rd_mu, 0); pthread_mutex_init(&S.wr_mu, 0); pthread_cond_init(&S.wr_cv, 0);
			if (n_lanes > 1 && (rc = ssq_dupset_create(device, &dset))) die("ssq_dupset_create", rc); /* shared by the lanes: its turn counter orders their batches (the signatures only matter in fused mode) */
			S.shared_set = dset != 0;
			for (k = 0; k < n_lanes; ++k) {
				la[k].S = &S; la[k].al = al;
				if (k > 0 && (rc = ssq_aligner_create(idx, &opt, fused ? &sb : 0, rg_id, &la[k].al))) die("ssq_aligner_create", rc);
				if (k > 0 && g_bam && (rc = ssq_aligner_set_bam(la[k].al, 1, 1))) die("ssq_aligner_set_bam", rc);
				if (dset && (rc = ssq_aligner_share_dupset(la[k].al, dset))) die("ssq_aligner_share_dupset", rc);
			}
			fflush(stdout);
			for (k = 0; k < n_lanes; ++k) pthread_create(&th[k], 0, lane_main, &la[k]);
			for (k = 0; k < n_lanes; ++k) pthread_join(th[k], 0);
			for (k = 1; k < n_lanes; ++k) ssq_aligner_free(la[k].al);
			if (S.failed) return 1;
			n_processed = S.n_processed;
			dev_ingest = 0;
			if (!S.fallback) break; /* input exhausted */
			ssq_aligner_set_turn(al, -1); /* the host tokeniser continues on the first aligner (it keeps the shared dup-set alive until the end) */
			f1 = fq_from_raw(&R1); if (two_files) f2 = fq_from_raw(&R2);
			continue;
		}
		size = read_batch(chunk_size * n_threads, f1, f2, &r1, &r2, &v, keep_comment);
		if (v.n == 0) break;
		fprintf(stderr, "[M::process] read %d sequences (%ld bp)...\n", v.n, size);
		if (smart_pe) { /* interleaved input: adjacent reads with equal names are mates, the others single-end */
			int has_last = 1;
			for (i = 1; i < v.n; ++i) {
				if (has_last) { if (same_name(&v, i, i - 1)) { n_pe += 2; has_last = 0; } else ++n_se; }
				else has_last = 1;
			}
			if (has_last) ++n_se;
			fprintf(stderr, "[M::process] %d single-end sequences; %d paired-end sequences\n", n_se, n_pe);
			mixed = n_se && n_pe;
		} else if (paired) n_pe = v.n; else n_se = v.n;
		if (!mixed) { /* the whole batch is one call; its text is already in input order */
			if (n_pe) check_pair_names(&v);
			fill_reads(&rd, &v, n_pe ? 1 : 0, n_processed);
			if ((rc = ssq_aligner_run(al, &rd, n_pe ? pes0 : 0, 1, &out))) die("ssq_aligner_run", rc);
			if (g_bam && (rc = fetch_bam_mode(al, &out))) die("ssq_aligner_fetch_bam", rc);
			if (fused) { put_frame(g_bam ? SSQ_STREAM_BAM_RUN : 0, out.text[0], out.len[0]); put_frame(1, out.text[1], out.len[1]); put_frame(2, out.text[2], out.len[2]); }
			else fwrite(out.text[0], 1, out.len[0], stdout);
		} else { /* single-end reads first, then the pairs (the reference's order of work); records go out in input order */
			int *id_se = (int*)malloc(sizeof(int) * v.n), *id_pe = (int*)malloc(sizeof(int) * v.n), has_last = 1, k_se = 0, k_pe = 0;
			char **txt = (char**)calloc(v.n, sizeof(char*)); size_t *len = (size_t*)calloc(v.n, sizeof(size_t));
			if (fused) { fprintf(stderr, "[E::bwa] interleaved input with unpaired reads in one batch cannot go through the fused samblaster stage; unset SSQ_FUSE_SAMBLASTER\n"); return 1; }
			blob_clear(&se); blob_clear(&pe);
			for (i = 1; i < v.n; ++i) {
				if (has_last) {
					if (same_name(&v, i, i - 1)) { id_pe[k_pe++] = i - 1; id_pe[k_pe++] = i; blob_push_from(&pe, &v, i - 1); blob_push_from(&pe, &v, i); has_last = 0; }
					else { id_se[k_se++] = i - 1; blob_push_from(&se, &v, i - 1); }
				} else has_last = 1;
			}
			if (has_last) { id_se[k_se++] = v.n - 1; blob_push_from(&se, &v, v.n - 1); }
			for (c = 0; c < 2; ++c) {
				const blob_t *b = c ? &pe : &se; const int *ids = c ? id_pe : id_se;
				fill_reads(&rd, b, c, n_processed + (c ? n_se : 0));
				if ((rc = ssq_aligner_run(al, &rd, c ? pes0 : 0, 1, &out))) die("ssq_aligner_run", rc);
				for (i = 0; i < b->n; ++i) { len[ids[i]] = (size_t)(out.read_off[i + 1] - out.read_off[i]); txt[ids[i]] = (char*)malloc(len[ids[i]] + 1); memcpy(txt[ids[i]], out.text[0] + out.read_off[i], len[ids[i]]); }
			}
			for (i = 0; i < v.n; ++i) { fwrite(txt[i], 1, len[i], stdout); free(txt[i]); }
			free(txt); free(len); free(id_se); free(id_pe);
		}
		n_processed += v.n;
	}
	fflush(stdout);
	ssq_aligner_free(al);
	ssq_index_free(idx);
	return 0;
}

static int main_index(int argc, char **argv)
{
	const char *prefix = 0, *fa = 0;
	int i, rc, device = getenv("SSQ_DEVICE") ? atoi(getenv("SSQ_DEVICE")) : 0;
	for (i = 1; i < argc; ++i) {
		if (!strcmp(argv[i], "-p") && i + 1 < argc) prefix = argv[++i];
		else if (!strcmp(argv[i], "-a") && i + 1 < argc) ++i; /* construction algorithm: the result is the same */
		else if (argv[i][0] != '-' && !fa) fa = argv[i];
	}
	if (!fa) { fprintf(stderr, "Usage: bwa index [-p prefix] <in.fasta>\n"); return 1; }
	if ((rc = ssq_index_build(fa, prefix ? prefix : fa, device))) die("ssq_index_build", rc);
	return 0;
}

int main(int argc, char **argv)
{
	if (argc < 2) { fprintf(stderr, "Usage: bwa <index|mem> [options]   (H100 shim over libssq, behaviour of bwa %s)\n", SHIM_VERSION); return 1; }
	if (!strcmp(argv[1], "index")) return main_index(argc - 1, argv + 1);
	if (!strcmp(argv[1], "mem")) return main_mem(argc - 1, argv + 1, argv[0]);
	fprintf(stderr, "[main] unrecognized command '%s'\n", argv[1]);
	return 1;
}
