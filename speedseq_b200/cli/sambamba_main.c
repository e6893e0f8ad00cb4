/* sambamba_main.c — the `sambamba` the pipeline's align step can be pointed at (speedseq.config `SAMBAMBA=`) when the `bwa` /
 * `samblaster` shims run in BAM mode (SSQ_FUSE_BAM, see ssq_fuse.h): the main records then arrive as coordinate-sorted runs of BAM
 * records made on the device instead of SAM text, and the two calls of speedseq/bin/speedseq:440-441
 *     $SAMBAMBA view -S -f bam -l 0 /dev/stdin | $SAMBAMBA sort -t T -m M --tmpdir=D -o out.bam /dev/stdin
 * become a pass-through and a merge of sorted runs:
 *   view : stdin that carries the run marker is copied to stdout unchanged;
 *   sort : the runs are merged by (reference, position, strand), equal keys in input order — the order sambamba's sort gives the
 *          whole input (tests/golden/syn3_bam_main: pinned on the reference's own sambamba) —, the header text is rewritten the way
 *          sambamba rewrites it (ssq_bam_header_text) and the result is written as BGZF to -o, compressed on -t threads.  Runs beyond
 *          the -m budget are merged and spilled to --tmpdir, like sambamba's own temporary files.
 * Everything else — other subcommands (index, merge, ...), and view / sort whose stdin is ordinary SAM / BAM (the splitter and
 * discordant streams, speedseq:444-448) — goes to the real sambamba named by SSQ_SAMBAMBA_REAL (or `sambamba.real` next to this
 * executable) with the bytes already read handed on, so one SAMBAMBA= line serves the whole script. */
#define _GNU_SOURCE
#include <errno.h>
#include <pthread.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/stat.h>
#include <sys/wait.h>
#include <unistd.h>
#include "ssq.h"
#include "ssq_fuse.h"

static const char *g_self;

static const char *real_path(void)
{
	static char buf[4096];
	const char *e = getenv("SSQ_SAMBAMBA_REAL");
	if (e && e[0]) return e;
	{ ssize_t n = readlink("/proc/self/exe", buf, sizeof buf - 16); if (n > 0) { buf[n] = 0; strcat(buf, ".real"); if (access(buf, X_OK) == 0) return buf; } }
	return 0;
}
static void need_real(const char *why)
{
	fprintf(stderr, "sambamba (GPU shim): %s needs the real sambamba: set SSQ_SAMBAMBA_REAL to its path (or install it as `sambamba.real` next to %s)\n", why, g_self);
	exit(1);
}
static void exec_real(char **argv, const char *why)
{
	const char *r = real_path();
	if (!r) need_real(why);
	execv(r, argv);
	fprintf(stderr, "sambamba (GPU shim): cannot execute %s: %s\n", r, strerror(errno));
	exit(1);
}
static int write_all(int fd, const void *p, size_t n)
{
	const char *c = (const char*)p;
	while (n) { ssize_t w = write(fd, c, n); if (w < 0) { if (errno == EINTR) continue; return -1; } c += w; n -= (size_t)w; }
	return 0;
}
/* the real program with our stdin: what was already read, then the rest */
static int feed_real(char **argv, const char *head, size_t n_head, const char *why)
{
	const char *r = real_path();
	int fd[2], st = 0;
	pid_t pid;
	static char buf[1 << 20];
	if (!r) need_real(why);
	if (pipe(fd)) { perror("pipe"); return 1; }
	pid = fork();
	if (pid < 0) { perror("fork"); return 1; }
	if (pid == 0) { dup2(fd[0], 0); close(fd[0]); close(fd[1]); execv(r, argv); fprintf(stderr, "sambamba (GPU shim): cannot execute %s: %s\n", r, strerror(errno)); _exit(127); }
	close(fd[0]);
	signal(SIGPIPE, SIG_IGN);
	if (write_all(fd[1], head, n_head) == 0) for (;;) { ssize_t n = read(0, buf, sizeof buf); if (n < 0 && errno == EINTR) continue; if (n <= 0) break; if (write_all(fd[1], buf, (size_t)n)) break; }
	close(fd[1]);
	while (waitpid(pid, &st, 0) < 0 && errno == EINTR) {}
	return WIFEXITED(st) ? WEXITSTATUS(st) : 1;
}

/* ---- what is on stdin?  Reads until it is known; the bytes stay in *head ---- */
typedef struct { char *p; size_t n, cap; int eof; } head_t;
static int head_more(head_t *h)
{
	ssize_t n;
	if (h->eof) return 0;
	if (h->n + (1 << 16) > h->cap) { h->cap = h->cap ? h->cap * 2 : 1 << 18; h->p = (char*)realloc(h->p, h->cap); }
	do n = read(0, h->p + h->n, h->cap - h->n); while (n < 0 && errno == EINTR);
	if (n <= 0) { h->eof = 1; return 0; }
	h->n += (size_t)n;
	return 1;
}
/* 1: SAM header text followed by the run marker (*body = offset of the first frame); 0: anything else */
static int sniff_runs(head_t *h, size_t *body)
{
	size_t at = 0;
	const size_t ml = strlen(SSQ_BAM_RUNS_MARKER);
	for (;;) {
		char *nl;
		while (at >= h->n) if (!head_more(h)) return 0;
		if (h->p[at] != '@') return 0;
		while (!(nl = (char*)memchr(h->p + at, '\n', h->n - at))) if (!head_more(h)) return 0;
		if ((size_t)(nl + 1 - (h->p + at)) == ml && !memcmp(h->p + at, SSQ_BAM_RUNS_MARKER, ml)) { *body = (size_t)(nl + 1 - h->p); return 1; }
		at = (size_t)(nl + 1 - h->p);
	}
}

/* ---- sorted runs: in memory or spilled; merged with a binary heap ---- */
typedef struct {
	const uint8_t *mem; size_t len, at;     /* in memory */
	FILE *fp; uint8_t *buf; size_t cap, fill, pos; /* or a spill file behind a window */
} src_t;
static const uint8_t *src_peek(src_t *s, size_t *rec_len)
{
	uint32_t bs;
	if (!s->fp) {
		if (s->at + 4 > s->len) return 0;
		memcpy(&bs, s->mem + s->at, 4);
		if (bs < 32 || s->at + 4 + (size_t)bs > s->len) { fprintf(stderr, "sambamba (GPU shim): a run is not a sequence of BAM records\n"); exit(1); }
		*rec_len = 4 + (size_t)bs;
		return s->mem + s->at;
	}
	for (;;) {
		const size_t have = s->fill - s->pos;
		size_t want = 4;
		if (have >= 4) { memcpy(&bs, s->buf + s->pos, 4); want = 4 + (size_t)bs; if (have >= want) { *rec_len = want; return s->buf + s->pos; } }
		if (s->pos) { memmove(s->buf, s->buf + s->pos, have); s->fill = have; s->pos = 0; }
		if (want > s->cap) { s->cap = want * 2; s->buf = (uint8_t*)realloc(s->buf, s->cap); }
		{ const size_t n = fread(s->buf + s->fill, 1, s->cap - s->fill, s->fp); if (!n) { if (have) { fprintf(stderr, "sambamba (GPU shim): truncated spill file\n"); exit(1); } return 0; } s->fill += n; }
	}
}
static void src_advance(src_t *s, size_t rec_len) { if (s->fp) s->pos += rec_len; else s->at += rec_len; }
static uint64_t rec_key(const uint8_t *p)
{
	int32_t ref, pos; uint16_t flag;
	memcpy(&ref, p + 4, 4); memcpy(&pos, p + 8, 4); memcpy(&flag, p + 18, 2); /* block_size | refID pos l_read_name mapq bin n_cigar flag ... (sam.c:443-467) */
	return ref < 0 ? ~0ull : ((uint64_t)(uint32_t)ref << 34 | (uint64_t)(uint32_t)(pos + 1) << 1 | (uint64_t)((flag >> 4) & 1));
}
typedef struct { uint64_t key; int src; } hent_t;
#define HLESS(a, b) ((a).key < (b).key || ((a).key == (b).key && (a).src < (b).src)) /* equal keys: the earlier source = earlier input */
static void heap_down(hent_t *h, int n, int i)
{
	for (;;) { int l = 2 * i + 1, r = l + 1, m = i; hent_t t; if (l < n && HLESS(h[l], h[m])) m = l; if (r < n && HLESS(h[r], h[m])) m = r; if (m == i) return; t = h[i]; h[i] = h[m]; h[m] = t; i = m; }
}
typedef void (*sink_fn)(void *ctx, const uint8_t *p, size_t n);
static void merge_sources(src_t *s, int n_src, sink_fn sink, void *ctx)
{
	hent_t *h = (hent_t*)malloc(sizeof(hent_t) * (size_t)(n_src ? n_src : 1));
	int n = 0, i;
	size_t rl;
	for (i = 0; i < n_src; ++i) { const uint8_t *p = src_peek(&s[i], &rl); if (p) { h[n].key = rec_key(p); h[n].src = i; ++n; } }
	for (i = n / 2 - 1; i >= 0; --i) heap_down(h, n, i);
	while (n) {
		src_t *c = &s[h[0].src];
		const uint8_t *p = src_peek(c, &rl);
		sink(ctx, p, rl);
		src_advance(c, rl);
		if ((p = src_peek(c, &rl))) h[0].key = rec_key(p); else h[0] = h[--n];
		heap_down(h, n, 0);
	}
	free(h);
}

/* ---- BGZF output on several threads, or on the device (SSQ_BGZF_GPU=1) ---- */
typedef struct { FILE *fp; const uint8_t *buf; size_t n; int threads, level; ssq_bgzf_t *z; } flush_t;
typedef struct { FILE *fp; uint8_t *buf, *alt; size_t n, cap; int threads, level; ssq_bgzf_t *z; pthread_t bg; int bg_live; flush_t job; } bgzf_out_t;
static void write_member_bytes(FILE *fp, void *p, size_t n)
{
	if (fwrite(p, 1, n, fp) != n) { perror("sambamba (GPU shim): write"); exit(1); }
	ssq_free(p);
}
typedef struct { const uint8_t *in; size_t n; int level; void *out; size_t out_len; int rc; } job_t;
static void *job_main(void *a) { job_t *j = (job_t*)a; j->rc = ssq_bgzf_compress(j->in, j->n, j->level, 0, &j->out, &j->out_len); return 0; }
static void *flush_main(void *a) /* one buffer: compressed in slices on `threads` threads, written in order */
{
	const flush_t *f = (const flush_t*)a;
	job_t jobs[64];
	pthread_t th[64];
	int nj = f->threads, k;
	const size_t blk = 0xff00; /* the payload of one block: slices end on block boundaries, so the file is the same for any thread count */
	size_t per, at = 0;
	if (f->z) { /* the whole buffer in one call on the device */
		void *out = 0; size_t len = 0;
		if (ssq_bgzf_deflate(f->z, f->buf, f->n, f->level, 0, &out, &len)) { fprintf(stderr, "sambamba (GPU shim): BGZF compression on the device (SSQ_BGZF_GPU=1) failed: %s\n", ssq_last_error()); exit(1); }
		write_member_bytes(f->fp, out, len);
		return 0;
	}
	per = ((f->n / blk + (size_t)nj) / (size_t)nj) * blk;
	for (k = 0; k < nj && at < f->n; ++k) { jobs[k].in = f->buf + at; jobs[k].n = f->n - at < per ? f->n - at : per; jobs[k].level = f->level; jobs[k].out = 0; jobs[k].out_len = 0; at += jobs[k].n; }
	nj = k;
	for (k = 1; k < nj; ++k) pthread_create(&th[k], 0, job_main, &jobs[k]);
	job_main(&jobs[0]);
	for (k = 1; k < nj; ++k) pthread_join(th[k], 0);
	for (k = 0; k < nj; ++k) {
		if (jobs[k].rc) { fprintf(stderr, "sambamba (GPU shim): BGZF compression failed: %s\n", ssq_last_error()); exit(1); }
		write_member_bytes(f->fp, jobs[k].out, jobs[k].out_len);
	}
	return 0;
}
static void bgzf_wait(bgzf_out_t *o) { if (o->bg_live) { pthread_join(o->bg, 0); o->bg_live = 0; } }
/* the filled buffer goes to a background thread (after the previous one has been written: the file keeps its order) while the
 * caller goes on merging into the other buffer */
static void bgzf_flush(bgzf_out_t *o)
{
	uint8_t *t;
	if (!o->n) return;
	bgzf_wait(o);
	o->job.fp = o->fp; o->job.buf = o->buf; o->job.n = o->n; o->job.threads = o->threads; o->job.level = o->level; o->job.z = o->z;
	if (pthread_create(&o->bg, 0, flush_main, &o->job)) flush_main(&o->job); else o->bg_live = 1;
	t = o->buf; o->buf = o->alt; o->alt = t;
	o->n = 0;
}
static void bgzf_put(void *ctx, const uint8_t *p, size_t n)
{
	bgzf_out_t *o = (bgzf_out_t*)ctx;
	while (n) { /* the buffer is a multiple of the block payload: every flush but the last ends on a block boundary */
		const size_t room = o->cap - o->n, k = n < room ? n : room;
		memcpy(o->buf + o->n, p, k); o->n += k; p += k; n -= k;
		if (o->n == o->cap) bgzf_flush(o);
	}
}
static void file_put(void *ctx, const uint8_t *p, size_t n) { if (fwrite(p, 1, n, (FILE*)ctx) != n) { perror("sambamba (GPU shim): spill write"); exit(1); } }

static size_t parse_mem(const char *s)
{
	char *e;
	double v = strtod(s, &e);
	if (*e == 'K' || *e == 'k') v *= 1e3; else if (*e == 'M' || *e == 'm') v *= 1e6; else if (*e == 'G' || *e == 'g') v *= 1e9;
	return v < 64e6 ? (size_t)64e6 : (size_t)v;
}

static int sort_runs(head_t *h, size_t body, const char *out_fn, int threads, int level, size_t mem_limit, const char *tmpdir)
{
	src_t *mem = 0, *spill = 0;
	int n_mem = 0, m_mem = 0, n_spill = 0, m_spill = 0, i;
	size_t in_mem = 0, at = body;
	char *hdr_text, *hdr_sorted = 0;
	bgzf_out_t o;
	char **spill_fn = 0;
	ssq_bgzf_t *z = 0;
	{ /* SSQ_BGZF_GPU=1: the sorted file is compressed on SSQ_DEVICE (an explicit choice: its deflate bytes differ from zlib's) */
		const char *g = getenv("SSQ_BGZF_GPU");
		if (g && !strcmp(g, "1")) {
			const char *dv = getenv("SSQ_DEVICE");
			if (ssq_bgzf_create(dv && dv[0] ? atoi(dv) : 0, &z)) { fprintf(stderr, "sambamba (GPU shim): SSQ_BGZF_GPU=1 asks for BGZF compression on the GPU, but: %s\n", ssq_last_error()); return 1; }
		}
	}
	/* header text without the markers of the private stream */
	hdr_text = (char*)malloc(body + 1);
	{ size_t w = 0, p = 0; while (p < body) { const char *nl = (const char*)memchr(h->p + p, '\n', body - p); const size_t l = (size_t)(nl + 1 - (h->p + p)); if (strncmp(h->p + p, "@CO\tssq-", 8) != 0) { memcpy(hdr_text + w, h->p + p, l); w += l; } p += l; } hdr_text[w] = 0; }
	/* frames */
	for (;;) {
		ssq_frame_hdr_t fh;
		uint8_t *run;
		size_t got = 0;
		while (h->n - at < sizeof fh && head_more(h)) {}
		if (h->n - at == 0) break;
		if (h->n - at < sizeof fh) { fprintf(stderr, "sambamba (GPU shim): truncated run stream\n"); return 1; }
		memcpy(&fh, h->p + at, sizeof fh); at += sizeof fh;
		if (memcmp(fh.magic, SSQ_FRAME_MAGIC, 8) != 0 || fh.stream != SSQ_STREAM_BAM_RUN) { fprintf(stderr, "sambamba (GPU shim): corrupt run stream\n"); return 1; }
		run = (uint8_t*)malloc(fh.len ? fh.len : 1);
		if (!run) { fprintf(stderr, "sambamba (GPU shim): out of memory\n"); return 1; }
		{ const size_t k = h->n - at < fh.len ? h->n - at : (size_t)fh.len; memcpy(run, h->p + at, k); at += k; got = k; }
		if (at == h->n) { h->n = 0; at = 0; } /* the look-ahead buffer is used up: read straight into the run */
		while (got < fh.len) { ssize_t n = read(0, run + got, fh.len - got); if (n < 0 && errno == EINTR) continue; if (n <= 0) { fprintf(stderr, "sambamba (GPU shim): truncated run stream\n"); return 1; } got += (size_t)n; }
		if (n_mem == m_mem) { m_mem = m_mem ? m_mem * 2 : 64; mem = (src_t*)realloc(mem, sizeof(src_t) * (size_t)m_mem); }
		memset(&mem[n_mem], 0, sizeof(src_t)); mem[n_mem].mem = run; mem[n_mem].len = fh.len; ++n_mem; in_mem += fh.len;
		if (in_mem > mem_limit) { /* merge what is held and spill it */
			char fn[4096];
			FILE *fp;
			mkdir(tmpdir, 0777); /* sambamba creates its --tmpdir too */
			snprintf(fn, sizeof fn, "%s/ssq_sort_%ld_%d.run", tmpdir, (long)getpid(), n_spill);
			if (!(fp = fopen(fn, "wb"))) { fprintf(stderr, "sambamba (GPU shim): cannot create %s: %s\n", fn, strerror(errno)); return 1; }
			merge_sources(mem, n_mem, file_put, fp);
			if (fclose(fp)) { perror("sambamba (GPU shim): spill"); return 1; }
			for (i = 0; i < n_mem; ++i) free((void*)mem[i].mem);
			n_mem = 0; in_mem = 0;
			if (n_spill == m_spill) { m_spill = m_spill ? m_spill * 2 : 16; spill_fn = (char**)realloc(spill_fn, sizeof(char*) * (size_t)m_spill); }
			spill_fn[n_spill++] = strdup(fn);
		}
	}
	/* sources in input order: the spills (each a range of consecutive batches), then what is still in memory */
	spill = (src_t*)calloc((size_t)(n_spill + n_mem + 1), sizeof(src_t));
	for (i = 0; i < n_spill; ++i) { if (!(spill[i].fp = fopen(spill_fn[i], "rb"))) { perror(spill_fn[i]); return 1; } spill[i].cap = 8u << 20; spill[i].buf = (uint8_t*)malloc(spill[i].cap); }
	for (i = 0; i < n_mem; ++i) spill[n_spill + i] = mem[i];
	/* output: header block(s), records, end-of-file block */
	memset(&o, 0, sizeof o);
	o.z = z;
	if (!(o.fp = fopen(out_fn, "wb"))) { fprintf(stderr, "sambamba (GPU shim): cannot create %s: %s\n", out_fn, strerror(errno)); return 1; }
	o.threads = threads < 1 ? 1 : threads > 64 ? 64 : threads; o.level = level;
	if (z) { o.cap = (size_t)0xff00 * 1024; o.buf = (uint8_t*)ssq_host_alloc(o.cap); o.alt = (uint8_t*)ssq_host_alloc(o.cap); } /* pinned: full-rate copies to the device */
	else { o.cap = (size_t)0xff00 * 256 * (size_t)o.threads; o.buf = (uint8_t*)malloc(o.cap); o.alt = (uint8_t*)malloc(o.cap); }
	if (!o.buf || !o.alt) { fprintf(stderr, "sambamba (GPU shim): out of memory\n"); return 1; }
	if (ssq_bam_header_text(hdr_text, 1, &hdr_sorted)) { fprintf(stderr, "sambamba (GPU shim): %s\n", ssq_last_error()); return 1; }
	{ /* "BAM\1", text, reference table from the @SQ lines */
		const uint32_t l_text = (uint32_t)strlen(hdr_sorted);
		uint32_t n_ref = 0;
		const char *p;
		bgzf_put(&o, (const uint8_t*)"BAM\1", 4); bgzf_put(&o, (const uint8_t*)&l_text, 4); bgzf_put(&o, (const uint8_t*)hdr_sorted, l_text);
		for (p = hdr_sorted; p && *p; p = strchr(p, '\n'), p = p ? p + 1 : 0) if (!strncmp(p, "@SQ\t", 4)) ++n_ref;
		bgzf_put(&o, (const uint8_t*)&n_ref, 4);
		for (p = hdr_sorted; p && *p; p = strchr(p, '\n'), p = p ? p + 1 : 0) if (!strncmp(p, "@SQ\t", 4)) {
			const char *e = strchr(p, '\n'), *sn = 0, *ln = 0, *f;
			char name[1024]; uint32_t l_name; int32_t l_ref;
			for (f = p; f && f < e; f = memchr(f + 1, '\t', (size_t)(e - f - 1))) { if (!strncmp(f, "\tSN:", 4)) sn = f + 4; else if (!strncmp(f, "\tLN:", 4)) ln = f + 4; }
			if (!sn || !ln) { fprintf(stderr, "sambamba (GPU shim): @SQ line without SN / LN\n"); return 1; }
			{ size_t k = 0; while (sn[k] != '\t' && sn[k] != '\n' && k + 1 < sizeof name) { name[k] = sn[k]; ++k; } name[k] = 0; l_name = (uint32_t)k + 1; }
			l_ref = (int32_t)atoll(ln);
			bgzf_put(&o, (const uint8_t*)&l_name, 4); bgzf_put(&o, (const uint8_t*)name, l_name); bgzf_put(&o, (const uint8_t*)&l_ref, 4);
		}
		bgzf_flush(&o); /* the header in blocks of its own, as sambamba writes it */
	}
	merge_sources(spill, n_spill + n_mem, bgzf_put, &o);
	bgzf_flush(&o);
	bgzf_wait(&o);
	{ void *eofb = 0; size_t el = 0; if (ssq_bgzf_compress("", 0, level, 1, &eofb, &el)) { fprintf(stderr, "sambamba (GPU shim): %s\n", ssq_last_error()); return 1; } fwrite(eofb, 1, el, o.fp); ssq_free(eofb); }
	if (fclose(o.fp)) { perror("sambamba (GPU shim): close"); return 1; }
	for (i = 0; i < n_spill; ++i) { fclose(spill[i].fp); unlink(spill_fn[i]); }
	if (z) { ssq_host_free(o.buf); ssq_host_free(o.alt); ssq_bgzf_free(z); }
	return 0;
}

int main(int argc, char **argv)
{
	head_t h;
	size_t body = 0;
	int i;
	g_self = argv[0];
	memset(&h, 0, sizeof h);
	if (argc < 2) exec_real(argv, "this call");
	if (!strcmp(argv[1], "view")) {
		int sam_in = 0; const char *in = 0;
		for (i = 2; i < argc; ++i) {
			if (!strcmp(argv[i], "-S") || !strcmp(argv[i], "--sam-input")) sam_in = 1;
			else if ((!strcmp(argv[i], "-f") || !strcmp(argv[i], "-l") || !strcmp(argv[i], "-o") || !strcmp(argv[i], "-t") || !strcmp(argv[i], "-F") || !strcmp(argv[i], "-L") || !strcmp(argv[i], "-s")) && i + 1 < argc) ++i;
			else if (argv[i][0] != '-' || !strcmp(argv[i], "-")) { if (!in) in = argv[i]; }
		}
		if (!sam_in || !in || (strcmp(in, "/dev/stdin") && strcmp(in, "-"))) exec_real(argv, "`view` of anything but SAM on stdin");
		if (!sniff_runs(&h, &body)) return feed_real(argv, h.p, h.n, "`view` of plain SAM text");
		/* our runs: BAM already; hand them on */
		{ static char buf[1 << 20]; if (write_all(1, h.p, h.n)) return 1; for (;;) { ssize_t n = read(0, buf, sizeof buf); if (n < 0 && errno == EINTR) continue; if (n <= 0) break; if (write_all(1, buf, (size_t)n)) return 1; } }
		return 0;
	}
	if (!strcmp(argv[1], "sort")) {
		const char *in = 0, *out_fn = 0, *tmpdir = "/tmp";
		int threads = 1, level = 6, by_name = 0;
		size_t mem_limit = (size_t)2e9;
		for (i = 2; i < argc; ++i) {
			if (!strcmp(argv[i], "-t") && i + 1 < argc) threads = atoi(argv[++i]);
			else if (!strncmp(argv[i], "--nthreads=", 11)) threads = atoi(argv[i] + 11);
			else if (!strcmp(argv[i], "-m") && i + 1 < argc) mem_limit = parse_mem(argv[++i]);
			else if (!strncmp(argv[i], "--memory-limit=", 15)) mem_limit = parse_mem(argv[i] + 15);
			else if (!strncmp(argv[i], "--tmpdir=", 9)) tmpdir = argv[i] + 9;
			else if (!strcmp(argv[i], "--tmpdir") && i + 1 < argc) tmpdir = argv[++i];
			else if (!strcmp(argv[i], "-o") && i + 1 < argc) out_fn = argv[++i];
			else if (!strncmp(argv[i], "--out=", 6)) out_fn = argv[i] + 6;
			else if (!strcmp(argv[i], "-l") && i + 1 < argc) level = atoi(argv[++i]);
			else if (!strncmp(argv[i], "--compression-level=", 20)) level = atoi(argv[i] + 20);
			else if (!strcmp(argv[i], "-n") || !strcmp(argv[i], "--sort-by-name") || !strcmp(argv[i], "-N")) by_name = 1;
			else if (argv[i][0] != '-' || !strcmp(argv[i], "-")) { if (!in) in = argv[i]; }
		}
		if (!in || (strcmp(in, "/dev/stdin") && strcmp(in, "-"))) exec_real(argv, "`sort` of a file");
		if (!sniff_runs(&h, &body)) return feed_real(argv, h.p, h.n, "`sort` of ordinary BAM");
		if (by_name || !out_fn) { fprintf(stderr, "sambamba (GPU shim): the run stream can only be coordinate-sorted into a file (-o)\n"); return 1; }
		if (getenv("SSQ_SORT_SPILL_BYTES")) mem_limit = 2 * (size_t)atoll(getenv("SSQ_SORT_SPILL_BYTES")); /* tests: force the spill path on small inputs */
		return sort_runs(&h, body, out_fn, threads, level, mem_limit / 2, tmpdir);
	}
	exec_real(argv, "this subcommand");
	return 1;
}
