/*
 * ssq.h — C-ABI of libssq.so, the H100-native (sm_90a) implementation of the `speedseq align` hot path.
 *
 * The reference's drop-in boundary for this path is a PROCESS boundary, not an FFI:
 * bin/speedseq sources speedseq.config (speedseq/bin/speedseq:15-24,361) and interpolates
 * $BWA and $SAMBLASTER into the pipeline text at speedseq/bin/speedseq:437-449 (interleaved)
 * and :467-479 (two files); the index is made by `$BWA index` at :389.  libssq.so is what the two
 * replacement executables (speedseq_b200/bin/bwa, speedseq_b200/bin/samblaster) link; its entry
 * points are the batch forms of the functions those tools spend their time in (SURVEY.md §8a).
 * Each declaration cites the reference call site it serves and names the upstream routine it
 * replaces (upstream sources are NOT vendored in the reference tree: .SUBMODULES.json:23-29,51-57).
 *
 * Conventions: plain pointers and sizes, caller-owned HOST buffers unless a name ends in _dev,
 * int return code (0 = ok, <0 = SSQ_E*), no global state other than the CUDA context, one CUDA
 * stream per handle.  Every entry point fails with SSQ_ENOGPU when no sm_90 (H100) device is usable —
 * there is no CPU fallback inside this library.
 */
#ifndef SSQ_H
#define SSQ_H
#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SSQ_OK        0
#define SSQ_ENOGPU   (-1)  /* no CUDA device / wrong architecture */
#define SSQ_EIO      (-2)  /* index files missing or malformed */
#define SSQ_ENOMEM   (-3)
#define SSQ_EINVAL   (-4)
#define SSQ_ECAP     (-5)  /* caller buffer too small; required size returned through *needed */
#define SSQ_ECUDA    (-6)  /* a CUDA call failed; see ssq_last_error() */
#define SSQ_ELEN     (-7)  /* a read is longer than SSQ_MAX_READ_LEN */
#define SSQ_EFORMAT  (-8)  /* FASTQ text the device tokeniser does not take (see ssq_aligner_upload_fastq); use the host tokeniser */
#define SSQ_EDATA    (-9)  /* compressed input is corrupt or truncated; see ssq_last_error() */

#define SSQ_MAX_READ_LEN 255

const char *ssq_last_error(void);
int ssq_device_count(void);

/* ---------------------------------------------------------------- options ----
 * Scoring/heuristic parameters of `bwa mem`; speedseq passes none of them on the command line
 * (speedseq/bin/speedseq:438), so ssq_opts_default() is what the pipeline runs with.
 * Replaces upstream mem_opt_init(). */
typedef struct {
	int32_t a, b, o_del, e_del, o_ins, e_ins;
	int32_t pen_unpaired, pen_clip5, pen_clip3, w, zdrop, T;
	int32_t min_seed_len, split_width, max_occ, max_chain_gap, max_mem_intv;
	int32_t min_chain_weight, max_chain_extend, max_ins, max_matesw, max_XA_hits;
	float split_factor, mask_level, drop_ratio, XA_drop_ratio, mask_level_redun;
	int32_t mapQ_coef_len, mapQ_coef_fac;
	int32_t n_threads; /* host threads for the per-pair bookkeeping and SAM formatting (`bwa mem -t`); does not change any result */
} ssq_opts_t;
void ssq_opts_default(ssq_opts_t *o);

/* ------------------------------------------------------------------ index ----
 * Device-resident FM index + packed reference.  ssq_index_load replaces upstream bwa_idx_load()
 * (start of `$BWA mem`, speedseq/bin/speedseq:438): reads PREFIX.{bwt,sa,pac,ann,amb} in the
 * on-disk format of the reference's goldens (speedseq/example/data/ *.fasta.{amb,ann,pac,bwt,sa})
 * and uploads them to `device`. */
typedef struct ssq_index ssq_index_t;
/* `$BWA index $REF` (speedseq/bin/speedseq:389): FASTA (plain or gz) -> PREFIX.{amb,ann,pac,bwt,sa}, byte-identical
 * to the reference's goldens for example/data and independent of the path that built them.  prefix == NULL means
 * prefix = fasta.  Replaces upstream bwa_idx_build().  Two ways to sort the suffixes of forward + reverse-complement text:
 *   2 device sort (csrc/ssq_sapass.cuh): 5 bytes of device memory per suffix for the rank array plus a working budget, fewer
 *     than 2^40 suffixes; the first sort runs in passes over buckets of leading 12-mers, then doubling rounds over the
 *     suffixes still tied.  GRCh37 (3.1 Gbp): 31 GB of rank array.
 *   3 host: induced sorting with 5-byte entries, no GPU touched (about 15 bytes of host memory per base pair).
 *     SSQ_INDEX_HOST=1 (or 40 / 64: entry width) forces it under the automatic choice.
 * The automatic choice (path 0) reads the device's *free* memory and leaves 1 GB + 1/32 of it to other users: path 2 when
 * the rank array, the text and a working budget of at least max(256 MB, 1.25 B per suffix: at most 32 first-sort passes) fit;
 * else path 3 (also for a reference past 2^31 - 2 suffixes with no usable device; a smaller one with no device gives
 * SSQ_ENOGPU).  Each first-sort pass reads the whole text, so a budget near that floor costs more passes.  A bucket of
 * suffixes sharing their first 12 bases that exceeds the budget is sorted on its own; when even that does not fit in free
 * device memory the call returns SSQ_ENOMEM rather than falling back.  Measured costs: DESIGN.md §8. */
int ssq_index_build(const char *fasta, const char *prefix, int device); /* = ssq_index_build_ex(fasta, prefix, device, NULL, NULL) */
typedef struct {
	int32_t path;        /* 0 auto, 2 device sort, 3 host (1 is not a path: SSQ_EINVAL) */
	int32_t pad;
	uint64_t work_bytes; /* path 2: working budget beyond rank array, text and bucket counts; 0 = from free memory at the start */
} ssq_index_build_opts_t;
typedef struct {
	int32_t path, pad;   /* the path that ran */
	int64_t passes, rounds, chunks; /* path 2: first-sort passes, doubling rounds, chunks over all rounds */
	int64_t unresolved_first, largest_group; /* suffixes still tied after the first sort, largest such group */
	int64_t oversize_groups;  /* buckets / groups larger than the budget, each sorted on its own */
	int64_t peak_device_bytes; /* path 2: most device memory held at once (rank array, text and working set) */
	int64_t ranges;      /* path 2: finalisation ranges (BWT / checkpoints / SA samples written per range of rows) */
} ssq_index_build_stats_t;
/* opt / st may be NULL.  SSQ_EINVAL: a path the reference is too large for; SSQ_ENOMEM (path 2): device memory short, the
 * message gives the sizes.  When path 0 took the host path, ssq_last_error() says why (empty when it was forced). */
int ssq_index_build_ex(const char *fasta, const char *prefix, int device, const ssq_index_build_opts_t *opt, ssq_index_build_stats_t *st);
int ssq_index_load(const char *prefix, int device, ssq_index_t **out);
void ssq_index_free(ssq_index_t *idx);
/* what: 0 l_pac, 1 seq_len(=2*l_pac), 2 primary, 3 n_seqs, 4 bwt words, 5 n_sa, 6 device bytes, 7 bytes per rank query (32|64),
 * 8 bytes per SA sample read (4|8), 9 SA sampling interval in device memory (on disk: 32; the loader derives a denser sample) */
uint64_t ssq_index_info(const ssq_index_t *idx, int what);

/* ----------------------------------------------------- kernel-level batches ----
 * Reads are passed as one byte per base (0=A 1=C 2=G 3=T 4=N), concatenated, with read_off[n+1]. */

/* SMEM seeding, all three passes, per read.  Replaces upstream mem_collect_intv() →
 * bwt_smem1a / bwt_seed_strategy1 / bwt_extend / bwt_2occ4 (inside `$BWA mem`, speedseq:438).
 * Output intervals of read i are out[out_off[i] .. out_off[i+1]) sorted by (qbeg<<32|qend). */
typedef struct { uint64_t k, l, s; uint32_t qbeg, qend; } ssq_smem_t;
int ssq_smem_batch(const ssq_index_t *idx, const ssq_opts_t *opt, int n_reads, const uint8_t *seq, const uint64_t *read_off,
                   ssq_smem_t *out, uint64_t out_cap, uint64_t *out_off, uint64_t *needed);

/* Suffix-array lookup of BWT rows.  Replaces upstream bwt_sa() / bwt_invPsi() (speedseq:438). */
int ssq_sa_lookup_batch(const ssq_index_t *idx, uint64_t n, const uint64_t *rows, uint64_t *pos);

/* Banded affine-gap seed extension.  Replaces upstream ksw_extend2() as called from
 * mem_chain2aln() (speedseq:438).  Sequences are one byte per base in qbuf/tbuf. */
typedef struct { uint64_t q_off, t_off; int32_t qlen, tlen, h0, w, end_bonus, zdrop; } ssq_sw_task_t;
typedef struct { int32_t score, qle, tle, gtle, gscore, max_off; } ssq_sw_result_t;
int ssq_sw_extend_batch(const ssq_opts_t *opt, int device, uint64_t n, const ssq_sw_task_t *tasks,
                        const uint8_t *qbuf, uint64_t qbuf_len, const uint8_t *tbuf, uint64_t tbuf_len, ssq_sw_result_t *out);

/* Local alignment in the evaluation order of the reference's striped SSE2 kernel.  Replaces upstream ksw_align2() as called from
 * mem_matesw() (mate rescue inside `$BWA mem`, speedseq:438): xtra = KSW_XSUBO|KSW_XSTART|(KSW_XBYTE if qlen*a < 250)|minsc.
 * One warp per problem, the SSE lanes mapped onto warp lanes (csrc/ssq_warp.cuh). */
typedef struct { uint64_t q_off, t_off; int32_t qlen, tlen, xtra, pad; } ssq_swl_task_t;
typedef struct { int32_t score, te, qe, score2, te2, tb, qb; } ssq_swl_result_t;
#define SSQ_KSW_XBYTE  0x10000
#define SSQ_KSW_XSTOP  0x20000
#define SSQ_KSW_XSUBO  0x40000
#define SSQ_KSW_XSTART 0x80000
int ssq_sw_local_batch(const ssq_opts_t *opt, int device, uint64_t n, const ssq_swl_task_t *tasks, const uint8_t *qbuf, uint64_t qbuf_len,
                       const uint8_t *tbuf, uint64_t tbuf_len, ssq_swl_result_t *out);

/* Banded global alignment with traceback.  Replaces upstream ksw_global2() as called from bwa_gen_cigar2() (CIGAR generation inside
 * `$BWA mem`, speedseq:438); the same warp routine as the pipeline's CIGAR stage (csrc/ssq_warp.cuh: sw_global_warp), one warp per
 * problem.  Task i aligns qbuf[q_off, +qlen) against tbuf[t_off, +tlen) in a band of half-width w; its CIGAR (op | len << 4, ops
 * 0 M, 1 I, 2 D) goes to cig[cig_off, +cig_cap).  cig_cap == 0: score only (n_cigar = 0).  n_cigar = -1: the CIGAR needs more than
 * cig_cap operations (nothing is cut short).  Every task must satisfy 1 <= qlen <= SSQ_MAX_READ_LEN, 1 <= tlen <= 2048, w >= 0 and
 * |tlen - qlen| <= w (the end cell lies in the band), and its buffers must be in range; otherwise SSQ_EINVAL and nothing runs. */
typedef struct { uint64_t q_off, t_off; int32_t qlen, tlen, w, cig_cap; uint64_t cig_off; } ssq_swg_task_t;
typedef struct { int32_t score, n_cigar; } ssq_swg_result_t;
int ssq_sw_global_batch(const ssq_opts_t *opt, int device, uint64_t n, const ssq_swg_task_t *tasks, const uint8_t *qbuf, uint64_t qbuf_len,
                        const uint8_t *tbuf, uint64_t tbuf_len, uint32_t *cig, uint64_t cig_len, ssq_swg_result_t *out);

/* Chains after seeding + SA lookup + chaining + chain filter.  Replaces upstream mem_chain() +
 * mem_chain_flt() (speedseq:438).  Flattened: read i owns chains [read_chain_off[i], read_chain_off[i+1]),
 * chain c owns seeds [chain_seed_off[c], chain_seed_off[c+1]). */
typedef struct { int64_t rbeg; int32_t qbeg, len; } ssq_seed_t;
int ssq_chain_batch(const ssq_index_t *idx, const ssq_opts_t *opt, int n_reads, const uint8_t *seq, const uint64_t *read_off,
                    ssq_seed_t *seeds, uint64_t seed_cap, uint64_t *chain_seed_off, uint64_t chain_cap, uint64_t *read_chain_off,
                    uint64_t *n_chains, uint64_t *n_seeds);

/* Duplicate marking over pair signatures, first occurrence in input order is kept.  Replaces the
 * signature hash sets of samblaster's markDupsDiscordants() (`$SAMBLASTER`, speedseq:439).
 * valid==0 entries (both ends unmapped) are never duplicates. */
typedef struct { uint64_t pos1, pos2; uint8_t strand1, strand2, valid, pad[5]; } ssq_dupsig_t;
int ssq_dupmark_batch(int device, uint64_t n, const ssq_dupsig_t *sig, uint8_t *is_dup);

/* Streaming form for inputs that arrive in pieces (the `samblaster` shim): the set remembers every signature it has seen,
 * so "first occurrence wins" holds across calls as if all batches had been one. */
typedef struct ssq_dupset ssq_dupset_t;
int ssq_dupset_create(int device, ssq_dupset_t **out);
int ssq_dupset_mark(ssq_dupset_t *set, uint64_t n, const ssq_dupsig_t *sig, uint8_t *is_dup);
uint64_t ssq_dupset_size(const ssq_dupset_t *set);
void ssq_dupset_free(ssq_dupset_t *set);

/* Device-pointer form used by the multi-GPU exchange (speedseq_b200/dist.py): keys already sit in HBM (received by an NCCL
 * all-to-all), element order = first-seen order, key = (5' position << 1 | strand) of the canonically ordered ends. */
int ssq_dupmark_keys_dev(int device, uint64_t n, const uint64_t *d_key1, const uint64_t *d_key2, const uint8_t *d_valid, uint8_t *d_is_dup, void *stream);

/* ------------------------------------------------- the alignment pipeline ----
 * Seeding → SA lookup → chaining → chain filter → seed extension → alignment regions, all on the
 * device (the single-end core of `$BWA mem`, upstream mem_align1_core() up to and including
 * mem_chain2aln(); stage 1 adds mem_sort_dedup_patch()).  Regions of read i are
 * out[out_off[i] .. out_off[i+1]) in the order the reference produces them. */
typedef struct {
	int64_t rb, re;
	int32_t qb, qe, rid, score, truesc, w, seedcov, seedlen0;
	float frac_rep;
	int32_t read_id;
} ssq_alnreg_t;

/* one-shot, HOST buffers in and out: regions only (parity tests of the seed -> extend half; the CLI shim and bench.py drive ssq_aligner_*) */
int ssq_align_batch(const ssq_index_t *idx, const ssq_opts_t *opt, int n_reads, const uint8_t *seq, const uint64_t *read_off,
                    int stage, ssq_alnreg_t *out, uint64_t out_cap, uint64_t *out_off, uint64_t *needed);

/* staged form: upload once, run the kernels any number of times with everything resident in HBM
 * (`value` in bench.py), fetch results when wanted */
typedef struct ssq_batch ssq_batch_t;
int ssq_batch_create(const ssq_index_t *idx, const ssq_opts_t *opt, int n_reads, const uint8_t *seq, const uint64_t *read_off, ssq_batch_t **out);
/* (re)load a batch object with new reads; device buffers are kept and grown, so one object serves a stream of batches.
 * ssq_batch_create(..., read_off == NULL) makes an empty object to be filled by ssq_batch_upload(). */
int ssq_batch_upload(ssq_batch_t *b, int n_reads, const uint8_t *seq, const uint64_t *read_off);
int ssq_batch_run(ssq_batch_t *b);                 /* all kernels of the path on the batch's stream; returns when the last is queued */
int ssq_batch_sync(ssq_batch_t *b);
int ssq_batch_fetch(ssq_batch_t *b, ssq_alnreg_t *out, uint64_t out_cap, uint64_t *out_off, uint64_t *needed);
void *ssq_batch_stream(ssq_batch_t *b);            /* cudaStream_t, for event timing on the launching stream */
int ssq_batch_set_stream(ssq_batch_t *b, void *stream); /* make several batch objects share one caller-owned stream */
/* per-run work counters measured on the device: what: 0 occ blocks read by seeding, 1 occ blocks read by SA walks,
 * 2 SA samples read, 3 SW extension calls, 4 SW cells, 5 SW algorithmic bytes, 6 kernels launched per run, 7 seeds, 8 regions */
uint64_t ssq_batch_counter(const ssq_batch_t *b, int what);
/* milliseconds of the last run per stage (CUDA events on the batch stream): 0 smem, 1 sa, 2 chain, 3 extend, 4 finalize */
float ssq_batch_stage_ms(const ssq_batch_t *b, int stage);
void ssq_batch_free(ssq_batch_t *b);

/* ------------------------------------------------------- `bwa mem` for one batch ----
 * What the `bwa` shim calls per batch of reads (upstream mem_process_seqs(); `$BWA mem`, speedseq:438,468): reads as ASCII
 * strings (names already stripped of /1 /2), paired = adjacent reads are mates.  n_processed = global ordinal of reads[0]
 * (tie-breaking hashes use it).  pes0 != NULL overrides the per-batch insert-size statistics (`-I`).  Returns the SAM
 * records of the batch in input order as one malloc'd string (free with ssq_free).  Seeding, chaining, all Smith-Waterman
 * variants and CIGAR/NM/MD generation run on the device; pairing, MAPQ and text formatting on the host. */
typedef struct { int32_t low, high, failed, pad; double avg, std; } ssq_pestat_t;
int ssq_mem_batch_sam(const ssq_index_t *idx, const ssq_opts_t *opt, int n_reads, const char *const *names, const char *const *seqs, const char *const *quals,
                      const char *const *comments, int64_t n_processed, int paired, const ssq_pestat_t *pes0, const char *rg_id, int verbose, char **sam_out, size_t *sam_len,
                      size_t *read_sam_off /* optional [n_reads+1]: byte range of each read's lines */);
void ssq_free(void *p);

/* ----------------------------------------- `bwa mem | samblaster`, HBM-resident ----
 * The whole pipe of speedseq/bin/speedseq:438-439 (interleaved) / :468-469 (two files) for one batch of reads:
 * `$BWA mem -t T [-p] [-C] [-I ..] -R RG REF FQ.. | $SAMBLASTER [--excludeDups] --addMateTags --maxSplitCount C
 * --minNonOverlap M --splitterFile F --discordantFile F`.  Reads go in as the FASTQ fields (concatenated, with offsets), the three
 * SAM record streams come out (main, splitters, discordants; headers are the caller's business: they depend on argv).  Between
 * the two copies everything stays on the device: alignment (upstream mem_process_seqs incl. mem_pestat's batch coupling — only
 * its histogram reduction runs on the host), pairing, MAPQ, CIGAR/NM/MD, samblaster's signature / discordant / splitter tests,
 * first-seen-wins duplicate marking against every earlier batch of the same aligner object, and the SAM text itself.
 * With sb == NULL or sb->enabled == 0 only text[0] is produced and it is exactly `bwa mem`'s records (what ssq_mem_batch_sam
 * returns).  One aligner object = one `bwa mem | samblaster` run: create, run batch after batch in input order, free. */
typedef struct {
	int32_t enabled;            /* 0: plain `bwa mem` records */
	int32_t exclude_dups;       /* --excludeDups: duplicates stay out of the splitter / discordant streams (speedseq:241) */
	int32_t add_mate_tags;      /* --addMateTags: MC:Z / MQ:i on every record of a pair (speedseq:439) */
	int32_t max_split_count;    /* --maxSplitCount (speedseq:242) */
	int32_t min_non_overlap;    /* --minNonOverlap (speedseq:243) */
	int32_t min_indel_size, max_unmapped_bases; /* samblaster defaults 50 / 50 */
	int32_t remove_dups;        /* --removeDups */
	int32_t want_split, want_disc; /* --splitterFile / --discordantFile given */
} ssq_sb_opts_t;
void ssq_sb_opts_default(ssq_sb_opts_t *o);

typedef struct {
	int32_t n_reads, paired;              /* paired: adjacent reads are mates (`-p` after smart pairing, or two files interleaved) */
	const char *seq; const uint64_t *seq_off;   /* bases as in the FASTQ (ASCII, any case), concatenated; seq_off[n_reads + 1] */
	const char *qual;                     /* qualities at the same offsets; NULL = none (FASTA input) */
	const char *name; const uint32_t *name_off; /* names without the /1 /2 suffix, concatenated, no terminators; name_off[n_reads + 1] */
	const char *comment; const uint32_t *comment_off; /* FASTQ comments for `-C`; NULL = none */
	int64_t n_processed;                  /* global ordinal of reads[0] (tie-breaking hashes use it) */
} ssq_reads_t;

typedef struct {
	const char *text[3]; size_t len[3];   /* 0 main SAM records, 1 splitters, 2 discordants; owned by the aligner, valid until its next run */
	const uint64_t *read_off;             /* [n_reads + 1]: byte range of each read's records in text[0] */
	uint64_t n_ids, n_dup;                /* QNAME blocks seen / marked duplicate in this batch */
	ssq_pestat_t pes[4];                  /* the insert-size statistics the batch was paired with */
} ssq_sam_t;

typedef struct ssq_aligner ssq_aligner_t;
int ssq_aligner_create(const ssq_index_t *idx, const ssq_opts_t *opt, const ssq_sb_opts_t *sb, const char *rg_id, ssq_aligner_t **out);
/* pes0 != NULL overrides the per-batch insert-size statistics (`-I`); verbose: mem_pestat's log lines on stderr like bwa */
int ssq_aligner_run(ssq_aligner_t *al, const ssq_reads_t *reads, const ssq_pestat_t *pes0, int verbose, ssq_sam_t *out);
/* the three phases of ssq_aligner_run, separately (bench.py times `compute` with the reads resident in HBM) */
int ssq_aligner_upload(ssq_aligner_t *al, const ssq_reads_t *reads);
int ssq_aligner_compute(ssq_aligner_t *al, const ssq_pestat_t *pes0, int verbose);
/* FASTQ ingest on the device instead of ssq_aligner_upload (upstream bseq_read -> kseq_read inside `$BWA mem`, speedseq:438,468;
 * tokenisation rules of speedseq/src/samtools-1.3.1/htslib-1.3.1/htslib/kseq.h:189-231).  fq1 / fq2: raw, uncompressed text of
 * the FASTQ input(s) from a record boundary on (fq2 == NULL: one file; interleaved: adjacent records are mates, `-p`); final: no
 * more text follows.  The device finds the records, closes the batch where bwa would (bases >= chunk_bases and an even number of
 * reads), strips /1 /2, and packs names, bases, qualities and (keep_comment, `-C`) comments into the aligner's batch buffers;
 * *used1 / *used2 = bytes of each text the batch covers (the caller keeps the rest for the next call).  *need_more: no complete
 * batch in the text and more text exists -> call again with more.  SSQ_EFORMAT: not the four-lines-per-record layout (multi-line
 * records, FASTA, unpaired reads in an interleaved file, files of different lengths): nothing was consumed, tokenise on the host. */
int ssq_aligner_upload_fastq(ssq_aligner_t *al, const char *fq1, size_t len1, int final1, const char *fq2, size_t len2, int final2, int interleaved, int keep_comment,
                             int64_t chunk_bases, int64_t n_processed, size_t *used1, size_t *used2, int *n_reads, int *need_more);
void *ssq_host_alloc(size_t bytes); /* page-locked host memory for the text buffers (full-rate host->device copies) */
void ssq_host_free(void *p);
int ssq_aligner_fetch(ssq_aligner_t *al, ssq_sam_t *out);
int ssq_aligner_reset_dups(ssq_aligner_t *al);     /* forget every signature seen so far (a new run) */
/* several aligner objects (one host thread + stream each) can work on consecutive batches of ONE run: they share a dup-set, and
 * each batch is given its turn number (0, 1, 2, ... since the last reset) so that "first seen wins" still follows input order */
int ssq_aligner_share_dupset(ssq_aligner_t *al, ssq_dupset_t *set);
int ssq_aligner_set_turn(ssq_aligner_t *al, long long turn); /* -1 (default): no ordering (a single aligner runs its batches in order anyway) */
void *ssq_aligner_stream(ssq_aligner_t *al);       /* cudaStream_t of the object, for event timing on the launching stream */
/* milliseconds of the last batch per stage (CUDA events): 0 upload, 1 seed..extend, 2 sort/dedup/patch, 3 insert-size statistics,
 * 4 mate rescue, 5 pairing/MAPQ/planning, 6 CIGAR/NM/MD, 7 samblaster + dup-set, 8 text, 9 fetch; 10.. = ssq_batch_stage_ms(0..4) */
float ssq_aligner_stage_ms(const ssq_aligner_t *al, int stage);
/* what < 100: ssq_batch_counter of the alignment stage; 100 alignments written (CIGAR tasks), 101-103 bytes of the three streams, 104 dup-set size,
 * 105 pairs that went through mate rescue, 106 alignments that needed the banded global DP for their CIGAR,
 * 107 local-SW passes run by the mate rescue, 108 their cells, 109 bases / 110 reads of the batch in the aligner */
uint64_t ssq_aligner_counter(const ssq_aligner_t *al, int what);
void ssq_aligner_free(ssq_aligner_t *al);

/* ----------------------------------------------------------------- BAM records ----
 * The downstream half of the pipe turns the SAM text straight back into BAM (`sambamba view -S -f bam -l 0 | sambamba sort`,
 * speedseq:440-441, :444-448).  With ssq_aligner_set_bam(al, 1, ..) the aligner additionally encodes the records of the three
 * streams as BAM on the device, straight from its structured alignments (layout: htslib sam.c:443-467, bin: hts.h:580-586),
 * coordinate-sorted within the batch by (reference, position, strand) with equal keys in input order — what sambamba's sort
 * produces (tests/golden/ex_bam_*: written by the reference's own sambamba, matched byte for byte).  blank_side_streams: the
 * splitter / discordant records carry no SEQ / QUAL, like after speedseq's gawk step (speedseq:443,446).
 * ssq_bam_header + ssq_bgzf_compress (host: zlib) make a complete .bam out of header and records; ssq_bam_merge_runs merges the
 * sorted runs of the batches of a run into the order `sambamba sort` gives the whole input. */
int ssq_aligner_set_bam(ssq_aligner_t *al, int enable, int blank_side_streams);
int ssq_aligner_fetch_bam(ssq_aligner_t *al, int stream, const void **records, size_t *len); /* after ssq_aligner_compute; owned by the aligner */
/* the SAM text of one stream alone (0 main, 1 splitters, 2 discordants), for callers that take the main records as BAM and only
 * want the side streams as text (speedseq:443,446 run them through gawk); after ssq_aligner_compute; owned by the aligner */
int ssq_aligner_fetch_text(ssq_aligner_t *al, int stream, const char **text, size_t *len);
int ssq_bam_header(const ssq_index_t *idx, const char *sam_header_text, int sorted, void **out, size_t *out_len); /* free with ssq_free */
/* the header text alone: sorted != 0 rewrites it the way `sambamba view -S | sambamba sort` does (@HD SO:coordinate first, sambamba's
 * tag order inside @SQ / @RG / @PG lines); free with ssq_free */
int ssq_bam_header_text(const char *sam_header_text, int sorted, char **out);
int ssq_bgzf_compress(const void *in, size_t n, int level, int with_eof, void **out, size_t *out_len);           /* free with ssq_free */
/* The same BGZF file layout, compressed on the device (csrc/ssq_bgzf.cu): the input is cut into 0xff00-byte payloads from its start
 * exactly as ssq_bgzf_compress cuts it, each payload becomes one gzip member (BC extra field, CRC-32, ISIZE) holding one deflate block
 * (stored, fixed or dynamic Huffman, whichever is smallest), so the decompressed file and its block boundaries are the host path's;
 * only the deflate bytes differ.  Level 0 writes stored blocks; levels 1-9 (and -1) all run the one device encoder.  The output is a
 * function of the input bytes and of level == 0 alone — not of how the input is split across calls, the launch or the stream.
 * An object owns device buffers, a stream and pinned staging, reused across calls; one host thread at a time. */
typedef struct ssq_bgzf ssq_bgzf_t;
int ssq_bgzf_create(int device, ssq_bgzf_t **out);
/* host buffers: same contract, block cutting and EOF handling as ssq_bgzf_compress; *out malloc'd, free with ssq_free */
int ssq_bgzf_deflate(ssq_bgzf_t *z, const void *in, size_t n, int level, int with_eof, void **out, size_t *out_len);
/* device buffers, on the object's stream (returns after it is done); SSQ_ECAP + *needed when out_cap is too small */
int ssq_bgzf_deflate_dev(ssq_bgzf_t *z, const void *d_in, size_t n, int level, int with_eof, void *d_out, size_t out_cap, size_t *out_len, size_t *needed);
void *ssq_bgzf_stream(ssq_bgzf_t *z);               /* cudaStream_t of the object, for event timing */
void ssq_bgzf_free(ssq_bgzf_t *z);
/* gzip decoding on the device (csrc/ssq_gunzip.cu): one deflate stream is split into chunks of chunk_bytes compressed bytes and
 * decoded chunk-parallel (speculative decoding from searched block starts, checked link by link and repaired, then verified with
 * CRC-32 and ISIZE).  End of stream as zlib's gzread: concatenated members are one stream, bytes after a member that do not start
 * with 1f 8b are ignored, an empty input is an empty output.  Corrupt or truncated input is SSQ_EDATA, with the compressed offset in
 * ssq_last_error(); never a short output.  An object holds about 1.6 GB of device memory (1 GB of chunk slots, 512 MB of window
 * text, the window's input), a stream and pinned staging; one host thread at a time.  Without a usable GPU create returns
 * SSQ_ENOGPU. */
typedef struct ssq_gunzip ssq_gunzip_t;
int ssq_gunzip_create(int device, size_t chunk_bytes, ssq_gunzip_t **out); /* chunk_bytes 0 = default (32 KB); 256 B .. 4 MB */
/* streaming: in[0, n) continues the object's stream (final: nothing follows it).  Decodes whole windows into out, keeps text it
 * could not deliver for the next call (which then consumes nothing), *used = leading input bytes the caller drops before the next
 * call, which passes the rest followed by more input; *done once the stream has ended and all its text was delivered.  After *done
 * or an error the next call starts a new stream.  Unless
 * final, nothing is decoded (and *used = 0) before n reaches one window of input (GZ_MAXCH chunks + 1 MB, 33 MB by default). */
int ssq_gunzip_inflate(ssq_gunzip_t *g, const void *in, size_t n, int final, size_t *used, void *out, size_t out_cap, size_t *out_len, int *done);
/* a whole stream, device buffers, on the object's stream (returns after it is done); SSQ_ECAP with *out_len = the text's size
 * when it does not fit.  Independent of the streaming state. */
int ssq_gunzip_inflate_dev(ssq_gunzip_t *g, const void *d_in, size_t n, void *d_out, size_t out_cap, size_t *out_len);
/* BGZF, member-parallel (what BAI virtual offsets are made of): the members are found by walking the BSIZE chain (the BC extra
 * subfield) from byte 0, each is decoded as its own chunk and checked against its CRC-32 and ISIZE.  Device buffers, on the object's
 * stream.  members: host array of 2 * members_cap values, (compressed offset, text offset) of member k at [2k, 2k + 1].
 * SSQ_EDATA: a member without BSIZE, a chain that does not land on a member header or does not end exactly at n, a truncated or
 * corrupt member, ISIZE over 64 KB.  SSQ_ECAP (with *out_len and *n_members set): the text or the table does not fit.  Leaves
 * ssq_gunzip_stats alone. */
int ssq_gunzip_inflate_bgzf_dev(ssq_gunzip_t *g, const void *d_in, size_t n, void *d_out, size_t out_cap, size_t *out_len, uint64_t *members, size_t members_cap, size_t *n_members);
/* since create: chunks decoded, chunks started at a searched sync point, chunks decoded again after a broken link, windows */
int ssq_gunzip_stats(const ssq_gunzip_t *g, int64_t out[4]);
void *ssq_gunzip_stream(ssq_gunzip_t *g);           /* cudaStream_t of the object, for event timing */
void ssq_gunzip_free(ssq_gunzip_t *g);
/* samblaster over name-grouped SAM text on the device (csrc/ssq_sbtext.cu): what the `samblaster` shim does with SAM it did not get
 * from the fused stage (`speedseq realign`, the default config, any other aligner's output).  The same decision routines as the
 * fused stage (ssq_dev3.cuh sb_*), first-seen-wins duplicate marking against the object's dup-set, and the three streams as text:
 * FLAG re-printed in decimal with 0x400 on duplicates, MC:Z / MQ:i (the mate's CIGAR and MAPQ fields, verbatim) appended when
 * absent, splitter QNAMEs suffixed _1 / _2, --removeDups / --excludeDups applied.  Only '\n' ends a line ('\r' stays in the last
 * field); a last line without '\n' is taken when final.
 * header: the SAM header text; its @SQ lines define the contig ids (first SN wins) and samblaster's padded offsets (LN + 2*500 + 1
 * each).  One object = one run; one host thread at a time.  Without a usable GPU create returns SSQ_ENOGPU. */
typedef struct ssq_sbtext ssq_sbtext_t;
typedef struct {
	const char *text[3]; size_t len[3];   /* 0 main records, 1 splitters, 2 discordants; pinned, owned by the object, valid until its next run */
	uint64_t n_ids, n_dup, n_disc_lines, n_split_lines; /* QNAME blocks taken / marked duplicate; lines written to streams 2 and 1 */
} ssq_sbtext_out_t;
int ssq_sbtext_create(int device, const ssq_sb_opts_t *sb, const char *header, size_t header_len, ssq_sbtext_t **out);
/* text[0, len): record lines from a line start on (len < 2^31); final: nothing follows.  Processes whole QNAME blocks, at most
 * max_blocks of them (0 = no limit); the last block is held back unless final (the next line may continue it); *used = bytes
 * consumed (0 when no whole block is in the text yet: call again with more).  SSQ_EFORMAT: a line in the range the device does
 * not take — fewer than 11 fields, a NUL byte, FLAG or POS not plain digits, a CIGAR the parser does not fully consume, an RNAME
 * other than `*` not in @SQ, a QNAME block over 256 lines, a mapped primary line with RNAME `*`; nothing is consumed and
 * ssq_last_error() names the line (the caller runs its host code over these lines, marking through ssq_sbtext_dupset). */
int ssq_sbtext_run(ssq_sbtext_t *s, const char *text, size_t len, int final, uint64_t max_blocks, size_t *used, ssq_sbtext_out_t *out);
ssq_dupset_t *ssq_sbtext_dupset(ssq_sbtext_t *s);   /* the set it marks against, so that a host fallback can share it */
void *ssq_sbtext_stream(ssq_sbtext_t *s);           /* cudaStream_t of the object, for event timing */
void ssq_sbtext_free(ssq_sbtext_t *s);
/* SAM text -> BAM records on the device (csrc/ssq_sam2bam.cu): what `sambamba view -S -f bam` makes of each record line
 * (speedseq:440-448, :1964-1971), byte for byte for every line it takes, with the records of a call sorted the way `sambamba sort` orders them — by (tid,
 * pos, reverse strand), records without a reference last, equal keys in input order — so that the runs of consecutive calls merge
 * into the sorted file (ssq_bam_merge_runs; the `sambamba` shim's sort).  Encoding and the lines the device refuses: the head of
 * csrc/ssq_sam2bam.cuh; in short, RNAME / RNEXT must be `*`, `=` (RNEXT) or an @SQ name, QUAL `*` or as long as SEQ, tags one of
 * A i Z H B (not f or B:f: there is no float reader on the device) with i in [-2^31, 2^32), and every field within the byte class
 * sambamba's parser enforces (QNAME [!-?A-~], SEQ [A-Za-z=.], QUAL / A [!-~], Z [ -~], H hex, tag names [A-Za-z][A-Za-z0-9]):
 * sambamba silently drops or blanks a field outside its class, the device refuses the line.  Only '\n' ends a line; a '\r' before
 * it is dropped.  header: the SAM header text; its @SQ lines (with SN and LN) give the tids, the first SN of a name wins.  One
 * host thread at a time per object.  Without a usable GPU create returns SSQ_ENOGPU. */
typedef struct ssq_sam2bam ssq_sam2bam_t;
int ssq_sam2bam_create(int device, const char *header, size_t header_len, ssq_sam2bam_t **out);
/* text[0, len): record lines from a line start on (len < 2^31); final: nothing follows.  Converts the whole lines (a last line
 * without '\n' only when final) and returns them as ONE run of BAM records (block_size included) in the order above: *run is
 * pinned, owned by the object and valid until its next call; *n_records = lines converted; *used = bytes consumed (a trailing
 * partial line is left for the next call unless final).  SSQ_EFORMAT: a line the device refuses; nothing is consumed and
 * ssq_last_error() gives its number (from 1 at text[0]) and text. */
int ssq_sam2bam_run(ssq_sam2bam_t *t, const char *text, size_t len, int final, size_t *used, const void **run, size_t *run_len, uint64_t *n_records);
void *ssq_sam2bam_stream(ssq_sam2bam_t *t);         /* cudaStream_t of the object, for event timing */
void ssq_sam2bam_free(ssq_sam2bam_t *t);
/* The BAI index of a coordinate-sorted BAM file on the device (csrc/ssq_bai.cu): what `sambamba index in.bam` (0.5.9) writes to
 * in.bam.bai, byte for byte — the call speedseq makes on each BAM of `align` and `realign` (speedseq:486-494, :1983-1985,
 * :2016-2023), and what sambamba's `sort -o` writes next to its output.  The rules and what is refused are at the head of
 * csrc/ssq_bai.cuh; in short, SSQ_EDATA for input that is not BGZF or does not inflate, SSQ_EFORMAT (with the record in
 * ssq_last_error()) for a text that is not a BAM file, records out of coordinate order, a refID outside the header, a record with
 * a reference and no position, a record that reaches past 2^29, a record without a reference before one with one, and an empty
 * BGZF member before the last.  seg_bytes: text per record walker (0 = 64 KB).  One host thread at a time per object; without a
 * usable GPU create returns SSQ_ENOGPU. */
typedef struct ssq_bai ssq_bai_t;
int ssq_bai_create(int device, size_t seg_bytes, ssq_bai_t **out);
/* bam[0, len): the whole BAM file (host memory; staged through pinned memory).  *bai_out: the index file's bytes, free with
 * ssq_free. */
int ssq_bai_build(ssq_bai_t *b, const void *bam, size_t len, void **bai_out, size_t *bai_len);
/* time of the last build in ms between CUDA events on the object's stream: 0 the input's staging through pinned memory, its copy
 * in and the BGZF inflation (host work between the member rounds included), 1 record walk and checks, 2 index assembly and the
 * copy back (the host's link checks and waits included in each) */
int ssq_bai_times(const ssq_bai_t *b, float ms[3]);
void *ssq_bai_stream(ssq_bai_t *b);                 /* cudaStream_t of the object, for event timing */
void ssq_bai_free(ssq_bai_t *b);
/* The merge of coordinate-sorted BAM files on the device (csrc/ssq_merge.cu): the records in the order `sambamba merge out.bam
 * in1.bam in2.bam ...` (0.5.9) writes them, and its merged header — the calls of `speedseq realign` with several libraries
 * (speedseq:2002-2009).  The inputs stream through windows of whole BGZF members of at most window_bytes compressed bytes each
 * (0 = 32 MB), so they need not fit in device memory.  The rules and what is refused are at the head of csrc/ssq_merge.cuh; in
 * short, SSQ_EDATA for an input that is not BGZF or does not inflate, SSQ_EFORMAT (the file and record in ssq_last_error()) for
 * headers that do not merge the way the device merges them (not all SO:coordinate, @HD lines or @SQ dictionaries that differ, an
 * @RG / @PG ID carried by two different lines, other header lines), a refID outside the header and records out of coordinate
 * order, SSQ_EINVAL for fewer than two inputs.  One host thread at a time per object; without a usable GPU create returns
 * SSQ_ENOGPU. */
typedef struct ssq_merge ssq_merge_t;
/* the output, piece by piece in file order; nonzero stops the merge (SSQ_EIO) */
typedef int (*ssq_merge_sink_t)(void *ctx, const void *p, size_t n);
int ssq_merge_create(int device, size_t window_bytes, ssq_merge_t **out);
/* paths[0, n_in): the inputs.  sink receives the merged file without its end-of-file block: the uncompressed BAM ("BAM\1", header,
 * reference table, records) when z is null; with z, BGZF members at `level` compressed on the device, the header in blocks of its
 * own.  Something may have reached sink before an error.  *n_records (may be null): records written. */
int ssq_merge_run(ssq_merge_t *m, const char *const *paths, int n_in, ssq_bgzf_t *z, int level, ssq_merge_sink_t sink, void *ctx, uint64_t *n_records);
/* the merged header text alone (`sambamba merge -H`), read on the host; the refusals of the header.  Free with ssq_free */
int ssq_merge_header(const char *const *paths, int n_in, char **text);
/* the last run in ms of host clock around synchronised work: 0 windows (read, copy in, inflate, record walk, keys), 1 the host heap,
 * 2 gathers and the output (compression on the device, the copy back and the sink included) */
int ssq_merge_times(const ssq_merge_t *m, float ms[3]);
void *ssq_merge_stream(ssq_merge_t *m);             /* cudaStream_t of the object, for event timing */
void ssq_merge_free(ssq_merge_t *m);
/* the sorted runs of consecutive batches -> one sorted record stream (stable: equal keys keep batch order); free with ssq_free */
int ssq_bam_merge_runs(int n_runs, const void *const *runs, const size_t *lens, void **out, size_t *out_len);

/* ------------------------------------------------------------------ several GPUs ----
 * Batches are dealt to the ranks round-robin with the index replicated (no collective); "first pair seen with a signature is
 * kept" (`$SAMBLASTER`, speedseq:439) stays global through one exchange per round, in C over NCCL: signatures go to the owner rank
 * hash(signature) mod N (grouped ncclSend/ncclRecv, 16 B per pair), the owner marks them against everything it has owned so far,
 * one byte per pair comes back (csrc/ssq_dist.cu).  One process per GPU: rank 0 makes the id, every rank creates its communicator
 * and hands it to its aligner object(s); ssq_aligner_compute then performs the round inside its duplicate stage (a collective: all
 * ranks run the same number of batches, empty ones included). */
typedef struct ssq_comm ssq_comm_t;
int ssq_comm_unique_id(void *id128);  /* 128 bytes, to be broadcast to the other ranks by whatever launched them */
int ssq_comm_create(const void *id128, int rank, int world, int device, ssq_comm_t **out);
int ssq_aligner_set_comm(ssq_aligner_t *al, ssq_comm_t *comm);
/* one round on explicit device arrays (key = 5' position << 1 | strand of the canonically ordered ends, array order = input order) */
int ssq_comm_mark_round(ssq_comm_t *comm, uint64_t n, const uint64_t *d_key1, const uint64_t *d_key2, const uint8_t *d_valid, uint8_t *d_is_dup, void *stream);
ssq_dupset_t *ssq_comm_dupset(ssq_comm_t *comm);            /* the signatures this rank owns (reset it on every rank to start a new run) */
uint64_t ssq_comm_counter(const ssq_comm_t *comm, int what); /* 0 bytes sent to other ranks, 1 bytes received back, 2 rounds */
void ssq_comm_free(ssq_comm_t *comm);

/* streaming dup-set on device pointers (what the aligner uses; also the owner-side step of the multi-GPU exchange) */
int ssq_dupset_mark_dev(ssq_dupset_t *set, uint64_t n, const uint64_t *d_key1, const uint64_t *d_key2, const uint8_t *d_valid, uint8_t *d_is_dup, void *stream);
int ssq_dupset_reset(ssq_dupset_t *set);
/* contig table for the SAM header: name/length of contig i (0 <= i < ssq_index_info(idx,3)) */
const char *ssq_index_contig(const ssq_index_t *idx, int i, int64_t *len);

#ifdef __cplusplus
}
#endif
#endif
