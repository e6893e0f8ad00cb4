/*
 * ssqo.h — CPU ORACLE for the `speedseq align` hot path.  TEST INFRASTRUCTURE ONLY.
 *
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * link or execute anything under oracle/.  The product (speedseq_b200/) never does.
 *
 * What it restates: the arithmetic behind `$BWA mem` and `$SAMBLASTER` as called at
 * speedseq/bin/speedseq:438-439,468-469 (and `$BWA index` at :389).  Those two tools are
 * un-vendored submodules in the reference checkout (src/bwa, src/samblaster are EMPTY; pins in
 * speedseq/.SUBMODULES.json:23-29,51-57 = lh3/bwa@d82444c1, GregoryFaust/samblaster@b6426391),
 * so this file set restates their *published* algorithms (BWA-MEM 0.7.12-series behaviour,
 * samblaster 0.1.2x behaviour; SURVEY.md Appendix A/B) in plain scalar C.
 *
 * PARITY STATUS
 *   - index build/load (.amb .ann .pac .bwt .sa): PINNED by the reference's own golden files
 *     speedseq/example/data/human_g1k_v37_20_42220611-42542245.fasta.{amb,ann,pac,bwt,sa}
 *     (tests/test_oracle_index.py rebuilds them byte-for-byte; a copy of the goldens' sha256 and a
 *     small derived fixture live under tests/golden/).
 *   - alignment records / dup flags / discordant+splitter sets: **parity unpinned** — the reference
 *     tree holds no golden SAM/BAM or known-answer vector for them (SURVEY.md §8c).
 */
#ifndef SSQO_H
#define SSQO_H
#include <stdint.h>
#include <stddef.h>
#include <stdio.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------ index ---- */
typedef struct {
	int64_t offset;
	int32_t len, n_ambs;
	uint32_t gi;
	char *name, *anno;
} ssqo_ann_t;

typedef struct { int64_t offset; int32_t len; char amb; } ssqo_hole_t;

typedef struct {
	int64_t l_pac;
	int32_t n_seqs;
	uint32_t seed;
	ssqo_ann_t *anns;
	int32_t n_holes;
	ssqo_hole_t *holes;
} ssqo_bns_t;

typedef struct {
	uint64_t primary, L2[5], seq_len; /* seq_len = 2*l_pac */
	uint64_t bwt_size;                /* in u32 words, occ-interleaved layout */
	uint32_t *bwt;
	int sa_intv;
	uint64_t n_sa;
	uint64_t *sa;
} ssqo_bwt_t;

typedef struct {
	ssqo_bwt_t bwt;
	ssqo_bns_t bns;
	uint8_t *pac; /* forward strand, 2 bit/base */
} ssqo_idx_t;

/* `bwa index` (speedseq:389): FASTA -> prefix.{amb,ann,pac,bwt,sa}. returns 0 on success */
int ssqo_index_build(const char *fasta, const char *prefix);
ssqo_idx_t *ssqo_idx_load(const char *prefix);
void ssqo_idx_destroy(ssqo_idx_t *idx);

/* suffix array of s[0..n) over alphabet [0,K), s[n-1] must be the unique smallest symbol */
void ssqo_sais(const int32_t *s, int32_t *sa, int32_t n, int32_t K);

/* --------------------------------------------------------------- FM index ---- */
typedef struct { uint64_t x[3], info; } ssqo_intv_t; /* x[0]=fwd k, x[1]=rev k, x[2]=size; info=qbeg<<32|qend */
typedef struct { size_t n, m; ssqo_intv_t *a; } ssqo_intv_v;

void ssqo_occ4(const ssqo_bwt_t *b, uint64_t k, uint64_t cnt[4]);
uint64_t ssqo_occ(const ssqo_bwt_t *b, uint64_t k, int c);
void ssqo_extend(const ssqo_bwt_t *b, const ssqo_intv_t *ik, ssqo_intv_t ok[4], int is_back);
int ssqo_smem1(const ssqo_bwt_t *b, int len, const uint8_t *q, int x, int min_intv, ssqo_intv_v *mem, ssqo_intv_v tmp[2]);
int ssqo_seed_strategy1(const ssqo_bwt_t *b, int len, const uint8_t *q, int x, int min_len, int max_intv, ssqo_intv_t *mem);
uint64_t ssqo_sa(const ssqo_bwt_t *b, uint64_t k);

/* counters that define the algorithmic bytes of the FM kernels (SURVEY.md §8d) */
typedef struct {
	uint64_t n_extend, n_occblk, n_sa, n_sa_steps;
	uint64_t n_sw_calls, sw_cells, sw_bytes;
} ssqo_counters_t;
extern __thread ssqo_counters_t ssqo_cnt;

/* -------------------------------------------------------------------- SW ---- */
int ssqo_ksw_extend2(int qlen, const uint8_t *query, int tlen, const uint8_t *target, int m, const int8_t *mat,
                     int o_del, int e_del, int o_ins, int e_ins, int w, int end_bonus, int zdrop, int h0,
                     int *qle, int *tle, int *gtle, int *gscore, int *max_off);
int ssqo_ksw_global2(int qlen, const uint8_t *query, int tlen, const uint8_t *target, int m, const int8_t *mat,
                     int o_del, int e_del, int o_ins, int e_ins, int w, int *n_cigar, uint32_t **cigar);
typedef struct { int score, te, qe, score2, te2, tb, qb; } ssqo_kswr_t;
#define SSQO_KSW_XBYTE  0x10000
#define SSQO_KSW_XSTOP  0x20000
#define SSQO_KSW_XSUBO  0x40000
#define SSQO_KSW_XSTART 0x80000
ssqo_kswr_t ssqo_ksw_align2(int qlen, uint8_t *query, int tlen, uint8_t *target, int m, const int8_t *mat,
                            int o_del, int e_del, int o_ins, int e_ins, int xtra);

/* ------------------------------------------------------------------- mem ---- */
typedef struct {
	int a, b, o_del, e_del, o_ins, e_ins, pen_unpaired, pen_clip5, pen_clip3, w, zdrop;
	uint64_t max_mem_intv;
	int T, flag, min_seed_len, min_chain_weight, max_chain_extend;
	float split_factor;
	int split_width, max_occ, max_chain_gap, n_threads, chunk_size;
	float mask_level, drop_ratio, XA_drop_ratio, mask_level_redun, mapQ_coef_len;
	int mapQ_coef_fac, max_ins, max_matesw, max_XA_hits, max_XA_hits_alt;
	int8_t mat[25];
} ssqo_opt_t;
#define SSQO_F_PE 0x2
void ssqo_opt_init(ssqo_opt_t *o);

typedef struct { int64_t rbeg; int32_t qbeg, len, score; } ssqo_seed_t;
typedef struct {
	int n, m, first, rid;
	uint32_t w:29, kept:2, is_alt:1;
	float frac_rep;
	int64_t pos;
	ssqo_seed_t *seeds;
} ssqo_chain_t;
typedef struct { size_t n, m; ssqo_chain_t *a; } ssqo_chain_v;

typedef struct {
	int64_t rb, re;
	int qb, qe;
	int rid;
	int score, truesc, sub, alt_sc, csub, sub_n, w, seedcov, secondary, secondary_all, seedlen0;
	int n_comp:30, is_alt:2;
	float frac_rep;
	uint64_t hash;
} ssqo_alnreg_t;
typedef struct { size_t n, m; ssqo_alnreg_t *a; } ssqo_alnreg_v;

typedef struct { int low, high, failed; double avg, std; } ssqo_pestat_t;

typedef struct {
	int l_seq, id;
	char *name, *comment, *seq, *qual, *sam;
} ssqo_read_t;

/* stage-level entry points (the parity tests compare the CUDA kernels against these) */
void ssqo_collect_intv(const ssqo_opt_t *opt, const ssqo_bwt_t *bwt, int len, const uint8_t *seq, ssqo_intv_v *out);
ssqo_chain_v ssqo_mem_chain(const ssqo_opt_t *opt, const ssqo_idx_t *idx, int len, const uint8_t *seq);
int ssqo_chain_flt(const ssqo_opt_t *opt, int n_chn, ssqo_chain_t *a);
void ssqo_chain2aln(const ssqo_opt_t *opt, const ssqo_idx_t *idx, int l_query, const uint8_t *query, const ssqo_chain_t *c, ssqo_alnreg_v *av);
ssqo_alnreg_v ssqo_align1(const ssqo_opt_t *opt, const ssqo_idx_t *idx, int l_seq, char *seq /* ascii or nt4, converted in place */);
int ssqo_sort_dedup_patch(const ssqo_opt_t *opt, const ssqo_idx_t *idx, uint8_t *query, int n, ssqo_alnreg_t *a);
int ssqo_mark_primary_se(const ssqo_opt_t *opt, int n, ssqo_alnreg_t *a, int64_t id);
int ssqo_approx_mapq_se(const ssqo_opt_t *opt, const ssqo_alnreg_t *a);
void ssqo_pestat(const ssqo_opt_t *opt, int64_t l_pac, int n, const ssqo_alnreg_v *regs, ssqo_pestat_t pes[4]);

/* whole `bwa mem` batch: reads (already name-trimmed) -> reads[i].sam ; n_processed = global read ordinal of reads[0] */
void ssqo_process_seqs(const ssqo_opt_t *opt, const ssqo_idx_t *idx, int64_t n_processed, int n, ssqo_read_t *reads,
                       const ssqo_pestat_t *pes0, const char *rg_id);

/* utility: reference fetch (2*l_pac coordinate space) */
uint8_t *ssqo_get_seq(int64_t l_pac, const uint8_t *pac, int64_t beg, int64_t end, int64_t *len);
int ssqo_pos2rid(const ssqo_bns_t *bns, int64_t pos_f);
int ssqo_intv2rid(const ssqo_bns_t *bns, int64_t rb, int64_t re);
uint64_t ssqo_hash64(uint64_t key);

/* CLI mains */
int ssqo_main_index(int argc, char **argv);
int ssqo_main_mem(int argc, char **argv);
int ssqo_main_samblaster(int argc, char **argv);

/* ------------------------------------------------------------ samblaster ---- */
/* batch form used by the GPU dup-mark parity tests: one signature per pair, first-seen wins */
typedef struct { uint64_t pos1, pos2; uint8_t strand1, strand2, valid; } ssqo_dupsig_t;
void ssqo_dupmark(size_t n, const ssqo_dupsig_t *sig, uint8_t *is_dup);

#ifdef __cplusplus
}
#endif
#endif
