// ssq_pipe.cu — `bwa mem | samblaster` for a batch of reads with everything between the FASTQ bytes and the three SAM streams
// resident in HBM.
//
// Reference call sites: `$BWA mem -t T [-p] [-C] [-I ..] -R RG REF FQ1 [FQ2] | $SAMBLASTER [--excludeDups] --addMateTags
// --maxSplitCount C --minNonOverlap M --splitterFile F --discordantFile F` at speedseq/bin/speedseq:438-439,468-469.
// Upstream routines replaced (un-vendored submodules of the reference): mem_process_seqs, mem_pestat, mem_sam_pe, mem_matesw,
// mem_pair, mem_mark_primary_se, mem_approx_mapq_se, mem_reg2aln, mem_gen_alt, mem_reg2sam, mem_aln2sam; samblaster's
// markDupsDiscordants, markSplitterUnmappedClipped and its line writer.
//
// Stages (all kernels hand-written for sm_90a; CUB only for scans and the radix sort inside the dup-set):
//   k_encode        ASCII bases -> one code per base
//   ssq_batch_run   seeding, SA look-up, chaining, extension                                   (ssq_kernels.cu)
//   k_dedup         sort / de-duplicate / patch the regions of a read                          (thread per read)
//   k_pestat        insert-size histogram of the batch                                         (thread per pair, atomics)
//     host:         quartiles / mean / std from the histogram (the reference's double sums replayed in sorted order),
//                   penalty table .721*log(2*erfc(|z|/sqrt2))*a over the integer insert sizes  -> back to the device
//   k_rescue_count  the rescue alignments the lists, as they stand, do not skip: count per pair   (thread per pair)
//   k_rescue_fill   ... as tasks (hit of the snapshot, orientation, window)                    (thread per marked pair)
//   k_rescue_sw     those alignments, striped-order local SW on all 32 lanes (ssq_warp.cuh)    (warp per task)
//   k_rescue        the reference's sequential rescue of a pair with the results looked up     (warp per marked pair)
//   k_plan          primary marking, pairing, MAPQ, list of alignments to write                (thread per pair / read)
//   k_cigar_fast / k_cigar_warp   position / CIGAR / NM / MD: ungapped per thread, banded DP + traceback per warp
//   k_sb            samblaster: pair signature, discordant bit, splitter masks                 (thread per pair / read)
//   dup-set         first-seen-wins over all batches of the run                                (ssq_kernels.cu)
//   k_text<false>   byte counts of each read's records in the three streams; scans
//   k_text<true>    the text
// Host round trips per batch: the size queries inside ssq_batch_run, the histogram, the rescue-task count, the task count and the
// text sizes.
#include <cuda_runtime.h>
#include <cub/cub.cuh>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "ssq_dev3.cuh"
#include "ssq_warp.cuh"
#include "ssq_pipe_host.h"
#include "ssq_host.h"
#include "ssq_batch.h"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { ssq_set_error("%s:%d: %s", __FILE__, __LINE__, cudaGetErrorString(e_)); return SSQ_ECUDA; } } while (0)
#define QMAX 256

// streaming dup-set, device-pointer form (ssq_kernels.cu)
extern "C" int ssq_dupset_mark_dev(ssq_dupset_t *set, uint64_t n, const uint64_t *d_k1, const uint64_t *d_k2, const uint8_t *d_valid, uint8_t *d_is_dup, void *stream);
extern "C" int ssq_dupset_reset(ssq_dupset_t *set);
extern "C" void ssq_dupset_wait_turn(ssq_dupset_t *set, long long turn);
extern "C" void ssq_dupset_end_turn(ssq_dupset_t *set, long long turn);
// multi-GPU exchange (ssq_dist.cu)
extern "C" int ssq_comm_mark_round(ssq_comm_t *c, uint64_t n, const uint64_t *d_k1, const uint64_t *d_k2, const uint8_t *d_valid, uint8_t *d_is_dup, void *stream);
extern "C" ssq_dupset_t *ssq_comm_dupset(ssq_comm_t *c);

// ================================================================================ kernels ====
__global__ void __launch_bounds__(256) k_encode(u64 n, const char *__restrict__ ascii, uint8_t *__restrict__ codes)
{
	const u64 i = ((u64)blockIdx.x * blockDim.x + threadIdx.x) * 4;
	if (i >= n) return;
#pragma unroll
	for (int k = 0; k < 4; ++k) {
		if (i + k >= n) break;
		const int c = ascii[i + k] | 0x20;
		codes[i + k] = c == 'a' ? 0 : c == 'c' ? 1 : c == 'g' ? 2 : c == 't' ? 3 : 4;
	}
}

// capacity of a read's region list: its own regions plus at most 4 rescued ones per mate hit that may trigger a rescue
__global__ void k_areg_cap(int n, int paired, int max_matesw, const u32 *__restrict__ n_regs, u64 *cap)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	u32 m = paired ? n_regs[i ^ 1] : 0;
	if (m > (u32)max_matesw) m = (u32)max_matesw;
	cap[i] = (u64)n_regs[i] + 4ull * m + (paired ? 4 : 0);
}

struct DedupSlab { i32 h[QMAX + 16], e[QMAX + 16]; uint8_t qbuf[QMAX], rbuf[2048]; };
__global__ void __launch_bounds__(128) k_dedup(PipeView V, DedupSlab *slabs, int *work)
{
	DedupSlab &s = slabs[(size_t)blockIdx.x * blockDim.x + threadIdx.x];
	AlnScratch A; A.qbuf = s.qbuf; A.rbuf = s.rbuf; A.rcap = 2048; A.g.h = s.h; A.g.e = s.e; A.g.z = 0; A.g.zcap = 0;
	(void)work;
	for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < V.n_reads; r += gridDim.x * blockDim.x) body_dedup(V, r, A); // neighbouring lanes take neighbouring reads: their region lists are adjacent in memory
}

__global__ void __launch_bounds__(256) k_pestat(PipeView V)
{
	const int p = blockIdx.x * blockDim.x + threadIdx.x;
	if (p >= V.n_reads >> 1) return;
	int dir; i64 is;
	if (body_pestat(V, p, &dir, &is)) atomicAdd(&V.hist[(size_t)dir * V.hist_n + is], 1u);
}

__global__ void __launch_bounds__(256) k_rescue_mark(PipeView V, u32 *list, unsigned int *n_list)
{
	const int p = blockIdx.x * blockDim.x + threadIdx.x;
	if (p >= V.n_reads >> 1) return;
	if (rescue_wanted(V, p)) list[atomicAdd(n_list, 1u)] = (u32)p;
}
// speculative form (ssq_dev2.cuh, RTask): the pairs with at least one rescue alignment the initial lists do not skip, each with a
// contiguous range of tasks
__global__ void __launch_bounds__(256) k_rescue_count(PipeView V, int win_cap, u32 *list, u32 *t_base, u32 *t_cnt, unsigned int *n_list, unsigned int *n_tasks)
{
	const int p = blockIdx.x * blockDim.x + threadIdx.x;
	if (p >= V.n_reads >> 1) return;
	const int c = rescue_enum(V, p, 0, 0, win_cap);
	if (c) { const unsigned int slot = atomicAdd(n_list, 1u); list[slot] = (u32)p; t_cnt[slot] = (u32)c; t_base[slot] = atomicAdd(n_tasks, (unsigned int)c); }
}
__global__ void __launch_bounds__(256) k_rescue_fill(PipeView V, int win_cap, const u32 *__restrict__ list, const u32 *__restrict__ t_base, const unsigned int *__restrict__ n_list, RTask *tasks)
{
	const unsigned int slot = blockIdx.x * blockDim.x + threadIdx.x;
	if (slot < *n_list) rescue_enum(V, (int)list[slot], tasks + t_base[slot], slot, win_cap);
}

// mate rescue: one warp per marked pair (ssq_warp.cuh).  Per-warp global scratch: the snapshot of the near-best hits of both ends
// (2 x 64 regions) and the list of sub-optimal rows of the current alignment (win_cap entries); DP state lives in shared memory
struct RescueCfg { int win_cap; size_t slab_bytes; };
// the alignments computed ahead: one warp per task, all of about the same size (one window), so the kernel has no tail
__global__ void __launch_bounds__(128) k_rescue_sw(PipeView V, const u32 *__restrict__ list, const RTask *__restrict__ tasks, const unsigned int *__restrict__ n_tasks, LocalRes *res, uint8_t *slabs, RescueCfg cfg, int *work)
{
	__shared__ WarpSwSmem sm[4];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	u64 *bl = (u64*)(slabs + ((size_t)blockIdx.x * 4 + wid) * cfg.slab_bytes + 128 * sizeof(AlnReg));
	const unsigned int n = *n_tasks;
	for (;;) {
		unsigned int k = 0;
		if (lane == 0) k = (unsigned int)atomicAdd(work, 1);
		k = __shfl_sync(WFULL, k, 0);
		if (k >= n) break;
		const RTask t = tasks[k];
		const LocalRes r = rescue_task_warp(V, t, (int)list[t.slot], sm[wid], bl, cfg.win_cap, lane);
		if (lane == 0) res[k] = r;
	}
}
// the replay: tasks == 0: every alignment is computed where the replay needs it
__global__ void __launch_bounds__(128) k_rescue(PipeView V, const u32 *__restrict__ list, const unsigned int *__restrict__ n_list, uint8_t *slabs, RescueCfg cfg, int *work,
                                                 const RTask *__restrict__ tasks, const LocalRes *__restrict__ res, const u32 *__restrict__ t_base, const u32 *__restrict__ t_cnt, unsigned int *n_miss)
{
	__shared__ WarpSwSmem sm[4];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	uint8_t *p = slabs + ((size_t)blockIdx.x * 4 + wid) * cfg.slab_bytes;
	AlnReg *bbuf = (AlnReg*)p;
	u64 *bl = (u64*)(p + 128 * sizeof(AlnReg));
	const unsigned int n = *n_list;
	for (;;) {
		unsigned int k = 0;
		if (lane == 0) k = (unsigned int)atomicAdd(work, 1);
		k = __shfl_sync(WFULL, k, 0);
		if (k >= n) break;
		if (tasks) {
			RCache rc; rc.t = tasks + t_base[k]; rc.res = res + t_base[k]; rc.n = (int)t_cnt[k]; rc.cur = 0; rc.miss = n_miss;
			body_rescue_warp(V, (int)list[k], bbuf, sm[wid], bl, cfg.win_cap, lane, &rc);
		} else body_rescue_warp(V, (int)list[k], bbuf, sm[wid], bl, cfg.win_cap, lane);
	}
}

__global__ void k_tslot_cap(int n, const u32 *__restrict__ n_areg, u64 *cap)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) cap[i] = 2ull * n_areg[i] + 1;
}
__global__ void __launch_bounds__(128) k_plan(PipeView V)
{
	const int u = blockIdx.x * blockDim.x + threadIdx.x;
	if (u >= (V.paired ? V.n_reads >> 1 : V.n_reads)) return;
	body_plan(V, u);
}
__global__ void k_ntasks(int n, const ReadMeta *__restrict__ meta, u64 *out)
{
	const int i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) out[i] = meta[i].n_tasks;
}
__global__ void k_compact(PipeView V)
{
	const int r = blockIdx.x * blockDim.x + threadIdx.x;
	if (r >= V.n_reads) return;
	const PTask *src = V.tslots + V.tslot_off[r];
	PTask *dst = V.tasks + V.tk_base[r];
	const int n = V.meta[r].n_tasks;
	for (int i = 0; i < n; ++i) dst[i] = src[i];
}

// CIGAR generation in two kernels.  k_cigar_fast (thread per alignment) finishes the alignments that need no dynamic programming
// — query and reference span of equal length and a zero band, i.e. at most two mismatches and no indel: more than nine in ten —
// and lists the others; k_cigar_warp gives every listed alignment a warp (banded global DP with lanes = band columns, ssq_warp.cuh).
__global__ void __launch_bounds__(128) k_cigar_fast(PipeView V, u64 n_tasks, u32 *gapped, unsigned int *n_gapped)
{
	const u64 t = (u64)blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= n_tasks) return;
	const PTask tk = V.tasks[t];
	const AlnReg &ar = V.areg[V.areg_off[tk.read] + tk.reg_idx];
	const ssq_opts_t &o = V.opt;
	const int lq = ar.qe - ar.qb, lr = (int)(ar.re - ar.rb);
	int tmp = infer_bw(lq, lr, ar.truesc, o.a, o.o_del, o.e_del), w2 = infer_bw(lq, lr, ar.truesc, o.a, o.o_ins, o.e_ins);
	w2 = w2 > tmp ? w2 : tmp;
	if (w2 > o.w) w2 = w2 < ar.w ? w2 : ar.w;
	const bool invalid = lq <= 0 || ar.rb >= ar.re || (ar.rb < V.ix.l_pac && ar.re > V.ix.l_pac);
	if (!invalid && !(lq == lr && w2 == 0)) { gapped[atomicAdd(n_gapped, 1u)] = (u32)t; return; } // (a zero band stays zero when the reference doubles it)
	uint8_t qbuf[QMAX], rbuf[QMAX];
	AlnScratch A; A.qbuf = qbuf; A.rbuf = rbuf; A.rcap = QMAX; A.g.h = A.g.e = 0; A.g.z = 0; A.g.zcap = 0;
	AlnOut a;
	reg2aln(V.ix, o, (int)(V.tc.read_off[tk.read + 1] - V.tc.read_off[tk.read]), V.tc.seq + V.tc.read_off[tk.read], ar, A, a, V.cigs + t * CIG_CAP, CIG_CAP, V.mds + t * MD_CAP, MD_CAP);
	if (a.n_cigar < 0 || a.n_cigar > CIG_CAP - 2 || a.md_len >= MD_CAP) PIPE_ERR(V, 4);
	V.outs[t] = a;
}
__global__ void __launch_bounds__(128) k_cigar_warp(PipeView V, const u32 *__restrict__ gapped, const unsigned int *__restrict__ n_gapped, uint8_t *zslabs, long zcap, int *work)
{
	__shared__ WarpGlSmem sm[4];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	uint8_t *z = zslabs + ((size_t)blockIdx.x * 4 + wid) * (size_t)zcap;
	const unsigned int n = *n_gapped;
	for (;;) {
		unsigned int k = 0;
		if (lane == 0) k = (unsigned int)atomicAdd(work, 1);
		k = __shfl_sync(WFULL, k, 0);
		if (k >= n) break;
		const u64 t = gapped[k];
		const PTask tk = V.tasks[t];
		const AlnReg &ar = V.areg[V.areg_off[tk.read] + tk.reg_idx];
		AlnOut a;
		reg2aln_warp(V.ix, V.opt, (int)(V.tc.read_off[tk.read + 1] - V.tc.read_off[tk.read]), V.tc.seq + V.tc.read_off[tk.read], ar, sm[wid], z, zcap, a, V.cigs + t * CIG_CAP, CIG_CAP,
		             V.mds + t * MD_CAP, MD_CAP, lane);
		if (lane == 0) {
			if (a.n_cigar < 0 || a.n_cigar > CIG_CAP - 2 || a.md_len >= MD_CAP) PIPE_ERR(V, 4);
			V.outs[t] = a;
		}
	}
}

// kernel-level entry: ksw_align2 problems over caller-supplied sequences, one warp each (parity target: the oracle's ssqo_ksw_align2)
__global__ void __launch_bounds__(128) k_sw_local_tasks(ssq_opts_t opt, u64 n, const ssq_swl_task_t *__restrict__ tk, const uint8_t *__restrict__ qbuf, const uint8_t *__restrict__ tbuf, ssq_swl_result_t *out,
                                                        u64 *bl_all, int b_cap)
{
	__shared__ WarpSwSmem sm[4];
	const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
	const u64 t = (u64)blockIdx.x * 4 + wid;
	if (t >= n) return;
	WarpSwSmem &W = sm[wid];
	const ssq_swl_task_t k = tk[t];
	for (int i = lane; i < k.qlen; i += 32) W.q[i] = qbuf[k.q_off + i];
	__syncwarp();
	TgtBuf tg; tg.t = tbuf + k.t_off;
	const LocalRes r = sw_local_warp(opt, k.qlen, k.tlen, tg, k.xtra, W, bl_all + t * (u64)b_cap, b_cap, lane);
	if (lane == 0) { ssq_swl_result_t o; o.score = r.score; o.te = r.te; o.qe = r.qe; o.score2 = r.score2; o.te2 = r.te2; o.tb = r.tb; o.qb = r.qb; out[t] = o; }
}

__global__ void __launch_bounds__(128) k_sb(PipeView V)
{
	const int u = blockIdx.x * blockDim.x + threadIdx.x;
	if (u >= (V.paired ? V.n_reads >> 1 : V.n_reads)) return;
	body_sb(V, u);
}
template <bool W>
__global__ void __launch_bounds__(128) k_text(PipeView V)
{
	const int r = blockIdx.x * blockDim.x + threadIdx.x;
	if (r >= V.n_reads) return;
	body_text<W>(V, r);
}
// ---- BAM stage (optional, SURVEY §8 f1): records encoded from the structured alignments, coordinate-sorted per batch ----
__global__ void k_nlines(int n, PipeView V, u64 *out) { const int r = blockIdx.x * blockDim.x + threadIdx.x; if (r < n) out[r] = (u64)read_n_lines(V, r); }
__global__ void __launch_bounds__(128) k_bam_size(PipeView V) { const int r = blockIdx.x * blockDim.x + threadIdx.x; if (r < V.n_reads) body_bam_size(V, r); }
__global__ void k_iota_u32(u64 n, u32 *p) { const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; if (i < n) p[i] = (u32)i; }
__global__ void k_gather_u64(u64 n, const u32 *__restrict__ perm, const u64 *__restrict__ in, u64 *out) { const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; if (i < n) out[i] = in[perm[i]]; }
__global__ void __launch_bounds__(128) k_bam_write(PipeView V, u64 n_lines) { const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; if (i < n_lines) body_bam_write(V, i); }

__global__ void k_count_u8(u64 n, const uint8_t *__restrict__ a, const uint8_t *__restrict__ b, unsigned long long *out) // out[0] += #a, out[1] += #b
{
	const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	if (a[i]) atomicAdd(out, 1ull);
	if (b && b[i]) atomicAdd(out + 1, 1ull);
}

// ================================================================================== host ====
struct PinBuf { // growable pinned host buffer
	void *p; size_t cap;
	PinBuf() : p(0), cap(0) {}
	~PinBuf() { if (p) cudaFreeHost(p); }
	int need(size_t bytes) {
		if (bytes <= cap) return 0;
		if (p) cudaFreeHost(p);
		const size_t want = bytes + bytes / 4 + 4096;
		if (cudaMallocHost(&p, want) != cudaSuccess) { p = 0; cap = 0; ssq_set_error("cudaMallocHost(%zu) failed", want); return SSQ_ENOMEM; }
		cap = want; return 0;
	}
};

enum { ST_UPLOAD, ST_ALIGN, ST_DEDUP, ST_PESTAT, ST_RESCUE, ST_PLAN, ST_CIGAR, ST_SB, ST_TEXT, ST_FETCH, ST_N };

struct ssq_aligner {
	const ssq_index *idx; ssq_opts_t opt; SbOpts sb; int device, n_sm;
	char rg_id[256];
	cudaStream_t st;
	ssq_batch_t *b;
	ssq_comm_t *comm; // set: the dup stage is one round of the cross-GPU exchange instead of a local look-up
	ssq_dupset_t *dups; int own_dups; long long turn; // turn >= 0: the dup stage waits for the batches with smaller turn numbers (shared set)
	// static tables
	DBuf d_logn, d_lg, d_ctg_names, d_ctg_off, d_sb_off, d_rg;
	// batch inputs
	DBuf d_ascii, d_qual, d_names, d_name_off, d_cmt, d_cmt_off;
	// FASTQ ingest on the device: raw text of the two inputs, newline positions, per-record fields
	DBuf fq_txt[2], fq_nl[2], fq_rec[2], fq_len, fq_cum, fq_res, fq_nlen, fq_clen, fq_noff, fq_coff;
	int n_reads, paired, has_qual, has_cmt; i64 n_processed; u64 total_bases; int max_len;
	// stages
	DBuf cubtmp, d_cap, d_aoff, d_na, d_areg, d_work, d_pes, d_hist, d_pen, d_slab /* per-thread scratch of whichever slab kernel runs (dedup, rescue, CIGAR tiers: never live together) */, d_rlist, d_tcap, d_tsoff, d_tslots, d_meta, d_pv, d_xcnt,
	     d_ntk, d_tkbase, d_tasks, d_outs, d_cigs, d_mds, d_redo, d_k1, d_k2, d_valid, d_dup, d_disc, d_smask, d_len[3], d_off[3], d_text[3], d_err, d_cnt;
	PinBuf h_text[3], h_roff, h_hist, h_small, h_bam[3];
	int want_bam, bam_blank_side; u64 bam_len[3], n_lines_total;
	int rescue_spec; DBuf d_rtbase, d_rtcnt, d_rtasks, d_rres; // speculative mate rescue: task ranges per marked pair, tasks, their results
	DBuf d_nl, d_lbase, d_lread, d_bkey, d_bkey2, d_bidx, d_bperm, d_bsize[3], d_bsz_s, d_boff[3], d_bam[3];
	PeStat pes[4];
	u64 text_len[3]; u64 n_tasks_total, n_ids, n_dup, n_disc_lines, n_split_lines, n_rescue_pairs, n_gapped, n_sw_local, sw_local_cells;
	cudaEvent_t ev[ST_N + 1];
	float stage_ms[ST_N];
	int computed;
};

static int scan_u64(ssq_aligner *a, const u64 *in, u64 *out, size_t n) // exclusive sum, out[n] = total
{
	size_t tmp = 0;
	cub::DeviceScan::ExclusiveSum(0, tmp, in, out, (int)n, a->st);
	if (a->cubtmp.need(tmp)) return SSQ_ENOMEM;
	CK(cub::DeviceScan::ExclusiveSum(a->cubtmp.p, tmp, in, out, (int)n, a->st));
	return 0;
}

extern "C" void ssq_sb_opts_default(ssq_sb_opts_t *o)
{
	memset(o, 0, sizeof *o);
	o->max_split_count = 2; o->min_non_overlap = 20; o->min_indel_size = 50; o->max_unmapped_bases = 50;
}

extern "C" void ssq_aligner_free(ssq_aligner_t *a)
{
	if (!a) return;
	cudaSetDevice(a->device);
	if (a->b) ssq_batch_free(a->b);
	if (a->dups && a->own_dups) ssq_dupset_free(a->dups);
	for (int i = 0; i <= ST_N; ++i) if (a->ev[i]) cudaEventDestroy(a->ev[i]);
	delete a;
}

extern "C" int ssq_aligner_create(const ssq_index_t *idx, const ssq_opts_t *opt, const ssq_sb_opts_t *sb, const char *rg_id, ssq_aligner_t **out)
{
	if (!idx || !opt || !out) return SSQ_EINVAL;
	int rc = ssq_use_device(idx->device);
	if (rc) return rc;
	if (getenv("SSQ_RESCUE_SPLIT")) { const int v = atoi(getenv("SSQ_RESCUE_SPLIT")); CK(cudaMemcpyToSymbol(ssq_rescue_split, &v, sizeof v)); } // 0: the 16-lane form of the local SW (ssq_warp.cuh)
	ssq_aligner *a = new ssq_aligner();
	a->idx = idx; a->opt = *opt; a->device = idx->device; a->b = 0; a->comm = 0; a->dups = 0; a->own_dups = 1; a->turn = -1; a->want_bam = 0; a->bam_blank_side = 1; a->bam_len[0] = a->bam_len[1] = a->bam_len[2] = 0; a->n_lines_total = 0; a->computed = 0; a->n_reads = 0;
	a->rescue_spec = !(getenv("SSQ_RESCUE_SPEC") && !atoi(getenv("SSQ_RESCUE_SPEC"))); // 0: every rescue alignment computed inside the sequential replay
	memset(a->ev, 0, sizeof a->ev); memset(a->stage_ms, 0, sizeof a->stage_ms); memset(a->pes, 0, sizeof a->pes);
	memset(&a->sb, 0, sizeof a->sb);
	if (sb) {
		a->sb.enabled = sb->enabled; a->sb.excludeDups = sb->exclude_dups; a->sb.addMateTags = sb->add_mate_tags; a->sb.maxSplitCount = sb->max_split_count;
		a->sb.minNonOverlap = sb->min_non_overlap; a->sb.minIndelSize = sb->min_indel_size; a->sb.maxUnmappedBases = sb->max_unmapped_bases;
		a->sb.removeDups = sb->remove_dups; a->sb.want_split = sb->want_split; a->sb.want_disc = sb->want_disc;
	}
	snprintf(a->rg_id, sizeof a->rg_id, "%s", rg_id ? rg_id : "");
	cudaDeviceProp prop;
	CK(cudaGetDeviceProperties(&prop, idx->device));
	a->n_sm = prop.multiProcessorCount;
	if ((rc = ssq_batch_create(idx, opt, 0, 0, 0, &a->b))) { ssq_aligner_free(a); return rc; }
	a->st = (cudaStream_t)ssq_batch_stream(a->b);
	if ((rc = ssq_dupset_create(idx->device, &a->dups))) { ssq_aligner_free(a); return rc; }
	for (int i = 0; i <= ST_N; ++i) CK(cudaEventCreate(&a->ev[i]));
	{ // tables over integers, computed with the host's libm exactly as the reference evaluates them (see ssq_dev3.cuh)
		const int n_logn = 8192, n_lg = 65536;
		std::vector<double> logn(n_logn); std::vector<i32> lg(n_lg);
		for (int i = 0; i < n_logn; ++i) logn[i] = i ? log((double)i) : 0.;
		for (int i = 0; i < n_lg; ++i) lg[i] = (int)(4.343 * log((double)(i + 1)) + .499);
		if (a->d_logn.need(n_logn * 8) || a->d_lg.need(n_lg * 4)) { ssq_aligner_free(a); return SSQ_ENOMEM; }
		CK(cudaMemcpy(a->d_logn.p, logn.data(), n_logn * 8, cudaMemcpyHostToDevice));
		CK(cudaMemcpy(a->d_lg.p, lg.data(), n_lg * 4, cudaMemcpyHostToDevice));
	}
	{ // contig names and samblaster's padded coordinate offsets
		const int ns = idx->n_seqs;
		std::vector<char> names; std::vector<u32> off(ns + 1, 0); std::vector<i64> sboff(ns + 1, 0);
		i64 total = 0;
		for (int i = 0; i < ns; ++i) {
			const size_t l = strlen(idx->names[i]);
			names.insert(names.end(), idx->names[i], idx->names[i] + l);
			off[i + 1] = (u32)names.size();
			sboff[i] = total; total += (i64)idx->ann_len[i] + 2 * SB_PAD + 1;
		}
		if (a->d_ctg_names.need(names.size() + 16) || a->d_ctg_off.need((ns + 1) * 4) || a->d_sb_off.need((ns + 1) * 8) || a->d_rg.need(256)) { ssq_aligner_free(a); return SSQ_ENOMEM; }
		CK(cudaMemcpy(a->d_ctg_names.p, names.data(), names.size(), cudaMemcpyHostToDevice));
		CK(cudaMemcpy(a->d_ctg_off.p, off.data(), (ns + 1) * 4, cudaMemcpyHostToDevice));
		CK(cudaMemcpy(a->d_sb_off.p, sboff.data(), (ns + 1) * 8, cudaMemcpyHostToDevice));
		CK(cudaMemcpy(a->d_rg.p, a->rg_id, 256, cudaMemcpyHostToDevice));
	}
	if (a->d_work.need(256) || a->d_err.need(64) || a->d_cnt.need(64) || a->d_pes.need(4 * sizeof(PeStat))) { ssq_aligner_free(a); return SSQ_ENOMEM; }
	*out = a;
	return SSQ_OK;
}

extern "C" int ssq_aligner_reset_dups(ssq_aligner_t *a) { return a ? ssq_dupset_reset(a->dups) : SSQ_EINVAL; }
extern "C" int ssq_aligner_share_dupset(ssq_aligner_t *a, ssq_dupset_t *set)
{
	if (!a || !set) return SSQ_EINVAL;
	if (a->dups && a->own_dups) ssq_dupset_free(a->dups);
	a->dups = set; a->own_dups = 0;
	return SSQ_OK;
}
extern "C" int ssq_aligner_set_comm(ssq_aligner_t *a, ssq_comm_t *comm)
{
	if (!a || !comm) return SSQ_EINVAL;
	if (a->dups && a->own_dups) ssq_dupset_free(a->dups);
	a->comm = comm; a->dups = ssq_comm_dupset(comm); a->own_dups = 0; // the owner-side set also keeps the turn counter of this rank's lanes
	return SSQ_OK;
}
extern "C" int ssq_aligner_set_turn(ssq_aligner_t *a, long long turn) { if (!a) return SSQ_EINVAL; a->turn = turn; return SSQ_OK; }
extern "C" void *ssq_aligner_stream(ssq_aligner_t *a) { return a ? (void*)a->st : 0; }
extern "C" float ssq_aligner_stage_ms(const ssq_aligner_t *a, int stage)
{
	if (!a || stage < 0) return -1.f;
	if (stage < ST_N) return a->stage_ms[stage];
	if (stage < ST_N + 5) return ssq_batch_stage_ms(a->b, stage - ST_N); // 0 smem, 1 sa, 2 chain, 3 extend, 4 select
	return -1.f;
}
extern "C" uint64_t ssq_aligner_counter(const ssq_aligner_t *a, int what)
{
	if (!a) return 0;
	if (what < 100) return ssq_batch_counter(a->b, what);
	switch (what) { case 100: return a->n_tasks_total; case 101: return a->text_len[0]; case 102: return a->text_len[1]; case 103: return a->text_len[2]; case 104: return ssq_dupset_size(a->dups); case 105: return a->n_rescue_pairs; case 106: return a->n_gapped; case 107: return a->n_sw_local; case 108: return a->sw_local_cells; case 109: return a->total_bases; case 110: return (u64)a->n_reads; }
	return 0;
}

// ---- stage 0: host blobs -> HBM ----
extern "C" int ssq_aligner_upload(ssq_aligner_t *a, const ssq_reads_t *rd)
{
	if (!a || !rd || rd->n_reads < 0 || (rd->n_reads && (!rd->seq || !rd->seq_off || !rd->name || !rd->name_off))) return SSQ_EINVAL;
	if (rd->paired && (rd->n_reads & 1)) { ssq_set_error("paired batch with an odd number of reads"); return SSQ_EINVAL; }
	int rc = ssq_use_device(a->device);
	if (rc) return rc;
	const int n = rd->n_reads;
	CK(cudaEventRecord(a->ev[ST_UPLOAD], a->st));
	a->n_reads = n; a->paired = rd->paired ? 1 : 0; a->n_processed = rd->n_processed; a->has_qual = rd->qual != 0; a->has_cmt = rd->comment != 0 && rd->comment_off != 0;
	a->computed = 0;
	const u64 total = n ? rd->seq_off[n] : 0;
	int max_len = 0;
	for (int i = 0; i < n; ++i) {
		const int l = (int)(rd->seq_off[i + 1] - rd->seq_off[i]);
		if (l > max_len) max_len = l;
		if (l > SSQ_MAX_READ_LEN) { // name the read: one long read must not leave the user guessing which of 10^8
			ssq_set_error("read %d ('%.*s') has %d bases; this build aligns reads of at most %d", i, (int)(rd->name_off[i + 1] - rd->name_off[i]), rd->name + rd->name_off[i], l, SSQ_MAX_READ_LEN);
			return SSQ_ELEN;
		}
	}
	a->total_bases = total; a->max_len = max_len;
	uint8_t *d_seq; u64 *d_off;
	if ((rc = ssq_batch_reserve(a->b, n, total, max_len, &d_seq, &d_off))) return rc;
	const size_t name_bytes = n ? rd->name_off[n] : 0, cmt_bytes = a->has_cmt && n ? rd->comment_off[n] : 0;
	if (a->d_ascii.need(total + 16) || a->d_qual.need(total + 16) || a->d_names.need(name_bytes + 16) || a->d_name_off.need((size_t)(n + 1) * 4) ||
	    a->d_cmt.need(cmt_bytes + 16) || a->d_cmt_off.need((size_t)(n + 1) * 4)) return SSQ_ENOMEM;
	if (n) {
		CK(cudaMemcpyAsync(a->d_ascii.p, rd->seq, total, cudaMemcpyHostToDevice, a->st));
		CK(cudaMemcpyAsync(d_off, rd->seq_off, (size_t)(n + 1) * 8, cudaMemcpyHostToDevice, a->st));
		if (a->has_qual) CK(cudaMemcpyAsync(a->d_qual.p, rd->qual, total, cudaMemcpyHostToDevice, a->st));
		CK(cudaMemcpyAsync(a->d_names.p, rd->name, name_bytes, cudaMemcpyHostToDevice, a->st));
		CK(cudaMemcpyAsync(a->d_name_off.p, rd->name_off, (size_t)(n + 1) * 4, cudaMemcpyHostToDevice, a->st));
		if (a->has_cmt) {
			CK(cudaMemcpyAsync(a->d_cmt.p, rd->comment, cmt_bytes, cudaMemcpyHostToDevice, a->st));
			CK(cudaMemcpyAsync(a->d_cmt_off.p, rd->comment_off, (size_t)(n + 1) * 4, cudaMemcpyHostToDevice, a->st));
		}
		if (total) k_encode<<<(unsigned)((total / 4 + 256) / 256), 256, 0, a->st>>>(total, a->d_ascii.as<char>(), d_seq);
		CK(cudaGetLastError());
	}
	CK(cudaEventRecord(a->ev[ST_ALIGN], a->st));
	CK(cudaStreamSynchronize(a->st)); // the caller may reuse its host buffers
	return SSQ_OK;
}

static PipeView make_view(ssq_aligner *a)
{
	PipeView V;
	memset(&V, 0, sizeof V);
	const BatchView bv = ssq_batch_view(a->b);
	V.ix = bv.ix; V.opt = a->opt; V.sb = a->sb;
	V.T.logn = a->d_logn.as<double>(); V.T.n_logn = 8192; V.T.lg4343 = a->d_lg.as<i32>(); V.T.n_lg = 65536;
	V.tc.ctg_names = a->d_ctg_names.as<char>(); V.tc.ctg_name_off = a->d_ctg_off.as<u32>();
	V.tc.names = a->d_names.as<char>(); V.tc.name_off = a->d_name_off.as<u32>();
	V.tc.seq = bv.seq; V.tc.read_off = bv.read_off;
	V.tc.qual = a->has_qual ? a->d_qual.as<char>() : 0;
	V.tc.cmt = a->has_cmt ? a->d_cmt.as<char>() : 0; V.tc.cmt_off = a->has_cmt ? a->d_cmt_off.as<u32>() : 0;
	V.tc.rg_id = a->d_rg.as<char>(); V.tc.rg_len = (i32)strlen(a->rg_id);
	V.n_reads = a->n_reads; V.paired = a->paired; V.n_processed = a->n_processed;
	V.task_off = bv.task_off; V.n_regs = bv.n_regs; V.regs = bv.regs;
	V.sb_off = a->d_sb_off.as<i64>();
	V.err = a->d_err.as<i32>(); V.cnt = (unsigned long long*)a->d_cnt.p;
	return V;
}

// ---- stages 1..8: everything on the device; leaves the text of the three streams in HBM ----
static int compute_impl(ssq_aligner_t *a, const ssq_pestat_t *pes0, int verbose);
extern "C" int ssq_aligner_compute(ssq_aligner_t *a, const ssq_pestat_t *pes0, int verbose)
{
	if (!a) return SSQ_EINVAL;
	const int rc = compute_impl(a, pes0, verbose);
	if (a->turn >= 0) { ssq_dupset_wait_turn(a->dups, a->turn); ssq_dupset_end_turn(a->dups, a->turn); } // whatever happened, later batches must not wait for this one
	return rc;
}
static int compute_impl(ssq_aligner_t *a, const ssq_pestat_t *pes0, int verbose)
{
	int rc = ssq_use_device(a->device);
	if (rc) return rc;
	const int n = a->n_reads, n_pairs = a->paired ? n >> 1 : 0, n_units = a->paired ? n >> 1 : n;
	cudaStream_t st = a->st;
	a->text_len[0] = a->text_len[1] = a->text_len[2] = 0; a->n_tasks_total = 0; a->n_ids = a->n_dup = a->n_disc_lines = a->n_split_lines = 0;
	CK(cudaEventRecord(a->ev[ST_ALIGN], st));
	if (n == 0) {
		if (a->comm && a->sb.enabled) { // an empty batch still takes part in its round of the exchange (the other ranks are waiting in it)
			if (a->turn >= 0) ssq_dupset_wait_turn(a->dups, a->turn);
			rc = ssq_comm_mark_round(a->comm, 0, 0, 0, 0, 0, (void*)st);
			if (a->turn >= 0) ssq_dupset_end_turn(a->dups, a->turn);
			if (rc) return rc;
		}
		for (int i = ST_ALIGN + 1; i <= ST_N; ++i) CK(cudaEventRecord(a->ev[i], st));
		a->computed = 1;
		return SSQ_OK;
	}
	if ((rc = ssq_batch_run(a->b))) return rc;
	CK(cudaEventRecord(a->ev[ST_DEDUP], st));
	PipeView V = make_view(a);
	CK(cudaMemsetAsync(a->d_err.p, 0, 64, st));
	CK(cudaMemsetAsync(a->d_cnt.p, 0, 64, st));
	// region lists
	u64 total_cap = 0;
	if (a->d_cap.need((size_t)(n + 2) * 8) || a->d_aoff.need((size_t)(n + 2) * 8) || a->d_na.need((size_t)(n + 1) * 4)) return SSQ_ENOMEM;
	k_areg_cap<<<(n + 255) / 256, 256, 0, st>>>(n, a->paired, a->opt.max_matesw, V.n_regs, a->d_cap.as<u64>());
	if ((rc = scan_u64(a, a->d_cap.as<u64>(), a->d_aoff.as<u64>(), (size_t)n + 1))) return rc;
	CK(cudaMemcpyAsync(&total_cap, a->d_aoff.as<u64>() + n, 8, cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	if (a->d_areg.need((total_cap + 1) * sizeof(AlnReg)) || a->d_pv.need((total_cap + 2) * sizeof(P64)) || a->d_xcnt.need((total_cap + 2) * 4)) return SSQ_ENOMEM;
	V.areg_off = a->d_aoff.as<u64>(); V.areg = a->d_areg.as<AlnReg>(); V.n_areg = a->d_na.as<u32>();
	V.pv = a->d_pv.as<P64>(); V.xcnt = a->d_xcnt.as<i32>();
	const int dedup_blocks = a->n_sm * 8;
	if (a->d_slab.need((size_t)dedup_blocks * 128 * sizeof(DedupSlab))) return SSQ_ENOMEM;
	int *work = a->d_work.as<int>();
	CK(cudaMemsetAsync(work, 0, 256, st));
	k_dedup<<<dedup_blocks, 128, 0, st>>>(V, a->d_slab.as<DedupSlab>(), work);
	CK(cudaGetLastError());
	CK(cudaEventRecord(a->ev[ST_PESTAT], st));
	// insert-size statistics and the pairing penalty table
	PeStat *pes = a->pes;
	memset(pes, 0, 4 * sizeof(PeStat));
	V.pes = a->d_pes.as<PeStat>();
	if (a->paired) {
		if (pes0) for (int d = 0; d < 4; ++d) { pes[d].low = pes0[d].low; pes[d].high = pes0[d].high; pes[d].failed = pes0[d].failed; pes[d].pad = 0; pes[d].avg = pes0[d].avg; pes[d].std = pes0[d].std; }
		else {
			const int hist_n = a->opt.max_ins + 1;
			if (a->d_hist.need((size_t)4 * hist_n * 4) || a->h_hist.need((size_t)4 * hist_n * 4)) return SSQ_ENOMEM;
			CK(cudaMemsetAsync(a->d_hist.p, 0, (size_t)4 * hist_n * 4, st));
			V.hist = a->d_hist.as<u32>(); V.hist_n = hist_n;
			k_pestat<<<(n_pairs + 255) / 256, 256, 0, st>>>(V);
			CK(cudaMemcpyAsync(a->h_hist.p, a->d_hist.p, (size_t)4 * hist_n * 4, cudaMemcpyDeviceToHost, st));
			CK(cudaStreamSynchronize(st));
			pestat_from_hist(a->opt, (const u32*)a->h_hist.p, hist_n, pes, verbose ? stderr : 0);
		}
		// penalty table over the integer distances each orientation admits
		std::vector<double> pen; int pn[4]; size_t pat[4];
		const size_t tot = pen_table(a->opt, pes, pen, pn, pat);
		if (a->d_pen.need((tot + 1) * 8)) return SSQ_ENOMEM;
		for (int d = 0; d < 4; ++d) { V.T.pen[d] = a->d_pen.as<double>() + pat[d]; V.T.pen_low[d] = pes[d].low; V.T.pen_n[d] = pn[d]; }
		if (tot) CK(cudaMemcpyAsync(a->d_pen.p, pen.data(), tot * 8, cudaMemcpyHostToDevice, st));
		CK(cudaMemcpyAsync(a->d_pes.p, pes, 4 * sizeof(PeStat), cudaMemcpyHostToDevice, st));
		CK(cudaStreamSynchronize(st)); // pen is a host temporary
	}
	CK(cudaEventRecord(a->ev[ST_RESCUE], st));
	if (a->paired) { // mate rescue
		int win = 0;
		for (int d = 0; d < 4; ++d) if (!pes[d].failed && pes[d].high - pes[d].low > win) win = pes[d].high - pes[d].low;
		RescueCfg cfg;
		cfg.win_cap = win + a->max_len + 16;
		if (cfg.win_cap > (1 << 20)) { ssq_set_error("insert-size bounds admit rescue windows of %d bases (limit 2^20)", cfg.win_cap); return SSQ_EINVAL; }
		cfg.slab_bytes = ((size_t)128 * sizeof(AlnReg) + (size_t)cfg.win_cap * 8 + 15) & ~(size_t)15;
		const int blocks = a->n_sm * 8; // 4 warps per block, 32 warps per SM
		if (a->d_rlist.need((size_t)(n_pairs + 1) * 4) || a->d_slab.need((size_t)blocks * 4 * cfg.slab_bytes)) return SSQ_ENOMEM;
		unsigned int *n_list = (unsigned int*)(work + 16);
		if (a->rescue_spec) { // every alignment the initial lists do not skip, computed ahead as evenly sized tasks; then the replay looks them up
			unsigned int *n_tasks = (unsigned int*)(work + 18), *n_miss = (unsigned int*)(work + 19), h_n[4] = {0, 0, 0, 0};
			if (a->d_rtbase.need((size_t)(n_pairs + 1) * 4) || a->d_rtcnt.need((size_t)(n_pairs + 1) * 4)) return SSQ_ENOMEM;
			k_rescue_count<<<(n_pairs + 255) / 256, 256, 0, st>>>(V, cfg.win_cap, a->d_rlist.as<u32>(), a->d_rtbase.as<u32>(), a->d_rtcnt.as<u32>(), n_list, n_tasks);
			CK(cudaMemcpyAsync(h_n, work + 16, 16, cudaMemcpyDeviceToHost, st));
			CK(cudaStreamSynchronize(st));
			const unsigned int nl = h_n[0], nt = h_n[2];
			if (nl) {
				if (a->d_rtasks.need(((size_t)nt + 1) * sizeof(RTask)) || a->d_rres.need(((size_t)nt + 1) * sizeof(LocalRes))) return SSQ_ENOMEM;
				k_rescue_fill<<<(nl + 255) / 256, 256, 0, st>>>(V, cfg.win_cap, a->d_rlist.as<u32>(), a->d_rtbase.as<u32>(), n_list, a->d_rtasks.as<RTask>());
				k_rescue_sw<<<blocks, 128, 0, st>>>(V, a->d_rlist.as<u32>(), a->d_rtasks.as<RTask>(), n_tasks, a->d_rres.as<LocalRes>(), a->d_slab.as<uint8_t>(), cfg, work + 3);
				k_rescue<<<blocks, 128, 0, st>>>(V, a->d_rlist.as<u32>(), n_list, a->d_slab.as<uint8_t>(), cfg, work + 1, a->d_rtasks.as<RTask>(), a->d_rres.as<LocalRes>(), a->d_rtbase.as<u32>(), a->d_rtcnt.as<u32>(), n_miss);
			}
		} else {
			k_rescue_mark<<<(n_pairs + 255) / 256, 256, 0, st>>>(V, a->d_rlist.as<u32>(), n_list);
			k_rescue<<<blocks, 128, 0, st>>>(V, a->d_rlist.as<u32>(), n_list, a->d_slab.as<uint8_t>(), cfg, work + 1, 0, 0, 0, 0, 0);
		}
		CK(cudaGetLastError());
	}
	CK(cudaEventRecord(a->ev[ST_PLAN], st));
	// planning: task slots, plan, compaction
	u64 total_slots = 0, total_tasks = 0;
	if (a->d_tcap.need((size_t)(n + 2) * 8) || a->d_tsoff.need((size_t)(n + 2) * 8) || a->d_meta.need((size_t)(n + 1) * sizeof(ReadMeta)) || a->d_ntk.need((size_t)(n + 2) * 8) || a->d_tkbase.need((size_t)(n + 2) * 8)) return SSQ_ENOMEM;
	k_tslot_cap<<<(n + 255) / 256, 256, 0, st>>>(n, V.n_areg, a->d_tcap.as<u64>());
	if ((rc = scan_u64(a, a->d_tcap.as<u64>(), a->d_tsoff.as<u64>(), (size_t)n + 1))) return rc;
	CK(cudaMemcpyAsync(&total_slots, a->d_tsoff.as<u64>() + n, 8, cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	if (a->d_tslots.need((total_slots + 1) * sizeof(PTask))) return SSQ_ENOMEM;
	V.tslot_off = a->d_tsoff.as<u64>(); V.tslots = a->d_tslots.as<PTask>(); V.meta = a->d_meta.as<ReadMeta>();
	k_plan<<<(n_units + 127) / 128, 128, 0, st>>>(V);
	k_ntasks<<<(n + 255) / 256, 256, 0, st>>>(n, V.meta, a->d_ntk.as<u64>());
	if ((rc = scan_u64(a, a->d_ntk.as<u64>(), a->d_tkbase.as<u64>(), (size_t)n + 1))) return rc;
	CK(cudaMemcpyAsync(&total_tasks, a->d_tkbase.as<u64>() + n, 8, cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	a->n_tasks_total = total_tasks;
	if (total_tasks >= 0xffffffffull) { ssq_set_error("more than 2^32-1 alignments to write in one batch"); return SSQ_EINVAL; }
	if (a->d_tasks.need((total_tasks + 1) * sizeof(PTask)) || a->d_outs.need((total_tasks + 1) * sizeof(AlnOut)) || a->d_cigs.need((total_tasks + 1) * CIG_CAP * 4) || a->d_mds.need((total_tasks + 1) * MD_CAP) ||
	    a->d_redo.need((total_tasks + 1) * 4)) return SSQ_ENOMEM;
	V.tk_base = a->d_tkbase.as<u64>(); V.tasks = a->d_tasks.as<PTask>(); V.outs = a->d_outs.as<AlnOut>(); V.cigs = a->d_cigs.as<u32>(); V.mds = a->d_mds.as<char>();
	k_compact<<<(n + 255) / 256, 256, 0, st>>>(V);
	CK(cudaGetLastError());
	CK(cudaEventRecord(a->ev[ST_CIGAR], st));
	if (total_tasks) { // CIGARs: the ones without dynamic programming per thread, the others per warp
		const long zcap = (long)QMAX * 768;
		const int blocks = a->n_sm * 6; // 4 warps per block, 24 warps per SM (22 KB of shared memory per block)
		if (a->d_slab.need((size_t)blocks * 4 * (size_t)zcap)) return SSQ_ENOMEM;
		unsigned int *n_gapped = (unsigned int*)(work + 17);
		k_cigar_fast<<<(unsigned)((total_tasks + 127) / 128), 128, 0, st>>>(V, total_tasks, a->d_redo.as<u32>(), n_gapped);
		k_cigar_warp<<<blocks, 128, 0, st>>>(V, a->d_redo.as<u32>(), n_gapped, a->d_slab.as<uint8_t>(), zcap, work + 2);
		CK(cudaGetLastError());
	}
	CK(cudaEventRecord(a->ev[ST_SB], st));
	if (a->d_k1.need((size_t)(n_units + 1) * 8) || a->d_k2.need((size_t)(n_units + 1) * 8) || a->d_valid.need(n_units + 16) || a->d_dup.need(n_units + 16) || a->d_disc.need(n_units + 16) || a->d_smask.need((size_t)(n + 1) * 8)) return SSQ_ENOMEM;
	V.k1 = a->d_k1.as<u64>(); V.k2 = a->d_k2.as<u64>(); V.valid = a->d_valid.as<uint8_t>(); V.dup = a->d_dup.as<uint8_t>(); V.disc = a->d_disc.as<uint8_t>(); V.split_mask = a->d_smask.as<u64>();
	if (a->sb.enabled) {
		k_sb<<<(n_units + 127) / 128, 128, 0, st>>>(V);
		CK(cudaGetLastError());
		if (a->turn >= 0) ssq_dupset_wait_turn(a->dups, a->turn);
		rc = a->comm ? ssq_comm_mark_round(a->comm, (u64)n_units, V.k1, V.k2, V.valid, V.dup, (void*)st) : ssq_dupset_mark_dev(a->dups, (u64)n_units, V.k1, V.k2, V.valid, V.dup, (void*)st);
		if (a->turn >= 0) { cudaStreamSynchronize(st); ssq_dupset_end_turn(a->dups, a->turn); } // the set must be complete before the next batch looks it up from another stream
		if (rc) return rc;
		k_count_u8<<<(n_units + 255) / 256, 256, 0, st>>>((u64)n_units, V.dup, 0, (unsigned long long*)a->d_cnt.p);
	}
	CK(cudaEventRecord(a->ev[ST_TEXT], st));
	// text: sizes, offsets, bytes
	for (int k = 0; k < 3; ++k) { if (a->d_len[k].need((size_t)(n + 2) * 8) || a->d_off[k].need((size_t)(n + 2) * 8)) return SSQ_ENOMEM; V.len[k] = a->d_len[k].as<u64>(); V.off[k] = a->d_off[k].as<u64>(); }
	k_text<false><<<(n + 127) / 128, 128, 0, st>>>(V);
	CK(cudaGetLastError());
	const int n_streams = a->sb.enabled ? 3 : 1;
	for (int k = 0; k < n_streams; ++k) {
		if ((rc = scan_u64(a, a->d_len[k].as<u64>(), a->d_off[k].as<u64>(), (size_t)n + 1))) return rc;
		CK(cudaMemcpyAsync(&a->text_len[k], a->d_off[k].as<u64>() + n, 8, cudaMemcpyDeviceToHost, st));
	}
	int h_err = 0; unsigned long long h_cnt[8] = {0, 0, 0, 0, 0, 0, 0, 0}; unsigned int h_work[2] = {0, 0};
	CK(cudaMemcpyAsync(h_work, work + 16, 8, cudaMemcpyDeviceToHost, st)); // pairs that went through mate rescue, alignments that needed the banded DP
	CK(cudaMemcpyAsync(&h_err, a->d_err.p, 4, cudaMemcpyDeviceToHost, st));
	CK(cudaMemcpyAsync(h_cnt, a->d_cnt.p, 64, cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	if (h_err) {
		ssq_set_error("batch capacity error (flags 0x%x):%s%s%s%s%s", h_err, h_err & 1 ? " mate rescue overflowed a region list;" : "", h_err & 2 ? " more alignments to write than task slots;" : "",
		              h_err & 4 ? " an alignment with too many CIGAR operations / MD characters or a traceback matrix beyond the per-thread capacity;" : "", h_err & 8 ? " a rescue window beyond the scratch sized from the insert-size bounds;" : "", h_err & ~15 ? " internal;" : "");
		return SSQ_ECAP;
	}
	for (int k = 0; k < 3; ++k) { if (a->d_text[k].need(a->text_len[k] + 64)) return SSQ_ENOMEM; V.text[k] = a->d_text[k].as<char>(); }
	k_text<true><<<(n + 127) / 128, 128, 0, st>>>(V);
	CK(cudaGetLastError());
	if (a->want_bam) { // the same records as BAM, sorted by (reference, position, strand) within the batch (stable: equal keys keep input order)
		u64 L = 0;
		if (a->d_nl.need((size_t)(n + 2) * 8) || a->d_lbase.need((size_t)(n + 2) * 8)) return SSQ_ENOMEM;
		k_nlines<<<(n + 255) / 256, 256, 0, st>>>(n, V, a->d_nl.as<u64>());
		if ((rc = scan_u64(a, a->d_nl.as<u64>(), a->d_lbase.as<u64>(), (size_t)n + 1))) return rc;
		CK(cudaMemcpyAsync(&L, a->d_lbase.as<u64>() + n, 8, cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		a->n_lines_total = L;
		if (L >= 0x7fffffffull) { ssq_set_error("more than 2^31-1 records in one batch"); return SSQ_EINVAL; }
		if (a->d_lread.need((L + 1) * 4) || a->d_bkey.need((L + 1) * 8) || a->d_bkey2.need((L + 1) * 8) || a->d_bidx.need((L + 1) * 4) || a->d_bperm.need((L + 1) * 4) || a->d_bsz_s.need((L + 2) * 8)) return SSQ_ENOMEM;
		for (int k = 0; k < 3; ++k) { if (a->d_bsize[k].need((L + 1) * 8) || a->d_boff[k].need((L + 2) * 8)) return SSQ_ENOMEM; V.bam_size[k] = a->d_bsize[k].as<u64>(); }
		V.line_base = a->d_lbase.as<u64>(); V.line_read = a->d_lread.as<u32>(); V.bam_key = a->d_bkey.as<u64>(); V.bam_blank_side = a->bam_blank_side;
		k_bam_size<<<(n + 127) / 128, 128, 0, st>>>(V);
		const unsigned gl = (unsigned)((L + 255) / 256);
		k_iota_u32<<<gl, 256, 0, st>>>(L, a->d_bidx.as<u32>());
		size_t tb = 0;
		cub::DeviceRadixSort::SortPairs(0, tb, a->d_bkey.as<u64>(), a->d_bkey2.as<u64>(), a->d_bidx.as<u32>(), a->d_bperm.as<u32>(), (int)L, 0, 64, st);
		if (a->cubtmp.need(tb)) return SSQ_ENOMEM;
		CK(cub::DeviceRadixSort::SortPairs(a->cubtmp.p, tb, a->d_bkey.as<u64>(), a->d_bkey2.as<u64>(), a->d_bidx.as<u32>(), a->d_bperm.as<u32>(), (int)L, 0, 64, st));
		V.bam_perm = a->d_bperm.as<u32>();
		for (int k = 0; k < n_streams; ++k) {
			k_gather_u64<<<gl, 256, 0, st>>>(L, a->d_bperm.as<u32>(), a->d_bsize[k].as<u64>(), a->d_bsz_s.as<u64>());
			if ((rc = scan_u64(a, a->d_bsz_s.as<u64>(), a->d_boff[k].as<u64>(), (size_t)L + 1))) return rc;
			CK(cudaMemcpyAsync(&a->bam_len[k], a->d_boff[k].as<u64>() + L, 8, cudaMemcpyDeviceToHost, st));
			V.bam_off[k] = a->d_boff[k].as<u64>();
		}
		for (int k = n_streams; k < 3; ++k) { a->bam_len[k] = 0; V.bam_off[k] = a->d_boff[0].as<u64>(); }
		CK(cudaStreamSynchronize(st));
		for (int k = 0; k < 3; ++k) { if (a->d_bam[k].need(a->bam_len[k] + 64)) return SSQ_ENOMEM; V.bam[k] = a->d_bam[k].as<char>(); }
		k_bam_write<<<(unsigned)((L + 127) / 128), 128, 0, st>>>(V, L);
		CK(cudaGetLastError());
		int h_err2 = 0;
		CK(cudaMemcpyAsync(&h_err2, a->d_err.p, 4, cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		if (h_err2 & 32) { ssq_set_error("a FASTQ comment (-C) is not TAG:TYPE:VALUE with TYPE in {Z, i, A}: it cannot become BAM tags"); return SSQ_EINVAL; }
	}
	CK(cudaEventRecord(a->ev[ST_FETCH], st));
	a->n_ids = (u64)n_units; a->n_dup = h_cnt[0]; a->n_rescue_pairs = h_work[0]; a->n_gapped = h_work[1]; a->n_sw_local = h_cnt[2]; a->sw_local_cells = h_cnt[3];
	a->computed = 1;
	return SSQ_OK;
}

// ---- stage 9: the three streams back to (pinned) host memory ----
extern "C" int ssq_aligner_fetch(ssq_aligner_t *a, ssq_sam_t *out)
{
	if (!a || !out || !a->computed) return SSQ_EINVAL;
	int rc = ssq_use_device(a->device);
	if (rc) return rc;
	const int n = a->n_reads;
	memset(out, 0, sizeof *out);
	for (int k = 0; k < 3; ++k) {
		if (a->h_text[k].need(a->text_len[k] + 1)) return SSQ_ENOMEM;
		if (a->text_len[k]) CK(cudaMemcpyAsync(a->h_text[k].p, a->d_text[k].p, a->text_len[k], cudaMemcpyDeviceToHost, a->st));
	}
	if (a->h_roff.need((size_t)(n + 1) * 8)) return SSQ_ENOMEM;
	if (n) CK(cudaMemcpyAsync(a->h_roff.p, a->d_off[0].p, (size_t)(n + 1) * 8, cudaMemcpyDeviceToHost, a->st));
	else *(u64*)a->h_roff.p = 0;
	CK(cudaEventRecord(a->ev[ST_N], a->st));
	CK(cudaStreamSynchronize(a->st));
	for (int i = 0; i < ST_N; ++i) { float ms = 0.f; if (cudaEventElapsedTime(&ms, a->ev[i], a->ev[i + 1]) != cudaSuccess) { cudaGetLastError(); ms = 0.f; } a->stage_ms[i] = ms; }
	for (int k = 0; k < 3; ++k) { ((char*)a->h_text[k].p)[a->text_len[k]] = 0; out->text[k] = (const char*)a->h_text[k].p; out->len[k] = a->text_len[k]; }
	out->read_off = (const uint64_t*)a->h_roff.p;
	out->n_ids = a->n_ids; out->n_dup = a->n_dup;
	for (int d = 0; d < 4; ++d) { out->pes[d].low = a->pes[d].low; out->pes[d].high = a->pes[d].high; out->pes[d].failed = a->pes[d].failed; out->pes[d].pad = 0; out->pes[d].avg = a->pes[d].avg; out->pes[d].std = a->pes[d].std; }
	return SSQ_OK;
}

// one stream's text alone (a caller that takes the main records as BAM still wants the two side streams as text)
extern "C" int ssq_aligner_fetch_text(ssq_aligner_t *a, int stream, const char **text, size_t *len)
{
	if (!a || !text || !len || stream < 0 || stream > 2 || !a->computed) return SSQ_EINVAL;
	int rc = ssq_use_device(a->device);
	if (rc) return rc;
	if (a->h_text[stream].need(a->text_len[stream] + 1)) return SSQ_ENOMEM;
	if (a->text_len[stream]) CK(cudaMemcpyAsync(a->h_text[stream].p, a->d_text[stream].p, a->text_len[stream], cudaMemcpyDeviceToHost, a->st));
	CK(cudaStreamSynchronize(a->st));
	((char*)a->h_text[stream].p)[a->text_len[stream]] = 0;
	*text = (const char*)a->h_text[stream].p; *len = a->text_len[stream];
	return SSQ_OK;
}

extern "C" int ssq_aligner_run(ssq_aligner_t *a, const ssq_reads_t *reads, const ssq_pestat_t *pes0, int verbose, ssq_sam_t *out)
{
	int rc;
	if ((rc = ssq_aligner_upload(a, reads))) return rc;
	if ((rc = ssq_aligner_compute(a, pes0, verbose))) return rc;
	return ssq_aligner_fetch(a, out);
}

extern "C" int ssq_sw_local_batch(const ssq_opts_t *opt, int device, uint64_t n, const ssq_swl_task_t *tasks, const uint8_t *qbuf, uint64_t qbuf_len, const uint8_t *tbuf, uint64_t tbuf_len,
                                  ssq_swl_result_t *out)
{
	if (!opt || (n && (!tasks || !qbuf || !tbuf || !out))) return SSQ_EINVAL;
	int rc = ssq_use_device(device);
	if (rc) return rc;
	if (n == 0) return SSQ_OK;
	int b_cap = 1;
	for (u64 i = 0; i < n; ++i) {
		if (tasks[i].qlen < 0 || tasks[i].qlen > SSQ_MAX_READ_LEN || tasks[i].tlen < 0 || tasks[i].q_off + tasks[i].qlen > qbuf_len || tasks[i].t_off + tasks[i].tlen > tbuf_len) { ssq_set_error("ssq_sw_local_batch: task %llu out of range", (unsigned long long)i); return SSQ_EINVAL; }
		if (tasks[i].tlen > b_cap) b_cap = tasks[i].tlen;
	}
	DBuf dt, dq, dtb, dout, dbl;
	if (dt.need(n * sizeof(ssq_swl_task_t)) || dq.need(qbuf_len + 16) || dtb.need(tbuf_len + 16) || dout.need(n * sizeof(ssq_swl_result_t)) || dbl.need(n * (size_t)b_cap * 8)) return SSQ_ENOMEM;
	CK(cudaMemcpy(dt.p, tasks, n * sizeof(ssq_swl_task_t), cudaMemcpyHostToDevice));
	CK(cudaMemcpy(dq.p, qbuf, qbuf_len, cudaMemcpyHostToDevice));
	CK(cudaMemcpy(dtb.p, tbuf, tbuf_len, cudaMemcpyHostToDevice));
	k_sw_local_tasks<<<(unsigned)((n + 3) / 4), 128>>>(*opt, n, dt.as<ssq_swl_task_t>(), dq.as<uint8_t>(), dtb.as<uint8_t>(), dout.as<ssq_swl_result_t>(), dbl.as<u64>(), b_cap);
	CK(cudaGetLastError());
	CK(cudaMemcpy(out, dout.p, n * sizeof(ssq_swl_result_t), cudaMemcpyDeviceToHost));
	return SSQ_OK;
}


// ============================================================== FASTQ ingest on the device ====
// Upstream bseq_read() -> kseq_read() (`$BWA mem`, speedseq/bin/speedseq:438,468); tokenisation rules of the reference's
// in-tree parser speedseq/src/samtools-1.3.1/htslib-1.3.1/htslib/kseq.h:189-231, restricted to the layout sequencers
// write: four lines per record ('@name[ comment]', bases, '+...', qualities).  Anything else (multi-line records, FASTA, blank
// lines, unequal files) is REPORTED (SSQ_EFORMAT) and left to the caller's host tokeniser, which handles every legal input.
//   k_fq_records   thread per record: field extents from the newline positions, checks, name without /1 /2, comment, lengths
//   scans          cumulative bases (the batch rule: bases >= chunk and an even number of reads), offsets of the packed fields
//   k_fq_cut       first record index at which bwa would close the batch
//   k_fq_gather    thread per read: copies name / bases / qualities / comment into the aligner's concatenated batch buffers
struct FqRec { u32 name_b, name_l, cmt_b, cmt_l, seq_b, seq_l, qual_b, bad; };
struct NlPred { const char *t; __device__ bool operator()(const u32 &i) const { return t[i] == '\n'; } };

__global__ void __launch_bounds__(256) k_fq_records(const char *__restrict__ txt, const u32 *__restrict__ nl, u32 n_lines, u32 txt_len, u32 n_rec, FqRec *rec, int *bad)
{
	const u32 r = blockIdx.x * blockDim.x + threadIdx.x;
	if (r >= n_rec) return;
	u32 b[4], e[4];
#pragma unroll
	for (int k = 0; k < 4; ++k) {
		const u32 li = 4 * r + k;
		b[k] = li ? nl[li - 1] + 1 : 0;
		e[k] = li < n_lines ? nl[li] : txt_len; // a final line without '\n'
		if (e[k] > b[k] && txt[e[k] - 1] == '\r') --e[k];
	}
	FqRec o; o.bad = 0;
	if (e[0] == b[0] || txt[b[0]] != '@' || e[2] == b[2] || txt[b[2]] != '+' || e[1] - b[1] != e[3] - b[3] || e[1] - b[1] > SSQ_MAX_READ_LEN) o.bad = 1;
	u32 p = b[0] + 1;
	while (p < e[0] && !(txt[p] == ' ' || (txt[p] >= 9 && txt[p] <= 13))) ++p; // isspace
	o.name_b = b[0] + 1; o.name_l = p - (b[0] + 1);
	o.cmt_b = p < e[0] ? p + 1 : e[0]; o.cmt_l = e[0] - o.cmt_b;
	if (o.name_l > 2 && txt[o.name_b + o.name_l - 2] == '/' && txt[o.name_b + o.name_l - 1] >= '0' && txt[o.name_b + o.name_l - 1] <= '9') o.name_l -= 2;
	if (o.name_l == 0) o.bad = 1;
	o.seq_b = b[1]; o.seq_l = e[1] - b[1]; o.qual_b = b[3];
	for (u32 q = b[1]; q < e[1]; ++q) if (txt[q] == ' ' || txt[q] == '\t') o.bad = 1; // kseq would stop the sequence at white space
	rec[r] = o;
	if (o.bad) atomicExch(bad, 1);
}
// bases per unit (two files: record i of both; one file: record i)
__global__ void k_fq_unit_len(u32 n, const FqRec *__restrict__ r1, const FqRec *__restrict__ r2, u64 *len)
{
	const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) len[i] = (u64)r1[i].seq_l + (r2 ? r2[i].seq_l : 0);
}
// cum = exclusive scan of len.  res[0] = first unit index closing the batch (two files: cum(i+1) >= chunk; one file: additionally i odd), else n
__global__ void k_fq_cut(u32 n, const u64 *__restrict__ cum, const u64 *__restrict__ len, u64 chunk, int one_file, unsigned int *res)
{
	const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	if (cum[i] + len[i] >= chunk && (!one_file || (i & 1))) atomicMin(res, i);
}
__global__ void k_fq_pairnames(u32 n_pairs, const char *__restrict__ t1, const FqRec *__restrict__ r1, const char *__restrict__ t2, const FqRec *__restrict__ r2, int stride, int *bad)
{
	const u32 p = blockIdx.x * blockDim.x + threadIdx.x;
	if (p >= n_pairs) return;
	const FqRec a = r1[stride == 2 ? 2 * p : p], b = stride == 2 ? r1[2 * p + 1] : r2[p];
	const char *ta = t1, *tb = stride == 2 ? t1 : t2;
	bool same = a.name_l == b.name_l;
	for (u32 k = 0; same && k < a.name_l; ++k) same = ta[a.name_b + k] == tb[b.name_b + k];
	if (!same) atomicExch(bad, 2);
}
// field lengths of read i of the batch (read i = record i of file 1, or records i/2 of files 1/2 alternately)
__global__ void k_fq_read_lens(u32 n_reads, const FqRec *__restrict__ r1, const FqRec *__restrict__ r2, int keep_comment, u64 *slen, u64 *nlen, u64 *clen, unsigned int *max_len)
{
	const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n_reads) return;
	const FqRec r = r2 ? ((i & 1) ? r2[i >> 1] : r1[i >> 1]) : r1[i];
	slen[i] = r.seq_l; nlen[i] = r.name_l; clen[i] = keep_comment ? r.cmt_l : 0;
	atomicMax(max_len, r.seq_l);
}
__global__ void __launch_bounds__(128) k_fq_gather(u32 n_reads, const char *__restrict__ t1, const FqRec *__restrict__ r1, const char *__restrict__ t2, const FqRec *__restrict__ r2, int keep_comment,
                                                   const u64 *__restrict__ soff, const u64 *__restrict__ noff64, const u64 *__restrict__ coff64, char *seq, char *qual, char *names, char *cmt,
                                                   u64 *read_off, u32 *name_off, u32 *cmt_off)
{
	const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i > n_reads) return;
	read_off[i] = soff[i]; name_off[i] = (u32)noff64[i]; cmt_off[i] = (u32)coff64[i];
	if (i == n_reads) return;
	const bool second = r2 && (i & 1);
	const FqRec r = r2 ? (second ? r2[i >> 1] : r1[i >> 1]) : r1[i];
	const char *t = second ? t2 : t1;
	for (u32 k = 0; k < r.seq_l; ++k) { seq[soff[i] + k] = t[r.seq_b + k]; qual[soff[i] + k] = t[r.qual_b + k]; }
	for (u32 k = 0; k < r.name_l; ++k) names[noff64[i] + k] = t[r.name_b + k];
	if (keep_comment) for (u32 k = 0; k < r.cmt_l; ++k) cmt[coff64[i] + k] = t[r.cmt_b + k];
}

extern "C" void *ssq_host_alloc(size_t bytes) { void *p = 0; return cudaMallocHost(&p, bytes) == cudaSuccess ? p : 0; }
extern "C" void ssq_host_free(void *p) { if (p) cudaFreeHost(p); }

extern "C" int ssq_aligner_upload_fastq(ssq_aligner_t *a, const char *fq1, size_t len1, int final1, const char *fq2, size_t len2, int final2, int interleaved, int keep_comment,
                                        int64_t chunk_bases, int64_t n_processed, size_t *used1, size_t *used2, int *n_reads_out, int *need_more)
{
	if (!a || !fq1 || !used1 || !n_reads_out || !need_more || (fq2 && !used2) || chunk_bases <= 0) return SSQ_EINVAL;
	if (len1 >= 0xfffffff0ull || len2 >= 0xfffffff0ull) { ssq_set_error("ssq_aligner_upload_fastq: at most 4 GB of text per call"); return SSQ_EINVAL; }
	int rc = ssq_use_device(a->device);
	if (rc) return rc;
	cudaStream_t st = a->st;
	*used1 = 0; if (used2) *used2 = 0; *n_reads_out = 0; *need_more = 0;
	a->computed = 0;
	CK(cudaEventRecord(a->ev[ST_UPLOAD], st));
	const int nf = fq2 ? 2 : 1;
	const char *src[2] = {fq1, fq2}; const size_t len[2] = {len1, len2}; const int fin[2] = {final1, final2};
	u32 n_lines[2] = {0, 0}, n_rec[2] = {0, 0};
	if (a->fq_res.need(256)) return SSQ_ENOMEM;
	CK(cudaMemsetAsync(a->fq_res.p, 0, 256, st));
	int *d_bad = a->fq_res.as<int>(); unsigned int *d_cut = (unsigned int*)a->fq_res.p + 1, *d_maxlen = (unsigned int*)a->fq_res.p + 2; u64 *d_cnt = (u64*)a->fq_res.p + 2;
	for (int f = 0; f < nf; ++f) { // text to the device, newline positions, records
		if (a->fq_txt[f].need(len[f] + 16) || a->fq_nl[f].need((len[f] / 2 + 16) * 4)) return SSQ_ENOMEM; // a record line is at least 1 byte + '\n'
		if (len[f]) CK(cudaMemcpyAsync(a->fq_txt[f].p, src[f], len[f], cudaMemcpyHostToDevice, st));
		if (len[f]) {
			size_t tb = 0;
			cub::CountingInputIterator<u32> it(0);
			NlPred pr; pr.t = a->fq_txt[f].as<char>();
			cub::DeviceSelect::If(0, tb, it, a->fq_nl[f].as<u32>(), d_cnt, (int)len[f], pr, st);
			if (a->cubtmp.need(tb)) return SSQ_ENOMEM;
			CK(cub::DeviceSelect::If(a->cubtmp.p, tb, it, a->fq_nl[f].as<u32>(), d_cnt, (int)len[f], pr, st));
			u64 h = 0;
			CK(cudaMemcpyAsync(&h, d_cnt, 8, cudaMemcpyDeviceToHost, st));
			CK(cudaStreamSynchronize(st));
			n_lines[f] = (u32)h;
		}
		u32 total_lines = n_lines[f];
		if (fin[f] && len[f] && src[f][len[f] - 1] != '\n') ++total_lines; // the last line has no newline
		n_rec[f] = total_lines / 4;
		if (fin[f] && (total_lines & 3)) { ssq_set_error("FASTQ text does not end on a record boundary"); return SSQ_EFORMAT; }
		if (a->fq_rec[f].need(((size_t)n_rec[f] + 1) * sizeof(FqRec))) return SSQ_ENOMEM;
		if (n_rec[f]) k_fq_records<<<(n_rec[f] + 255) / 256, 256, 0, st>>>(a->fq_txt[f].as<char>(), a->fq_nl[f].as<u32>(), n_lines[f], (u32)len[f], n_rec[f], a->fq_rec[f].as<FqRec>(), d_bad);
	}
	if (nf == 2 && final1 && final2 && n_rec[0] != n_rec[1]) { ssq_set_error("the two FASTQ files hold different numbers of records"); return SSQ_EFORMAT; }
	const u32 n_units = nf == 2 ? (n_rec[0] < n_rec[1] ? n_rec[0] : n_rec[1]) : n_rec[0];
	const bool all_final = final1 && (nf == 1 || final2);
	if (n_units == 0) { if (!all_final) *need_more = 1; a->n_reads = 0; return SSQ_OK; }
	// the batch rule
	const FqRec *r1 = a->fq_rec[0].as<FqRec>(), *r2 = nf == 2 ? a->fq_rec[1].as<FqRec>() : 0;
	if (a->fq_len.need(((size_t)n_units + 2) * 8) || a->fq_cum.need(((size_t)n_units + 2) * 8)) return SSQ_ENOMEM;
	k_fq_unit_len<<<(n_units + 255) / 256, 256, 0, st>>>(n_units, r1, r2, a->fq_len.as<u64>());
	if ((rc = scan_u64(a, a->fq_len.as<u64>(), a->fq_cum.as<u64>(), (size_t)n_units + 1))) return rc;
	const unsigned int none = 0xffffffffu;
	CK(cudaMemcpyAsync(d_cut, &none, 4, cudaMemcpyHostToDevice, st));
	k_fq_cut<<<(n_units + 255) / 256, 256, 0, st>>>(n_units, a->fq_cum.as<u64>(), a->fq_len.as<u64>(), (u64)chunk_bases, nf == 1, d_cut);
	unsigned int h_res[2] = {0, 0};
	CK(cudaMemcpyAsync(h_res, a->fq_res.p, 8, cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	if (h_res[0] == 1) { ssq_set_error("not plain four-line FASTQ (or a read longer than %d bases)", SSQ_MAX_READ_LEN); return SSQ_EFORMAT; }
	u32 take; // units in this batch
	if (h_res[1] != none) take = h_res[1] + 1;
	else if (all_final) take = n_units;
	else { *need_more = 1; a->n_reads = 0; return SSQ_OK; }
	const u32 n_reads = nf == 2 ? 2 * take : take;
	const int paired = nf == 2 || interleaved;
	if (paired && (n_reads & 1)) { ssq_set_error("interleaved FASTQ with an odd number of records"); return SSQ_EFORMAT; }
	if (paired) { // mates must carry the same name (bwa: smart pairing / "paired reads have different names"): anything else goes to the host path
		k_fq_pairnames<<<(n_reads / 2 + 255) / 256, 256, 0, st>>>(n_reads / 2, a->fq_txt[0].as<char>(), r1, nf == 2 ? a->fq_txt[1].as<char>() : 0, r2, nf == 2 ? 1 : 2, d_bad);
	}
	// packed fields
	if (a->fq_nlen.need(((size_t)n_reads + 2) * 8) || a->fq_clen.need(((size_t)n_reads + 2) * 8) || a->fq_noff.need(((size_t)n_reads + 2) * 8) || a->fq_coff.need(((size_t)n_reads + 2) * 8)) return SSQ_ENOMEM;
	u64 *slen = a->fq_len.as<u64>(), *soff = a->fq_cum.as<u64>(); // reused: per-read now
	if (a->fq_len.need(((size_t)n_reads + 2) * 8) || a->fq_cum.need(((size_t)n_reads + 2) * 8)) return SSQ_ENOMEM;
	slen = a->fq_len.as<u64>(); soff = a->fq_cum.as<u64>();
	k_fq_read_lens<<<(n_reads + 255) / 256, 256, 0, st>>>(n_reads, r1, r2, keep_comment, slen, a->fq_nlen.as<u64>(), a->fq_clen.as<u64>(), d_maxlen);
	if ((rc = scan_u64(a, slen, soff, (size_t)n_reads + 1))) return rc;
	if ((rc = scan_u64(a, a->fq_nlen.as<u64>(), a->fq_noff.as<u64>(), (size_t)n_reads + 1))) return rc;
	if ((rc = scan_u64(a, a->fq_clen.as<u64>(), a->fq_coff.as<u64>(), (size_t)n_reads + 1))) return rc;
	u64 tot[3] = {0, 0, 0}; unsigned int h2[3] = {0, 0, 0};
	CK(cudaMemcpyAsync(&tot[0], soff + n_reads, 8, cudaMemcpyDeviceToHost, st));
	CK(cudaMemcpyAsync(&tot[1], a->fq_noff.as<u64>() + n_reads, 8, cudaMemcpyDeviceToHost, st));
	CK(cudaMemcpyAsync(&tot[2], a->fq_coff.as<u64>() + n_reads, 8, cudaMemcpyDeviceToHost, st));
	CK(cudaMemcpyAsync(h2, a->fq_res.p, 12, cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	if (h2[0]) { ssq_set_error(h2[0] == 2 ? "adjacent records with different names (unpaired reads in an interleaved file)" : "not plain four-line FASTQ"); return SSQ_EFORMAT; }
	a->n_reads = (int)n_reads; a->paired = paired ? 1 : 0; a->n_processed = n_processed; a->has_qual = 1; a->has_cmt = keep_comment && tot[2] > 0;
	a->total_bases = tot[0]; a->max_len = (int)h2[2];
	uint8_t *d_seq; u64 *d_off;
	if ((rc = ssq_batch_reserve(a->b, (int)n_reads, tot[0], a->max_len, &d_seq, &d_off))) return rc;
	if (a->d_ascii.need(tot[0] + 16) || a->d_qual.need(tot[0] + 16) || a->d_names.need(tot[1] + 16) || a->d_name_off.need(((size_t)n_reads + 1) * 4) || a->d_cmt.need(tot[2] + 16) ||
	    a->d_cmt_off.need(((size_t)n_reads + 1) * 4)) return SSQ_ENOMEM;
	k_fq_gather<<<(n_reads + 1 + 127) / 128, 128, 0, st>>>(n_reads, a->fq_txt[0].as<char>(), r1, nf == 2 ? a->fq_txt[1].as<char>() : 0, r2, keep_comment, soff, a->fq_noff.as<u64>(), a->fq_coff.as<u64>(),
	                                                         a->d_ascii.as<char>(), a->d_qual.as<char>(), a->d_names.as<char>(), a->d_cmt.as<char>(), d_off, a->d_name_off.as<u32>(), a->d_cmt_off.as<u32>());
	if (tot[0]) k_encode<<<(unsigned)((tot[0] / 4 + 256) / 256), 256, 0, st>>>(tot[0], a->d_ascii.as<char>(), d_seq);
	CK(cudaGetLastError());
	// how much text the batch covers
	for (int f = 0; f < nf; ++f) {
		const u32 recs = nf == 2 ? take : n_reads, last_line = 4 * recs - 1;
		u32 pos = 0;
		if (last_line < n_lines[f]) { CK(cudaMemcpyAsync(&pos, a->fq_nl[f].as<u32>() + last_line, 4, cudaMemcpyDeviceToHost, st)); CK(cudaStreamSynchronize(st)); pos += 1; }
		else pos = (u32)len[f];
		if (f == 0) *used1 = pos; else *used2 = pos;
	}
	CK(cudaEventRecord(a->ev[ST_ALIGN], st));
	CK(cudaStreamSynchronize(st));
	*n_reads_out = (int)n_reads;
	return SSQ_OK;
}

// ---- BAM output (f1) ----
extern "C" int ssq_aligner_set_bam(ssq_aligner_t *a, int enable, int blank_side_streams)
{
	if (!a) return SSQ_EINVAL;
	a->want_bam = enable ? 1 : 0; a->bam_blank_side = blank_side_streams ? 1 : 0;
	return SSQ_OK;
}
extern "C" int ssq_aligner_fetch_bam(ssq_aligner_t *a, int stream, const void **records, size_t *len)
{
	if (!a || !records || !len || stream < 0 || stream > 2 || !a->computed || !a->want_bam) return SSQ_EINVAL;
	int rc = ssq_use_device(a->device);
	if (rc) return rc;
	if (a->h_bam[stream].need(a->bam_len[stream] + 1)) return SSQ_ENOMEM;
	if (a->bam_len[stream]) { CK(cudaMemcpyAsync(a->h_bam[stream].p, a->d_bam[stream].p, a->bam_len[stream], cudaMemcpyDeviceToHost, a->st)); CK(cudaStreamSynchronize(a->st)); }
	*records = a->h_bam[stream].p; *len = a->bam_len[stream];
	return SSQ_OK;
}
