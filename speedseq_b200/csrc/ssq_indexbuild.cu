// ssq_indexbuild.cu — `bwa index` on the GPU: FASTA -> PREFIX.{amb,ann,pac,bwt,sa}.
//
// Reference call site: `$BWA index $REF` at speedseq/bin/speedseq:389 (and :1925); the five files must be
// byte-identical to what upstream bwa writes — pinned by the reference's goldens
// speedseq/example/data/human_g1k_v37_20_42220611-42542245.fasta.{amb,ann,pac,bwt,sa} (tests/test_gpu_index.py).
// Upstream routines replaced (not vendored in the reference tree): bns_fasta2bntseq, bwt_pac2bwt/bwt_bwtgen,
// bwt_bwtupdate_core, bwt_cal_sa.
//
// Design: the text T = forward + reverse-complement strand never leaves its 2-bit packing; the suffix array of T$ is
// built by prefix doubling where every round is one LSD radix sort of (rank[i], rank[i+h]) pairs over all suffixes
// (CUB DeviceRadixSort — HBM-streaming plumbing), ranks are re-derived with a max-scan, and the loop stops when all ranks
// are distinct (h doubles from 16, so ~log2(longest repeat/16) rounds).  BWT symbols, the occ checkpoints every 128
// symbols and the SA samples every 32 rows are then gathered by streaming kernels and written in the reference's layout.
// The device sort holds 2*l_pac + 1 < 2^31 suffixes (1.07 Gbp).  Beyond that (whole GRCh37: 6.2 G suffixes) the suffix array is
// built on the host — induced sorting with 64-bit indices (ssq_sais.h), BWT / occ checkpoints / SA samples by host threads — and
// written in the same layout; no GPU is touched on that path (SSQ_INDEX_HOST=1 forces it for any size: the CPU tests pin it on
// the reference's goldens).  FASTA parsing and the lrand48() replacement of ambiguous bases are inherently sequential (the
// random stream is consumed in file order) and run on the host.
#include <cuda_runtime.h>
#include <cub/cub.cuh>
#include <zlib.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <ctype.h>
#include <string>
#include <vector>
#include <thread>
#include "ssq_host.h"
#include "ssq_sais.h"

#define CKB(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { ssq_set_error("%s:%d: %s", __FILE__, __LINE__, cudaGetErrorString(e_)); rc = SSQ_ECUDA; goto done; } } while (0)

// ---------------------------------------------------------------------------- host: FASTA ----
struct FaContig { std::string name, anno; i64 offset; i32 len, n_ambs; };
struct FaHole { i64 offset; i32 len; char amb; };

static inline int nt4(int c)
{
	switch (c) { case 'A': case 'a': return 0; case 'C': case 'c': return 1; case 'G': case 'g': return 2; case 'T': case 't': return 3; }
	return 4;
}

// streams the FASTA once: header line = name up to the first blank + optional comment; every non-blank residue
// character is one base; ambiguity codes become lrand48()&3 (seed 11) and are logged as holes, runs of the same
// letter merged
static int parse_fasta(const char *fn, std::vector<FaContig> &ctg, std::vector<FaHole> &holes, std::vector<uint8_t> &pac, i64 &l_pac)
{
	gzFile fp = strcmp(fn, "-") ? gzopen(fn, "r") : gzdopen(0, "r");
	if (!fp) return SSQ_EIO;
	std::vector<char> buf(1 << 20);
	bool in_header = false, at_line_start = true, name_done = false;
	int last = 0, n;
	FaContig *cur = 0;
	l_pac = 0;
	srand48(11);
	while ((n = gzread(fp, buf.data(), (unsigned)buf.size())) > 0) {
		for (int i = 0; i < n; ++i) {
			const int c = (unsigned char)buf[i];
			if (in_header) {
				if (c == '\n') { in_header = false; at_line_start = true; if (!cur->anno.empty() && cur->anno.back() == '\r') cur->anno.pop_back(); if (cur->anno.empty() && !cur->name.empty() && cur->name.back() == '\r') cur->name.pop_back(); }
				else if (!name_done) { if (isspace(c)) name_done = true; else cur->name.push_back((char)c); }
				else cur->anno.push_back((char)c);
				continue;
			}
			if (c == '\n') { at_line_start = true; continue; }
			if (at_line_start && c == '>') {
				ctg.push_back(FaContig());
				cur = &ctg.back();
				cur->offset = l_pac; cur->len = 0; cur->n_ambs = 0;
				in_header = true; name_done = false; last = 0;
				continue;
			}
			at_line_start = false;
			if (!cur || isspace(c)) continue;
			int b = nt4(c);
			if (b >= 4) {
				if (last == c) ++holes.back().len;
				else { FaHole h; h.offset = l_pac; h.len = 1; h.amb = (char)c; holes.push_back(h); ++cur->n_ambs; }
				b = (int)(lrand48() & 3);
			}
			last = c;
			if ((size_t)(l_pac >> 2) >= pac.size()) pac.resize(pac.size() ? pac.size() * 2 : (1 << 20), 0);
			pac[l_pac >> 2] |= (uint8_t)(b << ((~l_pac & 3) << 1));
			++l_pac; ++cur->len;
		}
	}
	gzclose(fp);
	return ctg.empty() || l_pac == 0 ? SSQ_EIO : SSQ_OK;
}

static int write_text_files(const char *prefix, const std::vector<FaContig> &ctg, const std::vector<FaHole> &holes, const std::vector<uint8_t> &pac, i64 l_pac)
{
	std::string p(prefix);
	FILE *fp = fopen((p + ".ann").c_str(), "w");
	if (!fp) return SSQ_EIO;
	fprintf(fp, "%lld %d %u\n", (long long)l_pac, (int)ctg.size(), 11u);
	for (size_t i = 0; i < ctg.size(); ++i) {
		fprintf(fp, "0 %s %s\n", ctg[i].name.c_str(), ctg[i].anno.empty() ? "(null)" : ctg[i].anno.c_str());
		fprintf(fp, "%lld %d %d\n", (long long)ctg[i].offset, ctg[i].len, ctg[i].n_ambs);
	}
	fclose(fp);
	if (!(fp = fopen((p + ".amb").c_str(), "w"))) return SSQ_EIO;
	fprintf(fp, "%lld %d %u\n", (long long)l_pac, (int)ctg.size(), (unsigned)holes.size());
	for (size_t i = 0; i < holes.size(); ++i) fprintf(fp, "%lld %d %c\n", (long long)holes[i].offset, holes[i].len, holes[i].amb);
	fclose(fp);
	if (!(fp = fopen((p + ".pac").c_str(), "wb"))) return SSQ_EIO;
	fwrite(pac.data(), 1, (size_t)((l_pac >> 2) + ((l_pac & 3) ? 1 : 0)), fp);
	uint8_t ct = 0;
	if (l_pac % 4 == 0) fwrite(&ct, 1, 1, fp);
	ct = (uint8_t)(l_pac % 4);
	fwrite(&ct, 1, 1, fp);
	fclose(fp);
	return SSQ_OK;
}

// ------------------------------------------------------------------------------ kernels ----
// symbol i of T (0 <= i < n = 2*l_pac) straight from the 2-bit forward strand
__device__ __forceinline__ u32 tsym(const uint8_t *__restrict__ pac, i64 l_pac, i64 i)
{
	if (i >= l_pac) { const i64 f = 2 * l_pac - 1 - i; return 3u - ((pac[f >> 2] >> ((~f & 3) << 1)) & 3u); }
	return (pac[i >> 2] >> ((~i & 3) << 1)) & 3u;
}

// round 0 key: 16 symbols (zero padded) then min(remaining,16); the sentinel suffix i==n gets the unique smallest key 0
__global__ void k_ib_init(const uint8_t *__restrict__ pac, i64 l_pac, u32 n1, u64 *key, u32 *idx)
{
	const u32 i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n1) return;
	const i64 n = 2 * l_pac;
	u64 k = 0;
	const i64 rem = n - i;
	const int m = rem < 16 ? (int)rem : 16;
	for (int j = 0; j < 16; ++j) k = k << 2 | (j < m ? tsym(pac, l_pac, (i64)i + j) : 0u);
	key[i] = k << 8 | (u64)m;
	idx[i] = i;
}
__global__ void k_ib_flags(u32 n1, const u64 *__restrict__ ks, u32 *head)
{
	const u32 j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= n1) return;
	head[j] = (j == 0 || ks[j] != ks[j - 1]) ? j : 0u;
}
__global__ void k_ib_scatter_rank(u32 n1, const u32 *__restrict__ idx, const u32 *__restrict__ rank_sorted, u32 *rank)
{
	const u32 j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j < n1) rank[idx[j]] = rank_sorted[j];
}
__global__ void k_ib_count_heads(u32 n1, const u32 *__restrict__ rank_sorted, unsigned long long *n_groups)
{
	const u32 j = blockIdx.x * blockDim.x + threadIdx.x;
	unsigned v = (j < n1 && rank_sorted[j] == j) ? 1u : 0u;
	for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
	if ((threadIdx.x & 31) == 0 && v) atomicAdd(n_groups, (unsigned long long)v);
}
__global__ void k_ib_pairkey(u32 n1, u32 h, const u32 *__restrict__ idx, const u32 *__restrict__ rank, u64 *key)
{
	const u32 j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= n1) return;
	const u32 i = idx[j];
	const u64 second = (u64)i + h < (u64)n1 ? (u64)rank[i + h] + 1 : 0;
	key[j] = (u64)rank[i] << 32 | second;
}
__global__ void k_ib_primary(u32 n1, const u32 *__restrict__ sa, u32 *primary)
{
	const u32 j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j < n1 && sa[j] == 0) *primary = j;
}
// BWT symbol stream without the '$' row, one byte per symbol
__global__ void k_ib_bwtsym(const uint8_t *__restrict__ pac, i64 l_pac, u32 n, u32 primary, const u32 *__restrict__ sa, uint8_t *bs)
{
	const u32 j = blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= n) return;
	const u32 r = j + (j >= primary);
	bs[j] = (uint8_t)tsym(pac, l_pac, (i64)sa[r] - 1);
}
// per 128-symbol block: the four symbol counts (for the checkpoint scan)
__global__ void k_ib_blockcnt(u32 n, u32 n_blk, const uint8_t *__restrict__ bs, u64 *c0, u64 *c1, u64 *c2, u64 *c3)
{
	const u32 b = blockIdx.x * blockDim.x + threadIdx.x;
	if (b >= n_blk) return;
	u32 c[4] = {0, 0, 0, 0};
	const u32 lo = b * 128, hi = lo + 128 < n ? lo + 128 : n;
	for (u32 j = lo; j < hi; ++j) ++c[bs[j]];
	c0[b] = c[0]; c1[b] = c[1]; c2[b] = c[2]; c3[b] = c[3];
}
// interleaved layout: block b at words [16b, 16b+16) = u64 occ[4] then 8 symbol words (MSB first); trailing checkpoint after the last word
__global__ void k_ib_interleave(u32 n, u32 n_blk, const uint8_t *__restrict__ bs, const u64 *__restrict__ c0, const u64 *__restrict__ c1,
                                const u64 *__restrict__ c2, const u64 *__restrict__ c3, u32 *out, u64 total_words)
{
	const u32 b = blockIdx.x * blockDim.x + threadIdx.x;
	if (b > n_blk) return;
	if (b == n_blk) { // final checkpoint: totals
		u32 *o = out + total_words - 8; // only 4-byte aligned when the symbol-word count is odd
		const u64 t[4] = {c0[n_blk], c1[n_blk], c2[n_blk], c3[n_blk]};
		for (int c = 0; c < 4; ++c) { o[2 * c] = (u32)t[c]; o[2 * c + 1] = (u32)(t[c] >> 32); }
		return;
	}
	u64 *o = (u64*)(out + (u64)b * 16);
	o[0] = c0[b]; o[1] = c1[b]; o[2] = c2[b]; o[3] = c3[b];
	for (u32 w = 0; w < 8; ++w) {
		const u32 lo = b * 128 + w * 16;
		if (lo >= n) break;
		u32 v = 0;
		for (u32 k = 0; k < 16; ++k) { const u32 j = lo + k; v = v << 2 | (j < n ? (u32)bs[j] : 0u); }
		out[(u64)b * 16 + 8 + w] = v;
	}
}
__global__ void k_ib_sasample(u32 n_sa, const u32 *__restrict__ sa, u64 *out)
{
	const u32 k = blockIdx.x * blockDim.x + threadIdx.x;
	if (k >= 1 && k < n_sa) out[k - 1] = (u64)sa[(u64)k * 32];
}

// ------------------------------------------------------------------------- host path ----
// PREFIX.bwt / PREFIX.sa from the 2-bit forward strand with everything on the host; bits: width of a suffix-array entry (32, 40, 64)
template <class SAP>
static int build_bwt_sa_host_impl(const char *prefix, const std::vector<uint8_t> &pac, i64 l_pac, std::vector<uint8_t> &s, SAP SA);
static int build_bwt_sa_host(const char *prefix, const std::vector<uint8_t> &pac, i64 l_pac, int bits)
{
	const u64 n1 = 2 * (u64)l_pac + 1;
	std::vector<uint8_t> s, raw;
	try { s.resize(n1); raw.resize(n1 * (size_t)(bits / 8) + 8); }
	catch (...) { ssq_set_error("not enough host memory for the suffix array of %llu symbols (%llu GB)", (unsigned long long)(n1 - 1), (unsigned long long)((n1 * (size_t)(bits / 8 + 1)) >> 30)); return SSQ_ENOMEM; }
	if (bits == 32) return build_bwt_sa_host_impl(prefix, pac, l_pac, s, (int32_t*)raw.data());
	if (bits == 64) return build_bwt_sa_host_impl(prefix, pac, l_pac, s, (int64_t*)raw.data());
	ssq_p40 v; v.p = raw.data();
	return build_bwt_sa_host_impl(prefix, pac, l_pac, s, v);
}
template <class SAP>
static int build_bwt_sa_host_impl(const char *prefix, const std::vector<uint8_t> &pac, i64 l_pac, std::vector<uint8_t> &s, SAP SA)
{
	const u64 n = 2 * (u64)l_pac, n1 = n + 1;
	std::vector<u32> out, cnt;
	int n_thr = (int)std::thread::hardware_concurrency();
	if (n_thr < 1) n_thr = 1;
	if (n_thr > 64) n_thr = 64;
	auto par = [&](u64 total, auto fn) { // fn(lo, hi) over [0, total) in n_thr contiguous pieces
		std::vector<std::thread> th;
		const u64 per = (total + n_thr - 1) / n_thr;
		for (int t = 0; t < n_thr; ++t) { const u64 lo = per * t, hi = lo + per < total ? lo + per : total; if (lo < hi) th.emplace_back(fn, lo, hi); }
		for (auto &x : th) x.join();
	};
	// T$ over {0: '$', 1..4: A C G T}: forward strand then its reverse complement (tsym on the device path)
	par(n, [&](u64 lo, u64 hi) {
		for (u64 i = lo; i < hi; ++i) {
			const bool fw = i < (u64)l_pac;
			const u64 p = fw ? i : n - 1 - i;
			const int b = pac[p >> 2] >> ((~p & 3) << 1) & 3;
			s[i] = (uint8_t)(1 + (fw ? b : 3 - b));
		}
	});
	s[n] = 0;
	ssq_sais(s.data(), SA, (int64_t)n1, (int64_t)5);
	u64 primary = 0;
	{
		std::vector<u64> found(n_thr + 1, ~0ull);
		std::vector<std::thread> th;
		const u64 per = (n1 + n_thr - 1) / n_thr;
		for (int t = 0; t < n_thr; ++t) th.emplace_back([&, t]() { const u64 lo = per * t, hi = lo + per < n1 ? lo + per : n1; for (u64 r = lo; r < hi; ++r) if ((i64)SA[(i64)r] == 0) found[t] = r; });
		for (auto &x : th) x.join();
		for (int t = 0; t < n_thr; ++t) if (found[t] != ~0ull) primary = found[t];
	}
	// interleaved occ/BWT: block b at words [16b, 16b+16) = u64 occ[4] then 8 words of 16 symbols (MSB first); totals after the last word
	const u64 n_blk = (n + 127) / 128, raw_words = (n + 15) / 16, total_words = raw_words + (n_blk + 1) * 8;
	try { out.assign(total_words, 0); cnt.assign((n_blk + 1) * 4, 0); } catch (...) { ssq_set_error("not enough host memory for the BWT"); return SSQ_ENOMEM; }
	par(n_blk, [&](u64 lo, u64 hi) {
		for (u64 b = lo; b < hi; ++b) {
			u32 c[4] = {0, 0, 0, 0};
			for (u32 w = 0; w < 8; ++w) {
				const u64 j0 = b * 128 + (u64)w * 16;
				if (j0 >= n) break;
				u32 v = 0;
				for (u32 k = 0; k < 16; ++k) {
					const u64 j = j0 + k;
					u32 sym = 0;
					if (j < n) { const u64 r = j + (j >= primary); sym = (u32)s[(u64)(i64)SA[(i64)r] - 1] - 1; ++c[sym]; }
					v = v << 2 | sym;
				}
				out[b * 16 + 8 + w] = v;
			}
			for (int k = 0; k < 4; ++k) cnt[b * 4 + k] = c[k];
		}
	});
	u64 run[4] = {0, 0, 0, 0};
	for (u64 b = 0; b <= n_blk; ++b) { // checkpoints: counts before the block; the last one (totals) sits 8 words before the end
		u32 *o = b < n_blk ? &out[b * 16] : &out[total_words - 8];
		for (int k = 0; k < 4; ++k) { o[2 * k] = (u32)run[k]; o[2 * k + 1] = (u32)(run[k] >> 32); if (b < n_blk) run[k] += cnt[b * 4 + k]; }
	}
	u64 L2[5] = {0, run[0], run[0] + run[1], run[0] + run[1] + run[2], run[0] + run[1] + run[2] + run[3]};
	std::string p(prefix);
	FILE *fp = fopen((p + ".bwt").c_str(), "wb");
	if (!fp) { ssq_set_error("cannot write %s.bwt", prefix); return SSQ_EIO; }
	fwrite(&primary, 8, 1, fp); fwrite(L2 + 1, 8, 4, fp); fwrite(out.data(), 4, out.size(), fp);
	if (fclose(fp)) { ssq_set_error("cannot write %s.bwt", prefix); return SSQ_EIO; }
	std::vector<u32>().swap(out); std::vector<u32>().swap(cnt);
	const u64 n_sa = (n + 32) / 32, sa_intv = 32, seq_len = n;
	std::vector<u64> smp(n_sa ? n_sa - 1 : 0);
	for (u64 k = 1; k < n_sa; ++k) smp[k - 1] = (u64)(i64)SA[(i64)(k * 32)];
	if (!(fp = fopen((p + ".sa").c_str(), "wb"))) { ssq_set_error("cannot write %s.sa", prefix); return SSQ_EIO; }
	fwrite(&primary, 8, 1, fp); fwrite(L2 + 1, 8, 4, fp); fwrite(&sa_intv, 8, 1, fp); fwrite(&seq_len, 8, 1, fp); fwrite(smp.data(), 8, smp.size(), fp);
	if (fclose(fp)) { ssq_set_error("cannot write %s.sa", prefix); return SSQ_EIO; }
	return SSQ_OK;
}

// -------------------------------------------------------------------------------- driver ----
extern "C" int ssq_index_build(const char *fasta, const char *prefix, int device)
{
	if (!fasta) return SSQ_EINVAL;
	if (!prefix) prefix = fasta;
	int rc;
	std::vector<FaContig> ctg; std::vector<FaHole> holes; std::vector<uint8_t> pac;
	i64 l_pac = 0;
	if ((rc = parse_fasta(fasta, ctg, holes, pac, l_pac))) { ssq_set_error("cannot read any sequence from %s", fasta); return rc; }
	pac.resize((size_t)(l_pac >> 2) + 2, 0);
	const i64 n64 = 2 * l_pac;
	const char *force = getenv("SSQ_INDEX_HOST"); // 1: host path with the narrowest entry type that fits, 40 / 64: with 40- / 64-bit entries
	if (n64 + 1 >= 0x7fffffffLL || (force && atoi(force))) { // beyond the device sort of this build (or asked for): everything on the host, no GPU needed
		if ((rc = write_text_files(prefix, ctg, holes, pac, l_pac))) { ssq_set_error("cannot write %s.{ann,amb,pac}", prefix); return rc; }
		const int f = force ? atoi(force) : 0; // entry width: what was asked for, else 32 bits while they suffice, else 40 (5 bytes per suffix)
		return build_bwt_sa_host(prefix, pac, l_pac, f == 64 ? 64 : (f == 40 || n64 + 1 >= 0x7fffffffLL) ? 40 : 32);
	}
	if ((rc = ssq_use_device(device))) return rc;
	if ((rc = write_text_files(prefix, ctg, holes, pac, l_pac))) { ssq_set_error("cannot write %s.{ann,amb,pac}", prefix); return rc; }
	const u32 n = (u32)n64, n1 = n + 1;
	const unsigned G1 = (n1 + 255) / 256;
	uint8_t *d_pac = 0, *d_bs = 0;
	u64 *d_key[2] = {0, 0}, *d_cnt[4] = {0, 0, 0, 0}, *d_cnts[4] = {0, 0, 0, 0}, *d_sas = 0;
	u32 *d_idx[2] = {0, 0}, *d_rank = 0, *d_head = 0, *d_misc = 0, *d_out = 0;
	void *d_tmp = 0;
	size_t tmp_bytes = 0, tb;
	unsigned long long n_groups = 0;
	u32 primary = 0;
	u64 L2[5] = {0, 0, 0, 0, 0};
	const u32 n_blk = (n + 127) / 128;
	const u64 raw_words = ((u64)n + 15) / 16, total_words = raw_words + ((u64)n_blk + 1) * 8;
	const u32 n_sa = (u32)(((u64)n + 32) / 32);
	std::vector<uint8_t> h_out;
	FILE *fp = 0;
	cub::DoubleBuffer<u64> kb; cub::DoubleBuffer<u32> vb;
	CKB(cudaMalloc(&d_pac, pac.size()));
	CKB(cudaMemcpy(d_pac, pac.data(), pac.size(), cudaMemcpyHostToDevice));
	for (int i = 0; i < 2; ++i) { CKB(cudaMalloc(&d_key[i], (size_t)n1 * 8)); CKB(cudaMalloc(&d_idx[i], (size_t)n1 * 4)); }
	CKB(cudaMalloc(&d_rank, (size_t)n1 * 4)); CKB(cudaMalloc(&d_head, (size_t)n1 * 4)); CKB(cudaMalloc(&d_misc, 64));
	kb = cub::DoubleBuffer<u64>(d_key[0], d_key[1]); vb = cub::DoubleBuffer<u32>(d_idx[0], d_idx[1]);
	cub::DeviceRadixSort::SortPairs(0, tmp_bytes, kb, vb, (int)n1, 0, 64);
	tb = 0; cub::DeviceScan::InclusiveScan(0, tb, d_head, d_head, cub::Max(), (int)n1); if (tb > tmp_bytes) tmp_bytes = tb;
	tb = 0; cub::DeviceScan::ExclusiveSum(0, tb, (u64*)0, (u64*)0, (int)n_blk + 1); if (tb > tmp_bytes) tmp_bytes = tb;
	CKB(cudaMalloc(&d_tmp, tmp_bytes));
	// round 0: 16-mer keys
	k_ib_init<<<G1, 256>>>(d_pac, l_pac, n1, kb.Current(), vb.Current());
	CKB(cub::DeviceRadixSort::SortPairs(d_tmp, tmp_bytes, kb, vb, (int)n1, 0, 40));
	for (u32 h = 16;; h <<= 1) {
		// ranks = position of the head of each run of equal keys
		k_ib_flags<<<G1, 256>>>(n1, kb.Current(), d_head);
		CKB(cub::DeviceScan::InclusiveScan(d_tmp, tmp_bytes, d_head, d_head, cub::Max(), (int)n1));
		k_ib_scatter_rank<<<G1, 256>>>(n1, vb.Current(), d_head, d_rank);
		CKB(cudaMemset(d_misc, 0, 16));
		k_ib_count_heads<<<G1, 256>>>(n1, d_head, (unsigned long long*)d_misc);
		CKB(cudaMemcpy(&n_groups, d_misc, 8, cudaMemcpyDeviceToHost));
		if (n_groups == n1) break;
		if (h >= n1) { ssq_set_error("suffix sort did not converge"); rc = SSQ_ECUDA; goto done; }
		k_ib_pairkey<<<G1, 256>>>(n1, h, vb.Current(), d_rank, kb.Current());
		CKB(cub::DeviceRadixSort::SortPairs(d_tmp, tmp_bytes, kb, vb, (int)n1, 0, 64));
	}
	{
		const u32 *d_sa = vb.Current(); // SA of T$ (n+1 rows)
		k_ib_primary<<<G1, 256>>>(n1, d_sa, d_misc + 4);
		CKB(cudaMemcpy(&primary, d_misc + 4, 4, cudaMemcpyDeviceToHost));
		CKB(cudaMalloc(&d_bs, (size_t)n + 16));
		k_ib_bwtsym<<<(n + 255) / 256, 256>>>(d_pac, l_pac, n, primary, d_sa, d_bs);
		for (int c = 0; c < 4; ++c) { CKB(cudaMalloc(&d_cnt[c], ((size_t)n_blk + 2) * 8)); CKB(cudaMalloc(&d_cnts[c], ((size_t)n_blk + 2) * 8)); CKB(cudaMemset(d_cnt[c], 0, ((size_t)n_blk + 2) * 8)); }
		k_ib_blockcnt<<<(n_blk + 255) / 256, 256>>>(n, n_blk, d_bs, d_cnt[0], d_cnt[1], d_cnt[2], d_cnt[3]);
		for (int c = 0; c < 4; ++c) CKB(cub::DeviceScan::ExclusiveSum(d_tmp, tmp_bytes, d_cnt[c], d_cnts[c], (int)n_blk + 1));
		for (int c = 0; c < 4; ++c) CKB(cudaMemcpy(&L2[c + 1], d_cnts[c] + n_blk, 8, cudaMemcpyDeviceToHost));
		for (int c = 2; c <= 4; ++c) L2[c] += L2[c - 1];
		CKB(cudaMalloc(&d_out, total_words * 4));
		CKB(cudaMemset(d_out, 0, total_words * 4));
		k_ib_interleave<<<(n_blk + 1 + 255) / 256, 256>>>(n, n_blk, d_bs, d_cnts[0], d_cnts[1], d_cnts[2], d_cnts[3], d_out, total_words);
		CKB(cudaGetLastError());
		h_out.resize(total_words * 4);
		CKB(cudaMemcpy(h_out.data(), d_out, total_words * 4, cudaMemcpyDeviceToHost));
		{
			std::string p(prefix);
			const u64 prim64 = primary;
			if (!(fp = fopen((p + ".bwt").c_str(), "wb"))) { ssq_set_error("cannot write %s.bwt", prefix); rc = SSQ_EIO; goto done; }
			fwrite(&prim64, 8, 1, fp); fwrite(L2 + 1, 8, 4, fp); fwrite(h_out.data(), 1, h_out.size(), fp);
			fclose(fp); fp = 0;
			CKB(cudaMalloc(&d_sas, (size_t)n_sa * 8));
			k_ib_sasample<<<(n_sa + 255) / 256, 256>>>(n_sa, d_sa, d_sas);
			h_out.resize((size_t)(n_sa - 1) * 8);
			CKB(cudaMemcpy(h_out.data(), d_sas, (size_t)(n_sa - 1) * 8, cudaMemcpyDeviceToHost));
			if (!(fp = fopen((p + ".sa").c_str(), "wb"))) { ssq_set_error("cannot write %s.sa", prefix); rc = SSQ_EIO; goto done; }
			const u64 sa_intv = 32, seq_len = n;
			fwrite(&prim64, 8, 1, fp); fwrite(L2 + 1, 8, 4, fp); fwrite(&sa_intv, 8, 1, fp); fwrite(&seq_len, 8, 1, fp);
			fwrite(h_out.data(), 1, h_out.size(), fp);
			fclose(fp); fp = 0;
		}
	}
done:
	if (fp) fclose(fp);
	cudaFree(d_pac); cudaFree(d_bs); cudaFree(d_rank); cudaFree(d_head); cudaFree(d_misc); cudaFree(d_out); cudaFree(d_tmp); cudaFree(d_sas);
	for (int i = 0; i < 2; ++i) { cudaFree(d_key[i]); cudaFree(d_idx[i]); }
	for (int c = 0; c < 4; ++c) { cudaFree(d_cnt[c]); cudaFree(d_cnts[c]); }
	return rc;
}
