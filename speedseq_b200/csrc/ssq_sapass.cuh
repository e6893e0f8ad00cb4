// ssq_sapass.cuh — the device suffix sort behind ssq_index_build_ex (path 2): references of any size up to 2^40 - 1 suffixes
// with 5 bytes of device memory per suffix plus a working budget.
//
// T = forward + reverse-complement strand (n = 2*l_pac symbols, read from the 2-bit forward packing by sp_sym), T$ has n1 = n + 1
// suffixes.  rank[i] is the row of the first suffix of i's current group: a u32 low plane and a u8 high plane (5 bytes per suffix).
//
//   first sort   one scan counts suffixes per bucket (first SP_BUCKET_SYM symbols); the host cuts the buckets into passes of at
//                most the budget's rows (a bucket larger than that is a pass of its own).  Per pass: compact the suffixes of the
//                pass's buckets with their key (SP_K symbols, zero padded, then the length min(rem, SP_K): a suffix shorter than the
//                key, and $, sorts before every longer suffix that shares its prefix), radix sort, rank = pass row + head offset,
//                and every group of size > 1 goes to the unresolved list as (group row, suffix) pairs in row order.
//   rounds       Larsson–Sadakane doubling restricted to the unresolved groups, depth h = SP_K, 2 SP_K, 4 SP_K, ...: the host cuts
//                the list into chunks of whole groups; per chunk, gather rank[i + h] for every member (all reads before any write),
//                sort by (group within the chunk, that rank), write the subgroup heads' rows, keep the subgroups of size > 1.
//                A round covers every chunk before the next begins, so every rank read in round h is at least h-ordered; as a
//                group is never split across chunks, a rank refined by an earlier chunk of the same round is still a valid
//                h-order rank.  Every unresolved member has i + h <= n: a suffix shorter than h is already unique.
//   finalise     the ranks are now the inverse suffix array.  Per range of BWT symbols [j0, j1) (j0 a multiple of 128): one scan
//                of the rank array scatters the suffix array of rows [j0, j1 + 1), then BWT symbols (the '$' row omitted: symbol
//                j is row j + (j >= primary)), occ checkpoints every 128 symbols carried across ranges, SA samples every 32 rows;
//                streamed to PREFIX.bwt / PREFIX.sa.
//
// Because of the $, the suffix array is unique, so the files do not depend on the budget, the pass cuts or the chunking.
// The driver sp_build is written once against a backend: SpDevice (ssq_indexbuild.cu: kernels + CUB) and the host loops of
// tests/hostsim/sapass_host.cpp, which restate it on the CPU with the same planners and per-element bodies.
#pragma once
#include <stdio.h>
#include <string.h>
#include <string>
#include <vector>
#include "ssq_dev.cuh"

void ssq_set_error(const char *fmt, ...);

#ifndef SP_ASSERT
#define SP_ASSERT(c) ((void)0)
#endif

#define SP_K 28                        // symbols in the first-sort key (2 bits each, then an 8-bit length)
#define SP_BUCKET_SYM 12               // leading symbols that name a bucket: the key's top 24 bits
#define SP_NBUCKET (1ull << (2 * SP_BUCKET_SYM))
#define SP_PASS_ROW_BYTES 40ull        // per row of a pass: keys, values, their alternates, compaction output (u64 each)
#define SP_CHUNK_ROW_BYTES 48ull       // per member of a chunk: the same five arrays + per-group row and start
#define SP_FIN_ROW_BYTES 11ull         // per row of a finalisation range: SA (u64), BWT byte, checkpoints, packed words, samples
#define SP_MAX_ROWS ((1ull << 30) - 1) // rows per pass / members per chunk (CUB's int item counts); one bucket or group may exceed it only up to SP_MAX_ALONE
#define SP_MAX_ALONE ((1ull << 31) - 2)
#define SP_GROUP_BITS 24               // round key: local group ordinal << 40 | rank[i + h]; chunks of several groups hold < 2^24 members
#define SP_MAX_N1 (1ull << 40)

// ------------------------------------------------------------------ per-element bodies ----
// symbol i of T (0 <= i < n = 2*l_pac) straight from the 2-bit forward strand
SSQ_HD u32 sp_sym(const uint8_t *pac, i64 l_pac, i64 i)
{
	if (i >= l_pac) { const i64 f = 2 * l_pac - 1 - i; return 3u - ((pac[f >> 2] >> ((~f & 3) << 1)) & 3u); }
	return (pac[i >> 2] >> ((~i & 3) << 1)) & 3u;
}
// first-sort key: SP_K symbols (zero padded) then min(n - i, SP_K); $ (i == n) gets the unique smallest key 0
SSQ_HD u64 sp_key(const uint8_t *pac, i64 l_pac, u64 i)
{
	const u64 rem = 2 * (u64)l_pac - i;
	const int m = rem < SP_K ? (int)rem : SP_K;
	u64 k = 0;
	for (int j = 0; j < SP_K; ++j) k = k << 2 | (j < m ? sp_sym(pac, l_pac, (i64)(i + j)) : 0u);
	return k << 8 | (u64)m;
}
SSQ_HD u64 sp_bucket(u64 key) { return key >> (64 - 2 * SP_BUCKET_SYM); }
SSQ_HD u64 sp_rank(const u32 *lo, const uint8_t *hi, u64 i) { return (u64)hi[i] << 32 | lo[i]; }
SSQ_HD void sp_set_rank(u32 *lo, uint8_t *hi, u64 i, u64 r) { lo[i] = (u32)r; hi[i] = (uint8_t)(r >> 32); }
// slot of a selected element in a compacted output (one atomic per warp on the device; in order on the host)
SSQ_HD u64 sp_claim(unsigned long long *ctr, bool sel)
{
#ifdef __CUDA_ARCH__
	const unsigned act = __activemask(), m = __ballot_sync(act, sel);
	if (!m) return ~0ull;
	const int lane = threadIdx.x & 31, leader = __ffs(m) - 1;
	unsigned long long base = 0;
	if (lane == leader) base = atomicAdd(ctr, (unsigned long long)__popc(m));
	base = __shfl_sync(act, base, leader);
	return sel ? base + __popc(m & ((1u << lane) - 1)) : ~0ull;
#else
	return sel ? (*ctr)++ : ~0ull;
#endif
}
SSQ_HD void sp_add(unsigned long long *p, unsigned long long v)
{
#ifdef __CUDA_ARCH__
	atomicAdd(p, v);
#else
	*p += v;
#endif
}

struct SpCount { // suffixes per bucket
	const uint8_t *pac; i64 l_pac; unsigned long long *cnt;
	SSQ_HD void operator()(u64 i) const { sp_add(cnt + sp_bucket(sp_key(pac, l_pac, i)), 1); }
};
struct SpSelect { // the suffixes of buckets [b0, b1) with their keys, in any order
	const uint8_t *pac; i64 l_pac; u64 b0, b1; u64 *key, *idx; unsigned long long *ctr;
	SSQ_HD void operator()(u64 i) const
	{
		const u64 k = sp_key(pac, l_pac, i), b = sp_bucket(k);
		const u64 at = sp_claim(ctr, b >= b0 && b < b1);
		if (at != ~0ull) { key[at] = k; idx[at] = i; }
	}
};
struct SpGather { // round key of a member: local group ordinal (already in key) << 40 | rank[i + h]
	const u32 *lo; const uint8_t *hi; u64 h, n; u64 *key; const u64 *idx;
	SSQ_HD void operator()(u64 j) const
	{
		SP_ASSERT(idx[j] + h <= n);
		key[j] = key[j] << 40 | sp_rank(lo, hi, idx[j] + h);
	}
};
struct SpHead { // sorted position j -> j at the first of a run of equal keys, else 0 (then a max-scan gives each row its head)
	const u64 *key; u64 *head;
	SSQ_HD void operator()(u64 j) const { head[j] = (j == 0 || key[j] != key[j - 1]) ? j : 0; }
};
struct SpRankPass { // first sort: rank = pass row + head offset; key[j] := the rank (the key is dead)
	u64 row0; const u64 *head, *idx; u64 *key; u32 *lo; uint8_t *hi;
	SSQ_HD void operator()(u64 j) const { const u64 r = row0 + head[j]; key[j] = r; sp_set_rank(lo, hi, idx[j], r); }
};
struct SpRankRound { // round: rank = group row + (head offset - group start in the chunk)
	const u64 *grow, *gstart, *head, *idx; u64 *key; u32 *lo; uint8_t *hi;
	SSQ_HD void operator()(u64 j) const
	{
		const u64 g = key[j] >> 40, r = grow[g] + head[j] - gstart[g];
		key[j] = r; sp_set_rank(lo, hi, idx[j], r);
	}
};
struct SpOpen { // 1 when sorted position j belongs to a group of size > 1 (flag[m] = 0 closes the scan)
	const u64 *head; u64 m; u64 *flag;
	SSQ_HD void operator()(u64 j) const
	{
		if (j == m) { flag[j] = 0; return; }
		const bool single = head[j] == j && (j + 1 == m || head[j + 1] == j + 1);
		flag[j] = single ? 0 : 1;
	}
};
struct SpKeep { // stable compaction of the open members: (group row, suffix) in sorted order
	const u64 *pos, *rank, *idx; u64 *out_row, *out_idx;
	SSQ_HD void operator()(u64 j) const { if (pos[j + 1] != pos[j]) { out_row[pos[j]] = rank[j]; out_idx[pos[j]] = idx[j]; } }
};
struct SpScatterSa { // inverse SA -> SA of rows [w0, w1)
	const u32 *lo; const uint8_t *hi; u64 w0, w1; u64 *sa;
	SSQ_HD void operator()(u64 i) const { const u64 r = sp_rank(lo, hi, i); if (r >= w0 && r < w1) sa[r - w0] = i; }
};
struct SpBwtSym { // BWT symbol j0 + jj without the '$' row; sa holds rows from w0
	const uint8_t *pac; i64 l_pac; u64 j0, primary, w0; const u64 *sa; uint8_t *bs;
	SSQ_HD void operator()(u64 jj) const { const u64 j = j0 + jj, r = j + (j >= primary); bs[jj] = (uint8_t)sp_sym(pac, l_pac, (i64)sa[r - w0] - 1); }
};
struct SpBlockCnt { // per 128-symbol block: the four symbol counts
	u64 cnt; const uint8_t *bs; u64 *c0, *c1, *c2, *c3;
	SSQ_HD void operator()(u64 b) const
	{
		u64 c = 0; // four 16-bit counters (at most 128 each): stays in a register, where an array indexed by the symbol would not
		const u64 lo = b * 128, hi = lo + 128 < cnt ? lo + 128 : cnt;
		for (u64 j = lo; j < hi; ++j) c += 1ull << (16 * bs[j]);
		c0[b] = c & 0xffff; c1[b] = c >> 16 & 0xffff; c2[b] = c >> 32 & 0xffff; c3[b] = c >> 48;
	}
};
// interleaved layout: block b at words [16b, 16b+16) = u64 occ[4] (carry + counts before the block) then 8 symbol words (MSB
// first); the last range also writes the totals checkpoint after its last word.  c* = exclusive sums of the block counts.
struct SpInterleave {
	u64 cnt, n_blk, total_words; const uint8_t *bs; const u64 *c0, *c1, *c2, *c3; u64 carry[4]; int last; u32 *out;
	SSQ_HD void operator()(u64 b) const
	{
		if (b == n_blk) {
			if (!last) return;
			u32 *o = out + total_words - 8; // only 4-byte aligned when the symbol-word count is odd
			const u64 t[4] = {carry[0] + c0[n_blk], carry[1] + c1[n_blk], carry[2] + c2[n_blk], carry[3] + c3[n_blk]};
			for (int c = 0; c < 4; ++c) { o[2 * c] = (u32)t[c]; o[2 * c + 1] = (u32)(t[c] >> 32); }
			return;
		}
		u64 *o = (u64*)(out + b * 16);
		o[0] = carry[0] + c0[b]; o[1] = carry[1] + c1[b]; o[2] = carry[2] + c2[b]; o[3] = carry[3] + c3[b];
		for (u32 w = 0; w < 8; ++w) {
			const u64 lo = b * 128 + w * 16;
			if (lo >= cnt) break;
			u32 v = 0;
			for (u32 k = 0; k < 16; ++k) { const u64 j = lo + k; v = v << 2 | (j < cnt ? (u32)bs[j] : 0u); }
			out[b * 16 + 8 + w] = v;
		}
	}
};
struct SpSaSample { // sample k0 + kk = row 32 (k0 + kk); sa holds rows from w0
	u64 k0, w0; const u64 *sa; u64 *out;
	SSQ_HD void operator()(u64 kk) const { out[kk] = (u64)sa[(k0 + kk) * 32 - w0]; }
};

// ------------------------------------------------------------------------------ planners ----
// bucket counts -> pass cuts: bucket ranges [cut[p], cut[p+1]) of at most cap rows; a bucket above cap is a pass of its own
inline void sp_plan_passes(const unsigned long long *cnt, u64 nb, u64 cap, std::vector<u64> &cut, i64 &oversize)
{
	cut.assign(1, 0);
	u64 acc = 0;
	for (u64 b = 0; b < nb; ++b) {
		if (acc && acc + cnt[b] > cap) { cut.push_back(b); acc = 0; }
		if (cnt[b] > cap) ++oversize;
		acc += cnt[b];
	}
	cut.push_back(nb);
}
// group sizes (list order) -> chunk cuts in groups: whole groups, at most cap members (and < 2^SP_GROUP_BITS when several);
// a group above that is a chunk of its own
inline void sp_plan_chunks(const std::vector<u64> &gsize, u64 cap, std::vector<u64> &cut, i64 &oversize)
{
	const u64 lim = cap < (1ull << SP_GROUP_BITS) - 1 ? cap : (1ull << SP_GROUP_BITS) - 1;
	cut.assign(1, 0);
	u64 acc = 0;
	for (u64 g = 0; g < gsize.size(); ++g) {
		if (acc && acc + gsize[g] > lim) { cut.push_back(g); acc = 0; }
		if (gsize[g] > cap) ++oversize;
		acc += gsize[g];
	}
	cut.push_back(gsize.size());
}
inline u64 sp_clamp(u64 v, u64 lo, u64 hi) { return v < lo ? lo : v > hi ? hi : v; }

// ---------------------------------------------------------------------------------- driver ----
struct SpBuf { void *p; u64 cap; };
enum { SP_PAC, SP_LO, SP_HI, SP_K0, SP_V0, SP_K1, SP_V1, SP_X, SP_AUX, SP_NBUF };
template <class B> struct SpBufs { // every working buffer of one build, released on every exit path
	B &be; SpBuf b[SP_NBUF];
	explicit SpBufs(B &e) : be(e) { memset(b, 0, sizeof b); }
	~SpBufs() { for (auto &x : b) be.release(x); }
	int need(int i, u64 bytes) { return be.need(b[i], bytes); }
	template <class T> T *at(int i) { return (T*)b[i].p; }
};

#define SPK(x) do { if ((rc = (x))) goto done; } while (0)

// one sorted pass or chunk after its sort: K = keys, V = suffixes, K2 / V2 free (m + 1 entries).  Writes the ranks (rank(j) as
// in SpRankPass / SpRankRound) and appends the open members (group row, suffix) to the host list, in sorted order.
template <class B, class RankF>
int sp_settle(B &be, SpBufs<B> &M, u64 *K, u64 *V, u64 *K2, u64 *V2, u64 m, RankF rf, std::vector<u64> &out_row, std::vector<u64> &out_idx)
{
	int rc = 0;
	u64 u = 0;
	u64 *X = M.template at<u64>(SP_X);
	SPK(be.each(m, SpHead{K, K2}));
	SPK(be.max_scan(K2, m));
	rf.head = K2; rf.idx = V; rf.key = K;
	SPK(be.each(m, rf));
	SPK(be.each(m + 1, SpOpen{K2, m, V2}));
	SPK(be.excl_sum(V2, m + 1));
	SPK(be.get(&u, V2 + m, 8));
	SPK(be.each(m, SpKeep{V2, K, V, K2, X})); // the heads in K2 are dead once the flags are summed
	if (u) {
		const size_t at = out_row.size();
		out_row.resize(at + u); out_idx.resize(at + u);
		SPK(be.get(out_row.data() + at, K2, u * 8));
		SPK(be.get(out_idx.data() + at, X, u * 8));
	}
done:
	return rc;
}

// PREFIX.bwt / PREFIX.sa of the l_pac-base text in h_pac (2-bit forward packing) within a working budget of `work` bytes beyond
// the rank planes, the text and the bucket counts; stats into st (st->path is the caller's).  chunk_work (0: work) narrows the
// rounds' chunks alone, so that the tests reach one-group chunks without thousands of passes.
template <class B>
int sp_build(B &be, const uint8_t *h_pac, size_t pac_bytes, i64 l_pac, const char *prefix, u64 work, ssq_index_build_stats_t *st, u64 chunk_work = 0)
{
	const u64 n = 2 * (u64)l_pac, n1 = n + 1;
	if (n1 >= SP_MAX_N1) { ssq_set_error("%llu suffixes: the multi-pass sort holds fewer than 2^40", (unsigned long long)n1); return SSQ_EINVAL; }
	const u64 pass_cap = sp_clamp(work / SP_PASS_ROW_BYTES, 1, SP_MAX_ROWS);
	const u64 chunk_cap = sp_clamp((chunk_work ? chunk_work : work) / SP_CHUNK_ROW_BYTES, 2, SP_MAX_ROWS);
	const u64 fin_rows = sp_clamp(work / SP_FIN_ROW_BYTES, 128, SP_MAX_ROWS) & ~127ull;
	const u64 aux0 = SP_NBUCKET * 8 + 64;
	int rc = 0;
	SpBufs<B> M(be);
	std::vector<u64> cut, cur_row, cur_idx, nxt_row, nxt_idx, gsize, gstart, up;
	std::vector<unsigned long long> bcnt;
	std::vector<uint8_t> h_out;
	u64 *K, *V, *K2, *V2, primary = 0, carry[4] = {0, 0, 0, 0}, L2[4];
	unsigned long long *ctr;
	u32 *lo; uint8_t *hi, *pac;
	FILE *fb = 0, *fs = 0;
	bool wrote = false;
	std::string p(prefix);
	const i64 ps = st->path;
	memset(st, 0, sizeof *st); st->path = ps;
	SPK(M.need(SP_PAC, pac_bytes)); SPK(M.need(SP_LO, n1 * 4)); SPK(M.need(SP_HI, n1));
	pac = M.template at<uint8_t>(SP_PAC); lo = M.template at<u32>(SP_LO); hi = M.template at<uint8_t>(SP_HI);
	SPK(be.put(pac, h_pac, pac_bytes));
	// ---- first sort: bucket counts, pass plan, one sort per pass
	SPK(M.need(SP_AUX, aux0));
	SPK(be.zero(M.b[SP_AUX].p, aux0));
	SPK(be.each(n1, SpCount{pac, l_pac, M.template at<unsigned long long>(SP_AUX)}));
	bcnt.resize(SP_NBUCKET);
	SPK(be.get(bcnt.data(), M.b[SP_AUX].p, SP_NBUCKET * 8));
	sp_plan_passes(bcnt.data(), SP_NBUCKET, pass_cap, cut, st->oversize_groups);
	st->passes = (i64)cut.size() - 1;
	{
		u64 row0 = 0;
		for (size_t q = 0; q + 1 < cut.size(); ++q) {
			u64 m = 0;
			for (u64 b = cut[q]; b < cut[q + 1]; ++b) m += bcnt[b];
			if (m > SP_MAX_ALONE) { ssq_set_error("%llu suffixes share their first %d symbols: more than one sort holds", (unsigned long long)m, SP_BUCKET_SYM); rc = SSQ_EINVAL; goto done; }
			for (int i = SP_K0; i <= SP_X; ++i) SPK(M.need(i, (m + 1) * 8));
			K = M.template at<u64>(SP_K0); V = M.template at<u64>(SP_V0); K2 = M.template at<u64>(SP_K1); V2 = M.template at<u64>(SP_V1);
			ctr = M.template at<unsigned long long>(SP_AUX) + SP_NBUCKET;
			SPK(be.zero(ctr, 8));
			SPK(be.each(n1, SpSelect{pac, l_pac, cut[q], cut[q + 1], K, V, ctr}));
			SPK(be.sort(K, V, K2, V2, m, 64));
			SpRankPass rf = {row0, 0, 0, 0, lo, hi};
			SPK(sp_settle(be, M, K, V, K2, V2, m, rf, cur_row, cur_idx));
			row0 += m;
		}
	}
	st->unresolved_first = (i64)cur_row.size();
	// ---- doubling rounds over the open groups, in chunks of whole groups
	for (u64 h = SP_K; !cur_row.empty(); h *= 2) {
		if (h > n) { ssq_set_error("suffix sort did not converge (depth %llu, %zu open)", (unsigned long long)h, cur_row.size()); rc = SSQ_ECUDA; goto done; }
		++st->rounds;
		gsize.clear(); gstart.clear();
		for (size_t j = 0; j < cur_row.size(); ++j) {
			if (j == 0 || cur_row[j] != cur_row[j - 1]) { gsize.push_back(0); gstart.push_back(j); }
			++gsize.back();
		}
		for (u64 s : gsize) if ((i64)s > st->largest_group) st->largest_group = (i64)s;
		sp_plan_chunks(gsize, chunk_cap, cut, st->oversize_groups);
		nxt_row.clear(); nxt_idx.clear();
		for (size_t q = 0; q + 1 < cut.size(); ++q) {
			const u64 g0 = cut[q], ng = cut[q + 1] - g0, j0 = gstart[g0], m = (cut[q + 1] < gsize.size() ? gstart[cut[q + 1]] : cur_row.size()) - j0;
			if (m > SP_MAX_ALONE) { ssq_set_error("a group of %llu suffixes: more than one sort holds", (unsigned long long)m); rc = SSQ_EINVAL; goto done; }
			++st->chunks;
			for (int i = SP_K0; i <= SP_X; ++i) SPK(M.need(i, (m + 1) * 8));
			SPK(M.need(SP_AUX, ng * 16 > aux0 ? ng * 16 : aux0));
			K = M.template at<u64>(SP_K0); V = M.template at<u64>(SP_V0); K2 = M.template at<u64>(SP_K1); V2 = M.template at<u64>(SP_V1);
			up.resize(m > 2 * ng ? m : 2 * ng);
			for (u64 g = 0; g < ng; ++g) for (u64 j = gstart[g0 + g]; j < gstart[g0 + g] + gsize[g0 + g]; ++j) up[j - j0] = g;
			SPK(be.put(K, up.data(), m * 8));
			SPK(be.put(V, cur_idx.data() + j0, m * 8));
			for (u64 g = 0; g < ng; ++g) { up[g] = cur_row[gstart[g0 + g]]; up[ng + g] = gstart[g0 + g] - j0; }
			u64 *grow = M.template at<u64>(SP_AUX);
			SPK(be.put(grow, up.data(), ng * 16));
			SPK(be.each(m, SpGather{lo, hi, h, n, K, V})); // every read of the chunk before its first write
			int bits = 40;
			while (bits < 64 && (1ull << (bits - 40)) < ng) ++bits;
			SPK(be.sort(K, V, K2, V2, m, bits));
			SpRankRound rf = {grow, grow + ng, 0, 0, 0, lo, hi};
			SPK(sp_settle(be, M, K, V, K2, V2, m, rf, nxt_row, nxt_idx));
		}
		cur_row.swap(nxt_row); cur_idx.swap(nxt_idx);
	}
	std::vector<u64>().swap(cur_row); std::vector<u64>().swap(cur_idx); std::vector<u64>().swap(nxt_row); std::vector<u64>().swap(nxt_idx);
	// ---- finalisation by ranges of BWT symbols
	{
		unsigned char rk[5];
		SPK(be.get(rk, lo, 4)); SPK(be.get(rk + 4, hi, 1));
		primary = (u64)rk[4] << 32 | ((u64)rk[0] | (u64)rk[1] << 8 | (u64)rk[2] << 16 | (u64)rk[3] << 24);
	}
	if (!(fb = fopen((p + ".bwt").c_str(), "wb")) || !(fs = fopen((p + ".sa").c_str(), "wb"))) { ssq_set_error("cannot write %s.{bwt,sa}", prefix); rc = SSQ_EIO; goto done; }
	{
		const u64 hdr[7] = {primary, 0, 0, 0, 0, 32, n};
		wrote = fwrite(hdr, 8, 5, fb) == 5 && fwrite(hdr, 8, 7, fs) == 7;
	}
	for (u64 j0 = 0; j0 < n; j0 += fin_rows) {
		const u64 j1 = j0 + fin_rows < n ? j0 + fin_rows : n, cnt = j1 - j0, last = j1 == n, w1 = last ? n1 : j1 + 1;
		const u64 nb = (cnt + 127) / 128, words = (cnt + 15) / 16 + nb * 8 + (last ? 8 : 0);
		const u64 k0 = j0 / 32 > 0 ? j0 / 32 : 1, k1 = last ? (n + 32) / 32 : j1 / 32;
		SPK(M.need(SP_K0, (w1 - j0) * 8)); SPK(M.need(SP_V0, cnt)); SPK(M.need(SP_AUX, (nb + 1) * 32));
		SPK(M.need(SP_K1, words * 4)); SPK(M.need(SP_X, (k1 > k0 ? k1 - k0 : 1) * 8));
		u64 *sa = M.template at<u64>(SP_K0), *c = M.template at<u64>(SP_AUX);
		uint8_t *bs = M.template at<uint8_t>(SP_V0);
		u32 *out = M.template at<u32>(SP_K1);
		SPK(be.each(n1, SpScatterSa{lo, hi, j0, w1, sa}));
		SPK(be.each(cnt, SpBwtSym{pac, l_pac, j0, primary, j0, sa, bs}));
		SPK(be.zero(c, (nb + 1) * 32));
		SPK(be.each(nb, SpBlockCnt{cnt, bs, c, c + nb + 1, c + 2 * (nb + 1), c + 3 * (nb + 1)}));
		for (int s = 0; s < 4; ++s) SPK(be.excl_sum(c + s * (nb + 1), nb + 1));
		SpInterleave il = {cnt, nb, words, bs, c, c + nb + 1, c + 2 * (nb + 1), c + 3 * (nb + 1), {carry[0], carry[1], carry[2], carry[3]}, (int)last, out};
		SPK(be.zero(out, words * 4));
		SPK(be.each(nb + 1, il));
		for (int s = 0; s < 4; ++s) { u64 t; SPK(be.get(&t, c + s * (nb + 1) + nb, 8)); carry[s] += t; }
		h_out.resize(words * 4);
		SPK(be.get(h_out.data(), out, words * 4));
		wrote = wrote && fwrite(h_out.data(), 1, h_out.size(), fb) == h_out.size();
		if (k1 > k0) {
			SPK(be.each(k1 - k0, SpSaSample{k0, j0, sa, M.template at<u64>(SP_X)}));
			h_out.resize((k1 - k0) * 8);
			SPK(be.get(h_out.data(), M.template at<u64>(SP_X), (k1 - k0) * 8));
			wrote = wrote && fwrite(h_out.data(), 1, h_out.size(), fs) == h_out.size();
		}
		++st->ranges;
	}
	L2[0] = carry[0]; for (int s = 1; s < 4; ++s) L2[s] = L2[s - 1] + carry[s];
	if (!wrote || fseek(fb, 8, SEEK_SET) || fwrite(L2, 8, 4, fb) != 4 || fseek(fs, 8, SEEK_SET) || fwrite(L2, 8, 4, fs) != 4) { ssq_set_error("cannot write %s.{bwt,sa}", prefix); rc = SSQ_EIO; goto done; }
	{
		const int eb = fclose(fb), es = fclose(fs);
		fb = fs = 0;
		if (eb || es) { ssq_set_error("cannot write %s.{bwt,sa}", prefix); rc = SSQ_EIO; goto done; }
	}
	st->peak_device_bytes = (i64)be.peak;
done:
	if (fb) fclose(fb);
	if (fs) fclose(fs);
	return rc;
}
#undef SPK
