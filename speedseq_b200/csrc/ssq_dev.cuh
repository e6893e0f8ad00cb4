// ssq_dev.cuh — device-side data layout and the per-read / per-seed routines of the alignment path.
//
// Everything that is arithmetic lives here as SSQ_HD templates so that (a) the __global__ wrappers in
// ssq_kernels.cu stay thin and (b) tests/hostsim can compile the very same
// routines for the host and compare them with the oracle on a box without a GPU (test-only harness,
// never part of libssq.so: the shipped library has no CPU path).
//
// Reference behaviour being reproduced (upstream bwa, not vendored in the speedseq tree; call site
// speedseq/bin/speedseq:438): SURVEY.md §8a rows a4-a7 and Appendix A.
#pragma once
#include <stdint.h>
#include <string.h>
#include "../../include/ssq.h"

#ifdef __CUDACC__
#define SSQ_HD __host__ __device__ __forceinline__
#define SSQ_D __device__ __forceinline__
#else
#define SSQ_HD inline
#endif

typedef uint64_t u64;
typedef int64_t i64;
typedef uint32_t u32;
typedef int32_t i32;

// three-input max: one VIMNMX3 (DPX) instruction on sm_90+; plain code on the host (tests/hostsim)
SSQ_HD int ssq_max2(int a, int b) { return a > b ? a : b; }
SSQ_HD int ssq_max3(int a, int b, int c)
{
#ifdef __CUDA_ARCH__
	return __vimax3_s32(a, b, c);
#else
	return ssq_max2(ssq_max2(a, b), c);
#endif
}

// ---------------------------------------------------------------- HBM layout of the index ----
// bwt  : the occ-interleaved BWT exactly as in PREFIX.bwt after its 40-byte header: one 64-byte block per
//        128 symbols = u64 occ[4] (A,C,G,T before the block) + u32 w[8] (16 symbols/word, MSB first).
//        64 B = two 32-B sectors = one L2 line half; cudaMalloc alignment keeps blocks line-aligned.
// sa   : u64 SA[32k], k=0..n_sa-1 (sa[0] = -1 like the reference loader).
// pac  : forward strand, 2 bit/base, base i at pac[i>>2] >> ((~i&3)<<1) & 3.
// ann  : per-contig offset/len for rid look-ups.
// bwt32: derived at load time when the index has fewer than 2^32 rows — the same BWT re-blocked for the GPU's 32-byte
//        sector: one block per 64 symbols = u32 occ[4] + u32 w[4].  A rank query reads exactly one sector and counts at
//        most four words.  (Larger indexes keep using the 64-byte on-disk blocks with u64 counts.)
struct DevIndex {
	const u32 *bwt;
	const u32 *bwt32;
	const u64 *sa;
	const uint8_t *pac;
	const i64 *ann_off;
	const i32 *ann_len;
	u64 primary, L2[5], seq_len, n_sa;
	i64 l_pac;
	i32 n_seqs, sa_intv;
	// denser suffix-array sample derived at load time (every sad_intv-th row; u32 when positions fit, 0xffffffff = -1): same
	// values the LF walk would reach, several times fewer dependent steps per look-up.  0 / null: walk to the on-disk sample.
	const u32 *sad32; const u64 *sad64; i32 sad_intv;
	// k-mer jump-start table (opt-in, SSQ_KMER_K): bi-intervals of every string of length 1..kmer_k, see kmer_off()
	const struct KmerEnt *kmer; i32 kmer_k;
};

struct Counters { // device-measured work, feeds roofline.achieved (algorithmic bytes, SURVEY.md §8d)
	unsigned long long occ_smem, occ_sa, sa_reads, sw_calls, sw_cells, sw_bytes, n_seeds, n_regs;
	unsigned long long dbg[16]; // kernel-internal cycle counters (diagnostics); [8..11]: rank-block counter before/after the two backward-sweep launches;
	                            // [12]: seeding queries answered from the k-mer table, [13]: seeding extensions through occ4_pair()
};

template <class U> struct IntvT { U x0, x1, x2; u32 qb, qe; }; // bi-interval + query span [qb,qe)
typedef IntvT<u64> Intv;   // any index
typedef IntvT<u32> Intv32; // indexes with fewer than 2^32 rows (the ones that have the re-blocked bwt32): half the registers and ALU work
template <class U> SSQ_HD Intv widen(const IntvT<U> &v) { Intv r; r.x0 = v.x0; r.x1 = v.x1; r.x2 = v.x2; r.qb = v.qb; r.qe = v.qe; return r; }

// ----------------------------------------------------------------------- occ / extension ----
// counts of A,C,G,T in rows [0,k] given the 16 words of the block holding k ('$'-less coordinate kk)
SSQ_HD void occ4_from_block(const u32 *blk, u64 kk, u64 cnt[4])
{
	const u64 *c64 = (const u64*)blk;
	int r = (int)(kk & 127) + 1; // symbols to count
	u32 acc[4] = {0, 0, 0, 0};
	cnt[0] = c64[0]; cnt[1] = c64[1]; cnt[2] = c64[2]; cnt[3] = c64[3];
#pragma unroll
	for (int j = 0; j < 8; ++j) {
		int n = r - 16 * j;
		if (n > 0) {
			u32 w = blk[8 + j];
			u32 m = n >= 16 ? 0x55555555u : (0x55555555u & ~(0xffffffffu >> (2 * n)));
			u32 lo = w & 0x55555555u, hi = (w >> 1) & 0x55555555u;
#ifdef __CUDA_ARCH__
			acc[0] += __popc(~hi & ~lo & m); acc[1] += __popc(~hi & lo & m);
			acc[2] += __popc(hi & ~lo & m);  acc[3] += __popc(hi & lo & m);
#else
			acc[0] += __builtin_popcount(~hi & ~lo & m); acc[1] += __builtin_popcount(~hi & lo & m);
			acc[2] += __builtin_popcount(hi & ~lo & m);  acc[3] += __builtin_popcount(hi & lo & m);
#endif
		}
	}
	cnt[0] += acc[0]; cnt[1] += acc[1]; cnt[2] += acc[2]; cnt[3] += acc[3];
}

// scalar context: one thread does the whole look-up (used by the SA walk, by hostsim, and as the
// thread-per-read variant of the seeding kernel)
// one 32-byte rank block (u32 occ[4] + 4 words of 16 symbols) = one sector, read with two 128-bit loads (the widest global
// load sm_90 has); both halves are issued before either is used, so a rank query still waits for one memory round trip
struct Blk32 { u32 c0, c1, c2, c3, w0, w1, w2, w3; };
SSQ_HD Blk32 load_blk32(const u32 *p)
{
	Blk32 b;
#ifdef __CUDA_ARCH__
	asm("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%8];\n\t"
	    "ld.global.nc.v4.u32 {%4,%5,%6,%7}, [%8+16];"
	             : "=r"(b.c0), "=r"(b.c1), "=r"(b.c2), "=r"(b.c3), "=r"(b.w0), "=r"(b.w1), "=r"(b.w2), "=r"(b.w3) : "l"(p));
#else
	b.c0 = p[0]; b.c1 = p[1]; b.c2 = p[2]; b.c3 = p[3]; b.w0 = p[4]; b.w1 = p[5]; b.w2 = p[6]; b.w3 = p[7];
#endif
	return b;
}
// occurrences of each base in rows [block start, kk] of a 64-symbol rank block
template <class U>
SSQ_HD void blk32_count(const Blk32 &b, U kk, U cnt[4])
{
	const int r = (int)(kk & 63) + 1; // symbols to count, 1..64
	// two 64-bit lanes of 32 symbols each, MSB-first within each original 32-bit word
	const u64 lo_w = (u64)b.w0 << 32 | b.w1, hi_w = (u64)b.w2 << 32 | b.w3;
	const int n0 = r < 32 ? r : 32, n1 = r - 32 > 0 ? r - 32 : 0;
	const u64 m0 = 0x5555555555555555ull & ~(n0 >= 32 ? 0ull : (~0ull >> (2 * n0)));
	const u64 m1 = n1 <= 0 ? 0ull : (0x5555555555555555ull & ~(n1 >= 32 ? 0ull : (~0ull >> (2 * n1))));
	const u64 l0 = lo_w & m0, h0 = (lo_w >> 1) & m0, l1 = hi_w & m1, h1 = (hi_w >> 1) & m1;
#ifdef __CUDA_ARCH__
	const int p3 = __popcll(h0 & l0) + __popcll(h1 & l1), ph = __popcll(h0) + __popcll(h1), pl = __popcll(l0) + __popcll(l1);
#else
	const int p3 = __builtin_popcountll(h0 & l0) + __builtin_popcountll(h1 & l1), ph = __builtin_popcountll(h0) + __builtin_popcountll(h1), pl = __builtin_popcountll(l0) + __builtin_popcountll(l1);
#endif
	cnt[3] = (U)b.c3 + (U)p3; cnt[2] = (U)b.c2 + (U)(ph - p3); cnt[1] = (U)b.c1 + (U)(pl - p3); cnt[0] = (U)b.c0 + (U)(r - ph - pl + p3);
}

struct ScalarFm {
	const DevIndex &ix;
	u32 n_blk, n_step, n_tab; // rank blocks (sectors) loaded; extensions through occ4_pair(); queries answered from the k-mer table
	SSQ_HD ScalarFm(const DevIndex &i) : ix(i), n_blk(0), n_step(0), n_tab(0) {}
	SSQ_HD void occ4(u64 k, u64 cnt[4])
	{
		if (k == (u64)-1) { cnt[0] = cnt[1] = cnt[2] = cnt[3] = 0; return; }
		u64 kk = k - (k >= ix.primary);
		if (ix.bwt32) { // one 32-byte sector: u32 occ[4] + 64 symbols
			const Blk32 b = load_blk32(ix.bwt32 + ((kk >> 6) << 3));
			++n_blk;
			blk32_count(b, kk, cnt);
			return;
		}
		const u32 *p = ix.bwt + ((kk >> 7) << 4);
		u32 blk[16];
#ifdef __CUDA_ARCH__
		const uint4 *p4 = (const uint4*)p;
		uint4 a = __ldg(p4), b = __ldg(p4 + 1), c = __ldg(p4 + 2), d = __ldg(p4 + 3);
		blk[0] = a.x; blk[1] = a.y; blk[2] = a.z; blk[3] = a.w; blk[4] = b.x; blk[5] = b.y; blk[6] = b.z; blk[7] = b.w;
		blk[8] = c.x; blk[9] = c.y; blk[10] = c.z; blk[11] = c.w; blk[12] = d.x; blk[13] = d.y; blk[14] = d.z; blk[15] = d.w;
#else
		memcpy(blk, p, 64);
#endif
		++n_blk;
		occ4_from_block(blk, kk, cnt);
	}
	SSQ_HD void occ4(u32 k, u32 cnt[4]) // 32-bit rows: only with bwt32
	{
		if (k == (u32)-1) { cnt[0] = cnt[1] = cnt[2] = cnt[3] = 0; return; }
		const u32 kk = k - (k >= (u32)ix.primary);
		const Blk32 b = load_blk32(ix.bwt32 + ((size_t)(kk >> 6) << 3));
		++n_blk;
		blk32_count(b, kk, cnt);
	}
	// both ends of an extension: counts up to rows k0 and k1 (k0 <= k1: the row before an interval and its last row)
	SSQ_HD void occ4_pair(u64 k0, u64 k1, u64 tk[4], u64 tl[4]) { ++n_step; occ4(k0, tk); occ4(k1, tl); }
	// 32-bit rows: once a string is longer than ~16 bases its interval spans a few rows, and both ends often lie in the same 64-row
	// block (36 % of the steps on the bench workload).  That block is then loaded once and both count vectors come from the same
	// registers (one sector instead of two); otherwise both loads are issued before either block is used (one round trip either way).
	SSQ_HD void occ4_pair(u32 k0, u32 k1, u32 tk[4], u32 tl[4])
	{
		++n_step;
		const u32 p = (u32)ix.primary, kk1 = k1 - (k1 >= p);
		const bool none0 = k0 == (u32)-1; // the interval starts at row 0: nothing before it (counted from k1's block, then cleared)
		const u32 kk0 = none0 ? kk1 : k0 - (k0 >= p);
		const Blk32 b0 = load_blk32(ix.bwt32 + ((size_t)(kk0 >> 6) << 3));
		Blk32 b1 = b0;
		if ((kk0 ^ kk1) >> 6) { b1 = load_blk32(ix.bwt32 + ((size_t)(kk1 >> 6) << 3)); ++n_blk; } // issued before either block is used
		++n_blk;
		blk32_count(b1, kk1, tl);
		blk32_count(b0, kk0, tk);
		if (none0) tk[0] = tk[1] = tk[2] = tk[3] = 0;
	}
	// ok[c] of a forward (is_back=0) or backward (is_back=1) extension of ik by every base c
	SSQ_HD void extend(const Intv &ik, Intv ok[4], int is_back)
	{
		u64 tk[4], tl[4];
		u64 kf = is_back ? ik.x0 : ik.x1; // the component looked up in the BWT
		u64 ko = is_back ? ik.x1 : ik.x0; // the component updated by accumulation
		occ4(kf - 1, tk);
		occ4(kf - 1 + ik.x2, tl);
		u64 nf[4], ns[4], no[4];
#pragma unroll
		for (int c = 0; c < 4; ++c) { nf[c] = ix.L2[c] + 1 + tk[c]; ns[c] = tl[c] - tk[c]; }
		no[3] = ko + (kf <= ix.primary && kf + ik.x2 - 1 >= ix.primary);
		no[2] = no[3] + ns[3]; no[1] = no[2] + ns[2]; no[0] = no[1] + ns[1];
#pragma unroll
		for (int c = 0; c < 4; ++c) {
			ok[c].x2 = ns[c];
			if (is_back) { ok[c].x0 = nf[c]; ok[c].x1 = no[c]; } else { ok[c].x1 = nf[c]; ok[c].x0 = no[c]; }
		}
	}
};

#define SSQ_SEL4(v0, v1, v2, v3, c) ((c) == 0 ? (v0) : (c) == 1 ? (v1) : (c) == 2 ? (v2) : (v3))
// only ok[c] of an extension, computed without runtime-indexed arrays (keeps everything in registers on the GPU)
template <class Fm, class U>
SSQ_HD void extend1(Fm &fm, const IntvT<U> &ik, int c, int is_back, IntvT<U> &out)
{
	const DevIndex &ix = fm.ix;
	U tk[4], tl[4];
	const U kf = is_back ? ik.x0 : ik.x1, ko = is_back ? ik.x1 : ik.x0;
	fm.occ4_pair((U)(kf - 1), (U)(kf - 1 + ik.x2), tk, tl);
	const U n0 = tl[0] - tk[0], n1 = tl[1] - tk[1], n2 = tl[2] - tk[2], n3 = tl[3] - tk[3];
	const U nf = SSQ_SEL4((U)ix.L2[0] + 1 + tk[0], (U)ix.L2[1] + 1 + tk[1], (U)ix.L2[2] + 1 + tk[2], (U)ix.L2[3] + 1 + tk[3], c);
	const U base = ko + (U)(kf <= (U)ix.primary && (U)(kf + ik.x2 - 1) >= (U)ix.primary);
	const U no = base + (c < 3 ? n3 : 0) + (c < 2 ? n2 : 0) + (c < 1 ? n1 : 0);
	out.x2 = SSQ_SEL4(n0, n1, n2, n3, c);
	if (is_back) { out.x0 = nf; out.x1 = no; } else { out.x1 = nf; out.x0 = no; }
	out.qb = out.qe = 0;
}

template <class U>
SSQ_HD void set_intv(const DevIndex &ix, int c, IntvT<U> &ik)
{
	ik.x0 = (U)(ix.L2[c] + 1); ik.x2 = (U)(ix.L2[c + 1] - ix.L2[c]); ik.x1 = (U)(ix.L2[3 - c] + 1); ik.qb = ik.qe = 0;
}

// ---------------------------------------------------------------- k-mer jump-start table ----
// A third to a half of the seeding's rank queries produce a string of at most 10-12 bases (tests/hostsim diagnostics: 38 % for
// K = 10, 51 % for K = 12): the first steps of every forward walk and, above all, the short prefixes that survive many backward
// sweeps.  The bi-interval of a string does not depend on how it was reached, so those queries can be answered — exactly — from a
// table of the bi-intervals of all strings of length 1..K: entry (L, code) at kmer_off(L) + code, code = the L bases as a 2L-bit
// number, first base in the top bits.  K = 10: 1.4 M entries x 16 B = 22 MB (L2-resident).  Indexes with < 2^32 rows only.
// Built at index load for every bwt32 index (SSQ_KMER_K overrides K, 0 turns it off) and read by the forward walks (k_smem_fwd,
// k_smem_p3).  K = 10 from an H100 sweep of K = 0, 8, 9, 10 on the bench workload (DESIGN.md §8); K = 11 (89 MB) is not L2-resident.
#define SSQ_KMER_K_DEFAULT 10
struct KmerEnt { u32 x0, x1, x2, pad; };
SSQ_HD u32 kmer_off(int L) { return ((1u << (2 * L)) - 4u) / 3u; } // 4 + 16 + ... + 4^(L-1)
SSQ_HD u32 kmer_entries(int K) { return kmer_off(K + 1); }
template <class Fm>
SSQ_HD KmerEnt kmer_compute(Fm &fm, const DevIndex &ix, int L, u32 code) // by the same forward extensions a walk would make
{
	Intv32 ik, okc;
	set_intv(ix, (int)(code >> (2 * (L - 1)) & 3u), ik);
	for (int j = 1; j < L; ++j) { extend1(fm, ik, 3 - (int)(code >> (2 * (L - 1 - j)) & 3u), 0, okc); ik = okc; }
	KmerEnt e; e.x0 = ik.x0; e.x1 = ik.x1; e.x2 = ik.x2; e.pad = 0;
	return e;
}
SSQ_HD Intv32 kmer_lookup(const DevIndex &ix, int L, u32 code)
{
	const KmerEnt e = ix.kmer[kmer_off(L) + code];
	Intv32 r; r.x0 = e.x0; r.x1 = e.x1; r.x2 = e.x2; r.qb = r.qe = 0;
	return r;
}

// ------------------------------------------------------------------------ SMEM search ----
// Per-read scratch: two ping-pong lists of at most len+1 intervals (shared memory on the device) and an
// output list `mem` (global scratch).  Fm is ScalarFm or the warp-cooperative context of ssq_fm.cu; with the
// latter every lane runs this code with identical values (warp-uniform control flow).
template <class Fm>
SSQ_HD int smem1(Fm &fm, const DevIndex &ix, int len, const uint8_t *q, int x, u64 min_intv,
                 Intv *mem, int mem_cap, int &mem_n, Intv *prev, Intv *curr, int &err)
{
	int i, j, c, ret, n_curr = 0, n_prev, base = mem_n;
	Intv ik, ok[4];
	if (q[x] > 3) return x + 1;
	if (min_intv < 1) min_intv = 1;
	set_intv(ix, q[x], ik);
	ik.qe = x + 1;
	for (i = x + 1; i < len; ++i) { // forward, remembering every change of interval size
		if (q[i] < 4) {
			c = 3 - q[i];
			fm.extend(ik, ok, 0);
			if (ok[c].x2 != ik.x2) {
				curr[n_curr++] = ik;
				if (ok[c].x2 < min_intv) break;
			}
			ik = ok[c]; ik.qe = i + 1;
		} else { curr[n_curr++] = ik; break; }
	}
	if (i == len) curr[n_curr++] = ik;
	for (j = 0; j < n_curr >> 1; ++j) { Intv t = curr[j]; curr[j] = curr[n_curr - 1 - j]; curr[n_curr - 1 - j] = t; } // longest first
	ret = (int)curr[0].qe;
	{ Intv *t = curr; curr = prev; prev = t; n_prev = n_curr; }
	for (i = x - 1; i >= -1; --i) { // backward, the whole set at once
		c = i < 0 ? -1 : q[i] < 4 ? q[i] : -1;
		n_curr = 0;
		for (j = 0; j < n_prev; ++j) {
			Intv p = prev[j];
			if (c >= 0) fm.extend(p, ok, 1);
			if (c < 0 || ok[c].x2 < min_intv) {
				if (n_curr == 0) { // nothing longer survives: p is left-maximal
					if (mem_n == base || (u32)(i + 1) < mem[mem_n - 1].qb) {
						if (mem_n >= mem_cap) { err = 1; return ret; }
						p.qb = (u32)(i + 1);
						mem[mem_n++] = p;
					}
				}
			} else if (n_curr == 0 || ok[c].x2 != curr[n_curr - 1].x2) {
				ok[c].qb = 0; ok[c].qe = p.qe;
				curr[n_curr++] = ok[c];
			}
		}
		if (n_curr == 0) break;
		{ Intv *t = curr; curr = prev; prev = t; n_prev = n_curr; }
	}
	for (j = 0; j < (mem_n - base) >> 1; ++j) { Intv t = mem[base + j]; mem[base + j] = mem[mem_n - 1 - j]; mem[mem_n - 1 - j] = t; }
	return ret;
}

template <class Fm>
SSQ_HD int seed_strategy1(Fm &fm, const DevIndex &ix, int len, const uint8_t *q, int x, int min_len, u64 max_intv, Intv &m)
{
	int i, c;
	Intv ik, ok[4];
	m.x0 = m.x1 = m.x2 = 0; m.qb = m.qe = 0;
	if (q[x] > 3) return x + 1;
	set_intv(ix, q[x], ik);
	for (i = x + 1; i < len; ++i) {
		if (q[i] < 4) {
			c = 3 - q[i];
			fm.extend(ik, ok, 0);
			if (ok[c].x2 < max_intv && i - x >= min_len) {
				m = ok[c]; m.qb = (u32)x; m.qe = (u32)(i + 1);
				return i + 1;
			}
			ik = ok[c];
		} else return i + 1;
	}
	return len;
}

// the three seeding passes of one read; result in mem[0..return) sorted by (qb,qe)
template <class Fm>
SSQ_HD int collect_intv(Fm &fm, const DevIndex &ix, const ssq_opts_t &opt, int len, const uint8_t *q,
                        Intv *mem, int mem_cap, Intv *bufA, Intv *bufB, int &err)
{
	int x = 0, n = 0, i, k, old_n, base;
	int split_len = (int)(opt.min_seed_len * opt.split_factor + .499f);
	if (len < opt.min_seed_len) return 0;
	while (x < len) { // pass 1: SMEMs
		if (q[x] < 4) {
			base = n;
			x = smem1(fm, ix, len, q, x, 1, mem, mem_cap, n, bufA, bufB, err);
			if (err) return 0;
			for (i = k = base; i < n; ++i) if ((int)(mem[i].qe - mem[i].qb) >= opt.min_seed_len) mem[k++] = mem[i];
			n = k;
		} else ++x;
	}
	old_n = n;
	for (k = 0; k < old_n; ++k) { // pass 2: re-seed long, nearly unique SMEMs from their midpoint
		Intv p = mem[k];
		int start = (int)p.qb, end = (int)p.qe, kk;
		if (end - start < split_len || p.x2 > (u64)opt.split_width) continue;
		base = n;
		smem1(fm, ix, len, q, (start + end) >> 1, p.x2 + 1, mem, mem_cap, n, bufA, bufB, err);
		if (err) return 0;
		for (i = kk = base; i < n; ++i) if ((int)(mem[i].qe - mem[i].qb) >= opt.min_seed_len) mem[kk++] = mem[i];
		n = kk;
	}
	if (opt.max_mem_intv > 0) { // pass 3: greedy forward seeds
		x = 0;
		while (x < len) {
			if (q[x] < 4) {
				Intv m;
				x = seed_strategy1(fm, ix, len, q, x, opt.min_seed_len, (u64)opt.max_mem_intv, m);
				if (m.x2 > 0) { if (n >= mem_cap) { err = 1; return 0; } mem[n++] = m; }
			} else ++x;
		}
	}
	// order by (qb<<32|qe); equal keys are identical intervals, so any sort gives the reference order
	for (i = 1; i < n; ++i) {
		Intv t = mem[i];
		u64 key = (u64)t.qb << 32 | t.qe;
		for (k = i; k > 0 && ((u64)mem[k - 1].qb << 32 | mem[k - 1].qe) > key; --k) mem[k] = mem[k - 1];
		mem[k] = t;
	}
	return n;
}

// Phase-split seeding (indexes with < 2^32 rows): the forward phase of an smem1() call does not depend on its backward phase (the
// next call starts at the forward phase's end), so forward walks and backward sweeps can run as separate kernels in which every
// lane is in the same phase.  A call travels between them as a SeedCall + its forward list (the intervals at which the size changed).
struct FwdEntry { u32 x0, x1, x2, qe; };
struct SeedCall { // 32 bytes: everything a lane needs to take the call over with one load
	u32 read, pk, min_intv, list_n; // pk = x | len << 8 | (base at x-1, 0..4) << 16 | (base at x-2) << 20
	u64 list_off, seq_off;          // forward list in the list pool; the read's bases
	SSQ_HD static u32 pack(int x, int len, int b0, int b1) { return (u32)x | (u32)len << 8 | (u32)b0 << 16 | (u32)b1 << 20; }
	SSQ_HD int x() const { return (int)(pk & 0xff); }
	SSQ_HD int len() const { return (int)(pk >> 8 & 0xff); }
	SSQ_HD int b0() const { return (int)(pk >> 16 & 0xf); }
	SSQ_HD int b1() const { return (int)(pk >> 20 & 0xf); }
};

// ------------------------------------------------------------- seeding as a state machine ----
// Same three passes as collect_intv(), unrolled into a machine whose only expensive transition is one rank query.
// A GPU lane owns one machine; all lanes of a warp meet at the query no matter which phase each is in.  advance() runs
// the cheap bookkeeping up to the next query (false = read done), post() consumes the query's result.  Every list
// operation happens in the same order as in smem1()/seed_strategy1().
// Lists: the two ping-pong interval lists behind get/set (shared memory with global overflow on the GPU, plain arrays
// in the host harness); their tails and the tail of the output list are mirrored in registers so that the backward
// phase never waits on a dependent memory read other than the rank query itself.
template <class U>
struct HostListsT { // plain arrays (hostsim, thread-per-read fallbacks)
	IntvT<U> *a[2];
	SSQ_HD IntvT<U> get(int id, int j) const { return a[id][j]; }
	SSQ_HD void set(int id, int j, const IntvT<U> &v) const { a[id][j] = v; }
};
typedef HostListsT<u64> HostLists;

// U: row type of the machine's intervals — u64 for any index, u32 when the index has fewer than 2^32 rows.  The output list
// `mem` always holds 64-bit intervals.
// P3 = false compiles the greedy pass out (its callers run it elsewhere and always pass skip_p3).
// TAB = true (32-bit rows, ix.kmer loaded): rank queries that produce a string of at most ix.kmer_k bases are answered from the
// k-mer jump-start table — table_hit() before extend1().
template <class Lists, class U = u64, bool P3 = true, bool TAB = false>
struct SmemMachineT {
	typedef IntvT<U> I;
	enum { NEXT_P1, NEXT_P2, NEXT_P3, FWD, BWD, S3, DONE };
	const FwdEntry *ext; // backward-only use: the forward list of the call, produced elsewhere (read from its end in the first sweep)
	const uint8_t *q; Intv *mem; Lists L;
	int len, mem_cap, n, state, pass, x, i, j, c, qc, ret, n_prev, n_curr, old_n, k2, err, min_seed_len, split_len, split_width, prev_id;
	int qi, qnext;     // base at position i (forward phases) and the prefetched base at i+1: the load is issued before the rank
	                   // query of step i and consumed after it, so the bookkeeping never waits on a query byte
	int cnext;         // backward phase: prefetched base at i-1
	int cb0, cb1;      // bases at x-1 and x-2 of the current smem1 call, fetched when it starts
	u32 code, win; int tabK; // TAB: last bases of the forward walk's string; FWD: its first tabK bases (left-aligned), BWD: the tabK bases from position i on
	int skip_p3;       // the greedy pass is done elsewhere (the GPU runs it as a kernel of its own, k_smem_p3)
	int rev;           // first backward sweep: the forward list is read from its end (longest match first) instead of being reversed
	int any_kept;      // this smem1 call has kept an interval (whether or not it was long enough to be stored)
	u32 last_qe;       // qe of the entry last pushed by the forward phase
	u32 last_mem_qb;   // qb of the interval this smem1 call kept last
	U curr_tail_x2;    // x2 of the entry last pushed to the current list
	U min_intv, max_mem_intv;
	I ik, in;
	int is_back;

	SSQ_HD int base_at(int p) const { return p >= 0 && p < len ? (int)q[p] : 4; }
	SSQ_HD void init(const ssq_opts_t &opt, int len_, const uint8_t *q_, Intv *mem_, int mem_cap_, const Lists &lists, int skip_p3_ = 0)
	{
		q = q_; len = len_; mem = mem_; mem_cap = mem_cap_; L = lists; prev_id = 0; skip_p3 = skip_p3_;
		n = 0; err = 0; x = 0; pass = 1; state = NEXT_P1; rev = 0; ext = 0; code = 0; win = 0; tabK = 0;
		min_seed_len = opt.min_seed_len; split_len = (int)(opt.min_seed_len * opt.split_factor + .499f); split_width = opt.split_width;
		max_mem_intv = (U)opt.max_mem_intv;
		if (len < opt.min_seed_len) { state = NEXT_P3; pass = 3; x = len; }
	}
	SSQ_HD void push_curr(const I &v) { L.set(prev_id ^ 1, n_curr++, v); curr_tail_x2 = v.x2; }
	SSQ_HD void start_smem1(const DevIndex &ix, int x_, U min_intv_)
	{
		x = x_; min_intv = min_intv_ < 1 ? 1 : min_intv_; any_kept = 0;
		set_intv(ix, q[x], ik); ik.qe = (u32)(x + 1);
		if (TAB) { tabK = ix.kmer_k; code = q[x]; win = (u32)q[x] << (2 * (tabK - 1)); }
		i = x + 1; qi = base_at(i); n_curr = 0; state = FWD;
		{ const int b0 = base_at(x - 1); cb0 = b0 < 4 ? b0 : -1; }
		{ const int b1 = base_at(x - 2); cb1 = b1 < 4 ? b1 : -1; }
	}
	// forward list complete.  smem1() reverses it (longest match first) before walking backwards; here the first backward sweep
	// reads it from the end instead, and its first entry's qe — smem1()'s return value — is the qe of the last push.
	SSQ_HD void end_forward()
	{
		ret = (int)last_qe;
		prev_id ^= 1; n_prev = n_curr; rev = 1;
		i = x - 1; j = 0; n_curr = 0;
		c = cb0; cnext = cb1;
		if (TAB) win = (win >> 2) | (u32)(c < 0 ? 0 : c) << (2 * (tabK - 1)); // positions x-1 .. x-1+tabK-1
		state = BWD;
	}
	// p is left-maximal at i+1 unless a longer match survived.  smem1() appends it and drops the intervals shorter than
	// min_seed_len when the call ends; the decision only needs to know THAT something was kept and its qb, so short ones are
	// not stored in the first place.  (smem1() also reverses the call's output; the final (qb, qe) sort makes that immaterial.)
	SSQ_HD void keep(const I &p_)
	{
		if (n_curr == 0 && (!any_kept || (u32)(i + 1) < last_mem_qb)) {
			any_kept = 1; last_mem_qb = (u32)(i + 1);
			if ((int)p_.qe - (i + 1) >= min_seed_len) {
				if (n >= mem_cap) { err = 1; return; }
				Intv p = widen(p_); p.qb = (u32)(i + 1);
				mem[n++] = p;
			}
		}
	}
	SSQ_HD void end_smem1() { if (pass == 1) { x = ret; state = NEXT_P1; } else if (pass == 0) state = DONE; else state = NEXT_P2; }
	// backward phase only: the call's forward list comes from outside; advance() returns false when the call is complete and
	// mem[0..n) holds its intervals (after init(); 32-bit rows only)
	SSQ_HD void start_backward(int x_, U min_intv_, const FwdEntry *list, int list_n, int b0, int b1) // b0, b1: bases at x-1, x-2 (4 = none / N)
	{
		x = x_; min_intv = min_intv_ < 1 ? 1 : min_intv_; any_kept = 0; pass = 0;
		ext = list; n_prev = list_n; rev = 1; prev_id = 0;
		ret = (int)list[list_n - 1].qe;
		i = x - 1; j = 0; n_curr = 0;
		c = b0 < 4 ? b0 : -1; cnext = b1 < 4 ? b1 : -1;
		state = BWD;
	}
	SSQ_HD I prev_entry(int jj) const
	{
		if (rev && ext) { const FwdEntry e = ext[n_prev - 1 - jj]; I r; r.x0 = (U)e.x0; r.x1 = (U)e.x1; r.x2 = (U)e.x2; r.qb = 0; r.qe = e.qe; return r; }
		return L.get(prev_id, rev ? n_prev - 1 - jj : jj);
	}
	// Runs the bookkeeping up to the next rank query.  true: `in` / `qc` / `is_back` describe it (only ok[qc] is needed);
	// false: the read is complete.  Every transition is a handful of instructions; the only loops are over N bases and over
	// pass-1 intervals that do not qualify for re-seeding.
	SSQ_HD bool advance(const DevIndex &ix)
	{
		for (;;) {
			if (err) return false;
			switch (state) {
			case DONE: return false;
			case NEXT_P1:
				while (x < len && q[x] > 3) ++x;
				if (x >= len) { old_n = n; k2 = 0; pass = 2; state = NEXT_P2; break; }
				start_smem1(ix, x, 1);
				break;
			case NEXT_P2: {
				bool started = false;
				while (k2 < old_n) {
					const Intv p = mem[k2++];
					const int start = (int)p.qb, end = (int)p.qe;
					if (end - start < split_len || p.x2 > (u64)split_width) continue;
					start_smem1(ix, (start + end) >> 1, (U)(p.x2 + 1));
					started = true;
					break;
				}
				if (!started) { pass = 3; x = 0; state = NEXT_P3; if (max_mem_intv == 0 || skip_p3 || !P3) x = len; }
				break;
			}
			case NEXT_P3:
				if (!P3) return false;
				while (x < len && q[x] > 3) ++x;
				if (x >= len) return false;
				set_intv(ix, q[x], ik);
				i = x + 1; qi = base_at(i); state = S3;
				break;
			case FWD:
				if (i >= len || qi > 3) { push_curr(ik); last_qe = ik.qe; end_forward(); break; }
				in = ik; is_back = 0; qc = 3 - qi;
				if (TAB) { code = code << 2 | (u32)qi; const int L = i + 1 - x; if (L <= tabK) win |= (u32)qi << (2 * (tabK - L)); }
				qnext = base_at(i + 1);
				return true;
			case BWD:
				if (j >= n_prev) { // one backward step done for the whole set
					if (n_curr == 0) { end_smem1(); break; }
					prev_id ^= 1; n_prev = n_curr; rev = 0;
					--i; j = 0; n_curr = 0;
					if (i < -1) { end_smem1(); break; }
					c = cnext;
					if (TAB) win = (win >> 2) | (u32)(c < 0 ? 0 : c) << (2 * (tabK - 1));
					{ const int b1 = base_at(i - 1); cnext = b1 < 4 ? b1 : -1; }
					break;
				}
				in = prev_entry(j);
				if (c < 0) { keep(in); ++j; break; }
				is_back = 1; qc = c;
				return true;
			case S3:
				if (!P3) return false;
				if (i >= len) { x = len; state = NEXT_P3; break; }
				if (qi > 3) { x = i + 1; state = NEXT_P3; break; }
				in = ik; is_back = 0; qc = 3 - qi;
				qnext = base_at(i + 1);
				return true;
			}
		}
	}
	// TAB: the query advance() has just set up, answered from the k-mer table when the string it produces is short enough
	SSQ_HD bool table_hit(const DevIndex &ix, I &okc) const
	{
		if (!TAB || tabK == 0) return false;
		int L; u32 cd;
		if (state == FWD) { L = i + 1 - x; if (L > tabK) return false; cd = code; }
		else if (state == BWD) { L = (int)in.qe - i; if (L > tabK) return false; cd = win >> (2 * (tabK - L)); }
		else return false;
		const Intv32 t = kmer_lookup(ix, L, cd);
		okc.x0 = (U)t.x0; okc.x1 = (U)t.x1; okc.x2 = (U)t.x2; okc.qb = okc.qe = 0;
		return true;
	}
	SSQ_HD void post(const I &okc) // okc = ok[qc] of the query
	{
		if (state == FWD) {
			if (okc.x2 != ik.x2) {
				push_curr(ik); last_qe = ik.qe;
				if (okc.x2 < min_intv) { end_forward(); return; }
			}
			ik = okc; ik.qe = (u32)(i + 1);
			++i; qi = qnext;
		} else if (state == BWD) {
			if (okc.x2 < min_intv) keep(in);
			else if (n_curr == 0 || okc.x2 != curr_tail_x2) { I t = okc; t.qb = 0; t.qe = in.qe; push_curr(t); }
			++j;
		} else if (P3) { // S3
			if (okc.x2 < max_mem_intv && i - x >= min_seed_len) {
				Intv m = widen(okc); m.qb = (u32)x; m.qe = (u32)(i + 1);
				if (m.x2 > 0) { if (n >= mem_cap) { err = 1; return; } mem[n++] = m; }
				x = i + 1; state = NEXT_P3;
			} else { ik = okc; ++i; qi = qnext; }
		}
	}
	// order by (qb,qe): only 4-byte keys (qb | qe | slot) move, the 32-byte records are gathered once when the caller
	// copies them out through key & 0xffff.  keys[] needs n entries.  returns the interval count.
	SSQ_HD int finish(u32 *keys)
	{
		if (err) return 0;
		for (int a = 0; a < n; ++a) {
			const u32 key = mem[a].qb << 24 | mem[a].qe << 16 | (u32)a; // qb,qe <= 255, a < 65536
			int k;
			for (k = a; k > 0 && (keys[k - 1] >> 16) > (key >> 16); --k) keys[k] = keys[k - 1];
			keys[k] = key;
		}
		return n;
	}
};

// The backward phase of one smem1() call on its own (phase-split seeding, 32-bit rows): the part of SmemMachineT that a lane of
// k_smem_bwd2 needs and nothing else (~35 words of state instead of ~58).  Same operations in the same order as the machine's
// BWD state: sweep the previous list (the call's forward list, read from its end, in the first sweep) one backward extension per
// entry; an entry whose extension falls below min_intv is left-maximal (keep), one whose extended size differs from the last one
// pushed survives into the next sweep.
template <class Lists>
struct BwdCallT {
	const uint8_t *q; Intv *mem; Lists L; const FwdEntry *ext;
	int len, n, i, j, c, cnext, n_prev, n_curr, prev_id, rev, any_kept, err, mem_cap, min_seed_len;
	u32 last_mem_qb, curr_tail_x2, min_intv;
	u32 win; int K; // k-mer table in use (K > 0): the K bases from position i on, first base in the top bits (N / beyond the read = 0: never part of a string looked up)
	Intv32 in;
	SSQ_HD int base_at(int p) const { return p >= 0 && p < len ? (int)q[p] : 4; }
	SSQ_HD void start(const ssq_opts_t &opt, int len_, const uint8_t *q_, Intv *mem_, int mem_cap_, const Lists &lists, int x, u32 min_intv_,
	                  const FwdEntry *list, int list_n, int b0, int b1)
	{
		q = q_; len = len_; mem = mem_; mem_cap = mem_cap_; L = lists; ext = list; min_seed_len = opt.min_seed_len;
		n = 0; err = 0; any_kept = 0; min_intv = min_intv_ < 1 ? 1 : min_intv_;
		n_prev = list_n; rev = 1; prev_id = 0; i = x - 1; j = 0; n_curr = 0;
		c = b0 < 4 ? b0 : -1; cnext = b1 < 4 ? b1 : -1;
		last_mem_qb = 0; curr_tail_x2 = 0;
		K = 0; win = 0;
	}
	SSQ_HD void use_table(int K_) // after start(): window over positions i .. i+K-1
	{
		K = K_; win = 0;
		for (int t = 0; t < K; ++t) { const int b = base_at(i + t); win = win << 2 | (u32)(b < 4 ? b : 0); }
	}
	// the query advance() has set up, answered from the table when the string it produces (q[i .. in.qe)) is short enough
	SSQ_HD bool table_hit(const DevIndex &ix, Intv32 &okc) const
	{
		const int L = (int)in.qe - i;
		if (K == 0 || L > K) return false;
		okc = kmer_lookup(ix, L, win >> (2 * (K - L)));
		return true;
	}
	SSQ_HD Intv32 entry(int jj) const
	{
		if (rev) { const FwdEntry e = ext[n_prev - 1 - jj]; Intv32 r; r.x0 = e.x0; r.x1 = e.x1; r.x2 = e.x2; r.qb = 0; r.qe = e.qe; return r; }
		return L.get(prev_id, jj);
	}
	SSQ_HD void keep(const Intv32 &p_)
	{
		if (n_curr == 0 && (!any_kept || (u32)(i + 1) < last_mem_qb)) {
			any_kept = 1; last_mem_qb = (u32)(i + 1);
			if ((int)p_.qe - (i + 1) >= min_seed_len) {
				if (n >= mem_cap) { err = 1; return; }
				Intv p = widen(p_); p.qb = (u32)(i + 1);
				mem[n++] = p;
			}
		}
	}
	// true: extend `in` backwards by base c (only that base's interval is needed); false: the call is complete, mem[0..n) is its output
	SSQ_HD bool advance()
	{
		for (;;) {
			if (err) return false;
			if (j >= n_prev) { // one backward step done for the whole set
				if (n_curr == 0) return false;
				prev_id ^= 1; n_prev = n_curr; rev = 0;
				--i; j = 0; n_curr = 0;
				if (i < -1) return false;
				c = cnext;
				if (K) win = (win >> 2) | (u32)(c < 0 ? 0 : c) << (2 * (K - 1)); // the base at the new i enters at the top, the last one leaves
				{ const int b1 = base_at(i - 1); cnext = b1 < 4 ? b1 : -1; }
			}
			in = entry(j);
			if (c < 0) { keep(in); ++j; continue; }
			return true;
		}
	}
	SSQ_HD void post(const Intv32 &okc)
	{
		if (okc.x2 < min_intv) keep(in);
		else if (n_curr == 0 || okc.x2 != curr_tail_x2) { Intv32 t = okc; t.qb = 0; t.qe = in.qe; L.set(prev_id ^ 1, n_curr++, t); curr_tail_x2 = t.x2; }
		++j;
	}
};

// number of SA look-ups an interval contributes (max_occ rows, evenly strided when it has more)
SSQ_HD int intv_occ_count(u64 s, int max_occ, u64 &step)
{
	step = s > (u64)max_occ ? s / max_occ : 1;
	u64 cnt = (s + step - 1) / step;
	return (int)(cnt < (u64)max_occ ? cnt : (u64)max_occ);
}

// ------------------------------------------------------------------------- SA look-up ----
SSQ_HD u64 sa_lookup(ScalarFm &fm, u64 k, unsigned long long &n_sa, bool use_dense = true)
{
	const DevIndex &ix = fm.ix;
	const bool dense = use_dense && ix.sad_intv > 0;
	const u64 intv = dense ? (u64)ix.sad_intv : (u64)ix.sa_intv;
	u64 sa = 0, mask = intv - 1;
	while (k & mask) { // walk LF until a sampled row
		++sa;
		if (k == ix.primary) { k = 0; continue; }
		u64 x = k - (k > ix.primary);
		int c;
		u64 cnt[4];
		if (ix.bwt32) { // symbol of row x and the counts up to row k come from the same 32-byte block (x == k - (k >= primary) here): one load
			const Blk32 b = load_blk32(ix.bwt32 + ((x >> 6) << 3));
			const int wsel = (int)(x & 0x3f) >> 4;
			const u32 wv = wsel == 0 ? b.w0 : wsel == 1 ? b.w1 : wsel == 2 ? b.w2 : b.w3;
			c = wv >> ((~x & 0xf) << 1) & 3;
			++fm.n_blk;
			blk32_count(b, x, cnt);
			k = ix.L2[c] + SSQ_SEL4(cnt[0], cnt[1], cnt[2], cnt[3], c);
			continue;
		}
		{ const u32 *p = ix.bwt + ((x >> 7) << 4) + 8; c = p[(x & 0x7f) >> 4] >> ((~x & 0xf) << 1) & 3; }
		fm.occ4(k, cnt);
		k = ix.L2[c] + cnt[c];
	}
	++n_sa;
	if (dense) {
		if (ix.sad32) { const u32 v = ix.sad32[k / intv]; return sa + (v == 0xffffffffu ? (u64)-1 : (u64)v); }
		return sa + ix.sad64[k / intv];
	}
	return sa + ix.sa[k / intv];
}

// ------------------------------------------------------------------- reference helpers ----
SSQ_HD int pos2rid(const DevIndex &ix, i64 pos_f)
{
	int left = 0, mid = 0, right = ix.n_seqs;
	if (pos_f >= ix.l_pac) return -1;
	while (left < right) {
		mid = (left + right) >> 1;
		if (pos_f >= ix.ann_off[mid]) {
			if (mid == ix.n_seqs - 1) break;
			if (pos_f < ix.ann_off[mid + 1]) break;
			left = mid + 1;
		} else right = mid;
	}
	return mid;
}
SSQ_HD i64 depos(const DevIndex &ix, i64 pos, int &is_rev) { is_rev = pos >= ix.l_pac; return is_rev ? (ix.l_pac << 1) - 1 - pos : pos; }
SSQ_HD int intv2rid(const DevIndex &ix, i64 rb, i64 re)
{
	int is_rev, rid_b, rid_e;
	if (rb < ix.l_pac && re > ix.l_pac) return -2;
	rid_b = pos2rid(ix, depos(ix, rb, is_rev));
	rid_e = rb < re ? pos2rid(ix, depos(ix, re - 1, is_rev)) : rid_b;
	return rid_b == rid_e ? rid_b : -1;
}
// base at coordinate p of the doubled (forward + reverse-complement) reference
SSQ_HD int ref_base(const DevIndex &ix, i64 p)
{
	if (p >= ix.l_pac) { i64 f = (ix.l_pac << 1) - 1 - p; return 3 - (ix.pac[f >> 2] >> ((~f & 3) << 1) & 3); }
	return ix.pac[p >> 2] >> ((~p & 3) << 1) & 3;
}
SSQ_HD int cal_max_gap(const ssq_opts_t &o, int qlen)
{
	int l_del = (int)((double)(qlen * o.a - o.o_del) / o.e_del + 1.);
	int l_ins = (int)((double)(qlen * o.a - o.o_ins) / o.e_ins + 1.);
	int l = l_del > l_ins ? l_del : l_ins;
	l = l > 1 ? l : 1;
	return l < o.w << 1 ? l : o.w << 1;
}

// ---------------------------------------------------------------------------- chaining ----
struct Seed { i64 rbeg; i32 qbeg, len; };
struct ChainRec { // chain under construction / after the filter
	i64 pos, first_r, last_r;
	i32 first_q, last_q, last_len, rid, n, w, first, kept, seed_start;
	float frac_rep;
};

// klib-style introsort restated on (key, payload) pairs, comparisons on key only ("a before b" iff LT(a,b));
// the order it leaves equal keys in is part of the reference's behaviour (see oracle/ssqo_sort.h)
template <class T, class LT>
SSQ_HD void ks_isort(T *a, long lo, long hi, LT lt)
{
	for (long i = lo + 1; i < hi; ++i)
		for (long j = i; j > lo && lt(a[j], a[j - 1]); --j) { T t = a[j]; a[j] = a[j - 1]; a[j - 1] = t; }
}
template <class T, class LT>
SSQ_HD void ks_combsort(T *a, long n, LT lt)
{
	const double shrink = 1.2473309501039786540366528676643;
	int swapped;
	long gap = n;
	do {
		if (gap > 2) { gap = (long)(gap / shrink); if (gap == 9 || gap == 10) gap = 11; }
		swapped = 0;
		for (long i = 0; i < n - gap; ++i)
			if (lt(a[i + gap], a[i])) { T t = a[i]; a[i] = a[i + gap]; a[i + gap] = t; swapped = 1; }
	} while (swapped || gap > 2);
	if (gap != 1) ks_isort(a, 0, n, lt);
}
template <class T, class LT>
SSQ_HD void ks_introsort(long n, T *a, LT lt)
{
	long s, t, i, j, k, top = 0;
	int d;
	long stl[64], str[64]; int std_[64];
	if (n < 1) return;
	if (n == 2) { if (lt(a[1], a[0])) { T x = a[0]; a[0] = a[1]; a[1] = x; } return; }
	for (d = 2; (1L << d) < n; ++d);
	s = 0; t = n - 1; d <<= 1;
	for (;;) {
		if (s < t) {
			T rp, x;
			if (--d == 0) { ks_combsort(a + s, t - s + 1, lt); t = s; continue; }
			i = s; j = t; k = i + ((j - i) >> 1) + 1;
			if (lt(a[k], a[i])) { if (lt(a[k], a[j])) k = j; }
			else k = lt(a[j], a[i]) ? i : j;
			rp = a[k];
			if (k != t) { x = a[k]; a[k] = a[t]; a[t] = x; }
			for (;;) {
				do ++i; while (lt(a[i], rp));
				do --j; while (i <= j && lt(rp, a[j]));
				if (j <= i) break;
				x = a[i]; a[i] = a[j]; a[j] = x;
			}
			x = a[i]; a[i] = a[t]; a[t] = x;
			if (i - s > t - i) {
				if (i - s > 16) { stl[top] = s; str[top] = i - 1; std_[top] = d; ++top; }
				s = t - i > 16 ? i + 1 : t;
			} else {
				if (t - i > 16) { stl[top] = i + 1; str[top] = t; std_[top] = d; ++top; }
				t = i - s > 16 ? i - 1 : s;
			}
		} else {
			if (top == 0) { ks_isort(a, 0, n, lt); return; }
			--top; s = stl[top]; t = str[top]; d = std_[top];
		}
	}
}

struct WIdx { i32 w, idx; };
struct KeptChain { i32 b, e, w, i; }; // query span, weight and sorted rank of a chain that survived the overlap filter so far
struct WIdxLt { SSQ_HD bool operator()(const WIdx &a, const WIdx &b) const { return a.w > b.w; } };

// Build the chains of one read from its seeds (in look-up order) and filter them.
//   seeds[0..n)      in : seeds of the read (rbeg from the SA look-up, qbeg/len from their interval)
//   chain_of[0..n)   scratch: chain index of each seed, -1 = dropped/absorbed
//   ch[0..n)         scratch: chain records (at most one chain per seed)
//   ord[0..n)        scratch: chain indices ordered by pos
//   sorted[0..n)     out: seeds regrouped chain by chain (chain order = filter order)
//   outc[0..n)       out: kept chains (seed_start relative to `sorted`)
// add_seed() is the per-seed step of mem_chain()'s loop (one call per seed, in order); finish() does the regrouping, the
// weights, the sort and the overlap filter and returns the number of kept chains.  On the GPU a lane keeps one ChainBuilder
// and all lanes of a warp meet at add_seed(), so a read with hundreds of seeds does not idle its 31 neighbours.
struct ChainBuilder {
	const Seed *seeds; i32 *chain_of; ChainRec *ch; i32 *ord; WIdx *wi; Seed *sorted; ChainRec *outc; KeptChain *kp;
	int n, n_ch, len, l_rep;

	SSQ_HD void init(int len_, int n_, const Seed *seeds_, int l_rep_, i32 *chain_of_, ChainRec *ch_, i32 *ord_, WIdx *wi_, Seed *sorted_, ChainRec *outc_, KeptChain *kp_)
	{
		len = len_; n = n_; seeds = seeds_; l_rep = l_rep_; chain_of = chain_of_; ch = ch_; ord = ord_; wi = wi_; sorted = sorted_; outc = outc_; kp = kp_; n_ch = 0; root = -1;
	}
	// Chains are kept in the order of `pos` (rbeg of their first seed).  The reference does it with a B-tree; the oracle restates
	// its look-up / insert on one ordered sequence: look-up = the first chain whose key equals pos, else the last chain with a
	// smaller key; a new chain goes directly after the slot the look-up returned.  Here the same order is kept by an index-based
	// binary search tree (left/right children in wi[].w / wi[].idx, which are free until finish()) on the composite key
	// (pos, tie) with tie = INT_MIN for the first chain of a pos and -index for later ones — exactly the order "first, then the
	// others newest first" that repeated insert-after-the-first produces.  Expected O(log n) per seed instead of O(n) shifts.
	int root;
	SSQ_HD void add_seed(const DevIndex &ix, const ssq_opts_t &opt, int i)
	{
		const i64 l_pac = ix.l_pac;
		const Seed s = seeds[i];
		const int rid = intv2rid(ix, s.rbeg, s.rbeg + s.len);
		chain_of[i] = -1;
		if (rid < 0) return;
		int slot = -1, exact = 0, merged = 0;
		for (int cur = n_ch ? root : -1; cur >= 0;) { // look-up
			const i64 p = ch[cur].pos;
			if (p < s.rbeg) { slot = cur; cur = wi[cur].idx; }
			else if (p > s.rbeg) cur = wi[cur].w;
			else if (ch[cur].w == (i32)0x80000000) { slot = cur; exact = 1; break; } // the first chain with this pos
			else cur = wi[cur].w;
		}
		if (slot >= 0) {
			ChainRec &c = ch[slot];
			i64 qend = c.last_q + c.last_len, rend = c.last_r + c.last_len;
			if (rid == c.rid) {
				if (s.qbeg >= c.first_q && s.qbeg + s.len <= qend && s.rbeg >= c.first_r && s.rbeg + s.len <= rend) merged = 1; // contained
				else if (!((c.last_r < l_pac || c.first_r < l_pac) && s.rbeg >= l_pac)) {
					i64 x = s.qbeg - c.last_q, y = s.rbeg - c.last_r;
					if (y >= 0 && x - y <= opt.w && y - x <= opt.w && x - c.last_len < opt.max_chain_gap && y - c.last_len < opt.max_chain_gap) {
						c.last_q = s.qbeg; c.last_r = s.rbeg; c.last_len = s.len; ++c.n;
						chain_of[i] = slot;
						merged = 1;
					}
				}
			}
		}
		if (!merged) {
			const int nn = n_ch;
			ChainRec &c = ch[nn];
			c.pos = s.rbeg; c.first_r = c.last_r = s.rbeg; c.first_q = c.last_q = s.qbeg; c.last_len = s.len;
			c.rid = rid; c.n = 1; c.first = -1; c.kept = 0; c.seed_start = 0; c.frac_rep = 0.f;
			c.w = exact ? -nn : (i32)0x80000000; // tie component of the key
			wi[nn].w = wi[nn].idx = -1;
			if (nn == 0) root = 0;
			else {
				for (int cur = root;;) {
					const i64 p = ch[cur].pos;
					const bool go_left = s.rbeg < p || (s.rbeg == p && c.w < ch[cur].w);
					i32 &child = go_left ? wi[cur].w : wi[cur].idx;
					if (child < 0) { child = nn; break; }
					cur = child;
				}
			}
			chain_of[i] = nn;
			++n_ch;
		}
	}
	// in-order traversal without a stack (threads the tree through the right links and restores them): ord[] = chains by key
	SSQ_HD void inorder()
	{
		int k = 0, cur = n_ch ? root : -1;
		while (cur >= 0) {
			if (wi[cur].w < 0) { ord[k++] = cur; cur = wi[cur].idx; }
			else {
				int pre = wi[cur].w;
				while (wi[pre].idx >= 0 && wi[pre].idx != cur) pre = wi[pre].idx;
				if (wi[pre].idx < 0) { wi[pre].idx = cur; cur = wi[cur].w; }
				else { wi[pre].idx = -1; ord[k++] = cur; cur = wi[cur].idx; }
			}
		}
	}
	SSQ_HD int finish(const ssq_opts_t &opt)
	{
		int i, k;
		if (n_ch == 0) return 0;
		inorder();
		// regroup seeds chain by chain, chains in pos order (= the order the reference's tree is traversed)
		{
			int off = 0;
			for (k = 0; k < n_ch; ++k) { ChainRec &c = ch[ord[k]]; c.seed_start = off; off += c.n; c.n = 0; }
			for (i = 0; i < n; ++i) if (chain_of[i] >= 0) { ChainRec &c = ch[chain_of[i]]; sorted[c.seed_start + c.n++] = seeds[i]; }
		}
		// weight = min(query coverage, reference coverage) of the seeds
		for (k = 0; k < n_ch; ++k) {
			ChainRec &c = ch[ord[k]];
			const Seed *s = sorted + c.seed_start;
			i64 end; int j, w = 0, tmp;
			for (j = 0, end = 0; j < c.n; ++j) {
				if (s[j].qbeg >= end) w += s[j].len; else if (s[j].qbeg + s[j].len > end) w += (int)(s[j].qbeg + s[j].len - end);
				end = end > s[j].qbeg + s[j].len ? end : s[j].qbeg + s[j].len;
			}
			tmp = w; w = 0;
			for (j = 0, end = 0; j < c.n; ++j) {
				if (s[j].rbeg >= end) w += s[j].len; else if (s[j].rbeg + s[j].len > end) w += (int)(s[j].rbeg + s[j].len - end);
				end = end > s[j].rbeg + s[j].len ? end : s[j].rbeg + s[j].len;
			}
			w = w < tmp ? w : tmp;
			c.w = w < 1 << 30 ? w : (1 << 30) - 1;
			c.first = -1; c.kept = 0;
			c.frac_rep = (float)l_rep / len;
			wi[k].w = c.w; wi[k].idx = ord[k];
		}
		ks_introsort((long)n_ch, wi, WIdxLt());
		// pairwise overlap filter over chains in decreasing weight.  The inner loop runs over the kept chains only through the
		// compact list kp[] (begin, end, weight, rank) — one sequential 16-byte load per pair instead of a chain of dependent
		// look-ups; a chain's query span comes from the fields kept while it was built (first seed's qbeg, last seed's end).
#define CH(i_) ch[wi[i_].idx]
		int n_kept = 0;
		{
			ChainRec &c0 = CH(0);
			c0.kept = 3;
			kp[0].b = c0.first_q; kp[0].e = c0.last_q + c0.last_len; kp[0].w = c0.w; kp[0].i = 0; n_kept = 1;
		}
		for (i = 1; i < n_ch; ++i) {
			int large_ovlp = 0;
			ChainRec &ci = CH(i);
			const int bi = ci.first_q, ei = ci.last_q + ci.last_len, wi_ = ci.w;
			for (k = 0; k < n_kept; ++k) {
				const KeptChain kj = kp[k];
				const int b_max = kj.b > bi ? kj.b : bi, e_min = kj.e < ei ? kj.e : ei;
				if (e_min > b_max) {
					const int li = ei - bi, lj = kj.e - kj.b, min_l = li < lj ? li : lj;
					if (e_min - b_max >= min_l * opt.mask_level && min_l < opt.max_chain_gap) {
						large_ovlp = 1;
						ChainRec &cj = CH(kj.i);
						if (cj.first < 0) cj.first = i;
						if (wi_ < kj.w * opt.drop_ratio && kj.w - wi_ >= opt.min_seed_len << 1) break;
					}
				}
			}
			if (k == n_kept) { kp[n_kept].b = bi; kp[n_kept].e = ei; kp[n_kept].w = wi_; kp[n_kept].i = i; ++n_kept; ci.kept = large_ovlp ? 2 : 3; }
		}
		for (i = 0; i < n_kept; ++i) { ChainRec &c = CH(kp[i].i); if (c.first >= 0) CH(c.first).kept = 1; }
		for (i = k = 0; i < n_ch; ++i) {
			if (CH(i).kept == 0 || CH(i).kept == 3) continue;
			if (++k >= opt.max_chain_extend) break;
		}
		for (; i < n_ch; ++i) if (CH(i).kept < 3) CH(i).kept = 0;
		for (i = k = 0; i < n_ch; ++i) if (CH(i).kept) outc[k++] = CH(i);
#undef CH
		return k;
	}
};

SSQ_HD int chain_and_filter(const DevIndex &ix, const ssq_opts_t &opt, int len, int n, const Seed *seeds, int l_rep,
                            i32 *chain_of, ChainRec *ch, i32 *ord, WIdx *wi, Seed *sorted, ChainRec *outc, KeptChain *kp)
{
	ChainBuilder b;
	b.init(len, n, seeds, l_rep, chain_of, ch, ord, wi, sorted, outc, kp);
	for (int i = 0; i < n; ++i) b.add_seed(ix, opt, i);
	return b.finish(opt);
}

// ----------------------------------------------------------------- banded SW extension ----
// ksw_extend2 semantics: row-sequential DP with per-row band trimming and z-drop (the trimming makes
// the result differ from an untrimmed band, so the evaluation order is part of the contract).
// Q(j) / T(i) fetch the j-th query and i-th target base of this extension (0..4).
// eh is a strided array of packed cells: low 16 bits = H, high 16 bits = E (both 0..32767).
struct EhAcc {
	u32 *base; int stride;
	SSQ_HD u32 get(int j) const { return base[(size_t)j * stride]; }
	SSQ_HD void set(int j, u32 v) const { base[(size_t)j * stride] = v; }
};

// PQ: the query base of column j rides in bits 29..31 of column j's word (H in bits 0..12, E in bits 16..28), so the inner loop reads
// nothing but that one word per cell — no per-cell query fetch from global memory.  Valid when no score can reach 2^13.
template <bool PQ, class QF, class TF>
SSQ_HD int sw_extend_impl(const ssq_opts_t &o, int qlen, QF Q, int tlen, TF T, int w, int end_bonus, int zdrop, int h0, const EhAcc &eh,
                          int &qle, int &tle, int &gtle, int &gscore_, int &max_off_, unsigned long long &cells)
{
	const int o_del = o.o_del, e_del = o.e_del, o_ins = o.o_ins, e_ins = o.e_ins;
	const int oe_del = o_del + e_del, oe_ins = o_ins + e_ins;
	const u32 QMASK = PQ ? 0xe0000000u : 0u, VMASK = ~QMASK;
	int i, j, beg, end, max, max_i, max_j, max_ins, max_del, max_ie, gscore, max_off;
	auto qbits = [&](int jj) -> u32 { return PQ && jj < qlen ? (u32)Q(jj) << 29 : 0u; };
	// row -1
	eh.set(0, (u32)h0 | qbits(0));
	{
		int h = h0 > oe_ins ? h0 - oe_ins : 0;
		if (qlen >= 1) eh.set(1, (u32)h | qbits(1));
		for (j = 2; j <= qlen && h > e_ins; ++j) { h -= e_ins; eh.set(j, (u32)h | qbits(j)); }
		for (; j <= qlen; ++j) eh.set(j, qbits(j));
	}
	max = o.a; // largest matrix entry is the match score
	max_ins = (int)((double)(qlen * max + end_bonus - o_ins) / e_ins + 1.);
	max_ins = max_ins > 1 ? max_ins : 1;
	w = w < max_ins ? w : max_ins;
	max_del = (int)((double)(qlen * max + end_bonus - o_del) / e_del + 1.);
	max_del = max_del > 1 ? max_del : 1;
	w = w < max_del ? w : max_del;
	max = h0; max_i = max_j = -1; max_ie = -1; gscore = -1; max_off = 0;
	beg = 0; end = qlen;
	for (i = 0; i < tlen; ++i) {
		int f = 0, h1, m = 0, mj = -1, t;
		const int tb = T(i);
		if (beg < i - w) beg = i - w;
		if (end > i + w + 1) end = i + w + 1;
		if (end > qlen) end = qlen;
		if (beg == 0) { h1 = h0 - (o_del + e_del * (i + 1)); if (h1 < 0) h1 = 0; } else h1 = 0;
		// the row's substitution scores for query bases 0..4, one byte each (the target base is fixed along a row)
		u64 sctab = 0;
		for (int qb = 0; qb < 5; ++qb) sctab |= (u64)(uint8_t)(int8_t)((qb > 3 || tb > 3) ? -1 : (qb == tb ? o.a : -o.b)) << (8 * qb);
		// row maximum and its column in one word: (h << 16 | column + 1) — equal maxima keep the LATER column, as the reference's
		// `mj = m > h ? mj : j` does; used in the packed form only (h < 2^13 there)
		int mpk = 0;
		// one cell: consumes the packed (H(i-1,j-1), E(i,j)) word of column j, leaves (H(i,j-1), E(i+1,j)) there
		auto cell = [&](const u32 p, const int qb, const int jj) {
			int M = (int)(p & 0xffffu), e = (int)((p & VMASK) >> 16), h;
			const int sc = (int)(int8_t)(sctab >> (8 * qb));
			M = M ? M + sc : 0;
			h = ssq_max3(M, e, f);
			if (PQ) mpk = ssq_max2(mpk, h << 16 | (jj + 1)); else { mj = m > h ? mj : jj; m = m > h ? m : h; }
			e = ssq_max3(e - e_del, M - oe_del, 0);
			eh.set(jj, (u32)h1 | (u32)e << 16 | (p & QMASK));
			h1 = h;
			f = ssq_max3(f - e_ins, M - oe_ins, 0);
		};
		// four columns per trip: their row-state words are fetched before the first of them is rewritten (column j's store does
		// not touch columns j+1..j+3), so the loads overlap the dependent arithmetic of the cells
		for (j = beg; j + 4 <= end; j += 4) {
			const u32 p0 = eh.get(j), p1 = eh.get(j + 1), p2 = eh.get(j + 2), p3 = eh.get(j + 3);
			if (PQ) { cell(p0, (int)(p0 >> 29), j); cell(p1, (int)(p1 >> 29), j + 1); cell(p2, (int)(p2 >> 29), j + 2); cell(p3, (int)(p3 >> 29), j + 3); }
			else {
				const int q0 = Q(j), q1 = Q(j + 1), q2 = Q(j + 2), q3 = Q(j + 3);
				cell(p0, q0, j); cell(p1, q1, j + 1); cell(p2, q2, j + 2); cell(p3, q3, j + 3);
			}
		}
		for (; j < end; ++j) { const u32 p = eh.get(j); cell(p, PQ ? (int)(p >> 29) : Q(j), j); }
		if (PQ) { m = mpk >> 16; mj = (mpk & 0xffff) - 1; }
		(void)t;
		cells += (unsigned long long)(end > beg ? end - beg : 0);
		eh.set(end, PQ ? ((u32)h1 | (eh.get(end) & QMASK)) : (u32)h1);
		if (j == qlen) { max_ie = gscore > h1 ? max_ie : i; gscore = gscore > h1 ? gscore : h1; }
		if (m == 0) break;
		if (m > max) {
			max = m; max_i = i; max_j = mj;
			int d = mj - i; d = d < 0 ? -d : d;
			max_off = max_off > d ? max_off : d;
		} else if (zdrop > 0) {
			if (i - max_i > mj - max_j) { if (max - m - ((i - max_i) - (mj - max_j)) * e_del > zdrop) break; }
			else { if (max - m - ((mj - max_j) - (i - max_i)) * e_ins > zdrop) break; }
		}
		for (j = beg; j < end && (eh.get(j) & VMASK) == 0; ++j);
		beg = j;
		for (j = end; j >= beg && (eh.get(j) & VMASK) == 0; --j);
		end = j + 2 < qlen ? j + 2 : qlen;
	}
	qle = max_j + 1; tle = max_i + 1; gtle = max_ie + 1; gscore_ = gscore; max_off_ = max_off;
	return max;
}
template <class QF, class TF>
SSQ_HD int sw_extend(const ssq_opts_t &o, int qlen, QF Q, int tlen, TF T, int w, int end_bonus, int zdrop, int h0, const EhAcc &eh,
                     int &qle, int &tle, int &gtle, int &gscore_, int &max_off_, unsigned long long &cells)
{
	if ((long long)h0 + (long long)qlen * o.a < 8192) // no H or E can exceed h0 + qlen * a
		return sw_extend_impl<true>(o, qlen, Q, tlen, T, w, end_bonus, zdrop, h0, eh, qle, tle, gtle, gscore_, max_off_, cells);
	return sw_extend_impl<false>(o, qlen, Q, tlen, T, w, end_bonus, zdrop, h0, eh, qle, tle, gtle, gscore_, max_off_, cells);
}

// One alignment-region candidate per seed of a kept chain: left then right extension (h0 of the right one is
// the left score), up to two band widths each — mem_chain2aln()'s body for a single seed.
struct RegCand { // == ssq_alnreg_t minus read_id bookkeeping
	i64 rb, re;
	i32 qb, qe, rid, score, truesc, w, seedcov, seedlen0;
	float frac_rep;
};

SSQ_HD void chain_window(const DevIndex &ix, const ssq_opts_t &opt, int l_query, const Seed *cs, int n, i64 &rmax0, i64 &rmax1)
{
	const i64 l_pac = ix.l_pac;
	rmax0 = l_pac << 1; rmax1 = 0;
	for (int i = 0; i < n; ++i) {
		i64 b = cs[i].rbeg - (cs[i].qbeg + cal_max_gap(opt, cs[i].qbeg));
		i64 e = cs[i].rbeg + cs[i].len + ((l_query - cs[i].qbeg - cs[i].len) + cal_max_gap(opt, l_query - cs[i].qbeg - cs[i].len));
		rmax0 = rmax0 < b ? rmax0 : b;
		rmax1 = rmax1 > e ? rmax1 : e;
	}
	rmax0 = rmax0 > 0 ? rmax0 : 0;
	rmax1 = rmax1 < l_pac << 1 ? rmax1 : l_pac << 1;
	if (rmax0 < l_pac && l_pac < rmax1) { if (cs[0].rbeg < l_pac) rmax1 = l_pac; else rmax0 = l_pac; }
	// clamp to the contig holding the chain (bns_fetch_seq)
	int is_rev;
	int rid = pos2rid(ix, depos(ix, cs[0].rbeg, is_rev));
	i64 far_beg = ix.ann_off[rid], far_end = far_beg + ix.ann_len[rid];
	if (is_rev) { i64 t = far_beg; far_beg = (l_pac << 1) - far_end; far_end = (l_pac << 1) - t; }
	rmax0 = rmax0 > far_beg ? rmax0 : far_beg;
	rmax1 = rmax1 < far_end ? rmax1 : far_end;
}

// ---- mem_chain2aln()'s per-seed body, cut into pieces so that the GPU can run all left extensions, then all right
// ---- extensions, each as size-sorted passes; extend_seed() below is the straight composition of the same pieces
struct ExtInfo { i64 rmax0, rmax1, rbeg; i32 qbeg, len, lq, rid; }; // geometry of one seed's extension problem
struct ExtRes { i32 score, qle, tle, gtle, gscore, max_off; };

SSQ_HD void ext_prep(const DevIndex &ix, const ssq_opts_t &opt, int l_query, const ChainRec &c, const Seed *cs, int si, ExtInfo &e)
{
	chain_window(ix, opt, l_query, cs, c.n, e.rmax0, e.rmax1);
	e.rbeg = cs[si].rbeg; e.qbeg = cs[si].qbeg; e.len = cs[si].len; e.lq = l_query; e.rid = c.rid;
}
SSQ_HD int ext_left_qlen(const ExtInfo &e) { return e.qbeg; }
SSQ_HD int ext_left_tlen(const ExtInfo &e) { return (int)(e.rbeg - e.rmax0); }
SSQ_HD int ext_right_qlen(const ExtInfo &e) { return e.lq - (e.qbeg + e.len); }
SSQ_HD int ext_right_tlen(const ExtInfo &e) { return (int)(e.rmax1 - (e.rbeg + e.len)); }
SSQ_HD bool ext_needs_retry(const ssq_opts_t &opt, const ExtRes &r) { return r.max_off >= (opt.w >> 1) + (opt.w >> 2); } // implies the score moved

SSQ_HD void ext_left_run(const DevIndex &ix, const ssq_opts_t &opt, const uint8_t *query, const ExtInfo &e, int w, const EhAcc &eh, ExtRes &r, unsigned long long &cells)
{
	const uint8_t *qp = query + e.qbeg - 1;
	const i64 rp = e.rbeg - 1;
	r.score = sw_extend(opt, e.qbeg, [&](int j) { return (int)qp[-j]; }, ext_left_tlen(e), [&](int t) { return ref_base(ix, rp - t); },
	                    w, opt.pen_clip5, opt.zdrop, e.len * opt.a, eh, r.qle, r.tle, r.gtle, r.gscore, r.max_off, cells);
}
SSQ_HD void ext_right_run(const DevIndex &ix, const ssq_opts_t &opt, const uint8_t *query, const ExtInfo &e, int sc0, int w, const EhAcc &eh, ExtRes &r, unsigned long long &cells)
{
	const int qe = e.qbeg + e.len;
	const i64 re = e.rbeg + e.len;
	const uint8_t *qp = query + qe;
	r.score = sw_extend(opt, e.lq - qe, [&](int j) { return (int)qp[j]; }, ext_right_tlen(e), [&](int t) { return ref_base(ix, re + t); },
	                    w, opt.pen_clip3, opt.zdrop, sc0, eh, r.qle, r.tle, r.gtle, r.gscore, r.max_off, cells);
}
// after the left side: score / qb / rb / truesc (has_left == false: the seed starts the read)
SSQ_HD void ext_left_fin(const ssq_opts_t &opt, const ExtInfo &e, bool has_left, const ExtRes &r, RegCand &a)
{
	a.rid = e.rid;
	if (has_left) {
		a.score = r.score;
		if (r.gscore <= 0 || r.gscore <= r.score - opt.pen_clip5) { a.qb = e.qbeg - r.qle; a.rb = e.rbeg - r.tle; a.truesc = r.score; }
		else { a.qb = 0; a.rb = e.rbeg - r.gtle; a.truesc = r.gscore; }
	} else { a.score = a.truesc = e.len * opt.a; a.qb = 0; a.rb = e.rbeg; }
}
// after the right side: score / qe / re / truesc, then seed coverage and band bookkeeping
SSQ_HD void ext_right_fin(const ssq_opts_t &opt, const ExtInfo &e, bool has_right, const ExtRes &r, int aw0, int aw1, const ChainRec &c, const Seed *cs, RegCand &a)
{
	if (has_right) {
		const int sc0 = a.score, qe = e.qbeg + e.len;
		const i64 re = e.rbeg + e.len;
		a.score = r.score;
		if (r.gscore <= 0 || r.gscore <= r.score - opt.pen_clip3) { a.qe = qe + r.qle; a.re = re + r.tle; a.truesc += r.score - sc0; }
		else { a.qe = e.lq; a.re = re + r.gtle; a.truesc += r.gscore - sc0; }
	} else { a.qe = e.lq; a.re = e.rbeg + e.len; }
	a.seedcov = 0;
	for (int i = 0; i < c.n; ++i)
		if (cs[i].qbeg >= a.qb && cs[i].qbeg + cs[i].len <= a.qe && cs[i].rbeg >= a.rb && cs[i].rbeg + cs[i].len <= a.re) a.seedcov += cs[i].len;
	a.w = aw0 > aw1 ? aw0 : aw1;
	a.seedlen0 = e.len;
	a.frac_rep = c.frac_rep;
}

SSQ_HD void extend_seed(const DevIndex &ix, const ssq_opts_t &opt, int l_query, const uint8_t *query, const ChainRec &c, const Seed *cs,
                        int si, const EhAcc &eh, RegCand &a, Counters *cnt /* may be null */)
{
	ExtInfo e;
	ExtRes r;
	int aw0 = opt.w, aw1 = opt.w;
	unsigned long long cells = 0, calls = 0, bytes = 0;
	ext_prep(ix, opt, l_query, c, cs, si, e);
	const bool has_left = ext_left_qlen(e) > 0, has_right = ext_right_qlen(e) > 0;
	if (has_left) {
		ext_left_run(ix, opt, query, e, opt.w, eh, r, cells);
		++calls; bytes += (unsigned long long)e.qbeg + (ext_left_tlen(e) + 3) / 4 + 24;
		if (ext_needs_retry(opt, r)) { // second and last band width
			aw0 = opt.w << 1;
			ext_left_run(ix, opt, query, e, aw0, eh, r, cells);
			++calls; bytes += (unsigned long long)e.qbeg + (ext_left_tlen(e) + 3) / 4 + 24;
		}
	}
	ext_left_fin(opt, e, has_left, r, a);
	if (has_right) {
		const int sc0 = a.score;
		ext_right_run(ix, opt, query, e, sc0, opt.w, eh, r, cells);
		++calls; bytes += (unsigned long long)ext_right_qlen(e) + (ext_right_tlen(e) + 3) / 4 + 24;
		if (ext_needs_retry(opt, r)) {
			aw1 = opt.w << 1;
			ext_right_run(ix, opt, query, e, sc0, aw1, eh, r, cells);
			++calls; bytes += (unsigned long long)ext_right_qlen(e) + (ext_right_tlen(e) + 3) / 4 + 24;
		}
	}
	ext_right_fin(opt, e, has_right, r, aw0, aw1, c, cs, a);
	if (cnt) {
#ifdef __CUDA_ARCH__
		atomicAdd(&cnt->sw_calls, calls); atomicAdd(&cnt->sw_cells, cells); atomicAdd(&cnt->sw_bytes, bytes);
#else
		cnt->sw_calls += calls; cnt->sw_cells += cells; cnt->sw_bytes += bytes;
#endif
	}
}

// Replay of mem_chain2aln()'s seed loop for ONE chain with every seed's candidate already computed:
// walks the seeds from longest to shortest, skips those explained by an accepted region of this read
// (regions of earlier chains included), appends the rest to out[0..n_out).  With `have` flags the replay stops at the first
// seed it needs whose candidate is missing and returns its index (-1 = chain complete): the GPU extends seeds lazily, in rounds.
// The walk can also be RESUMED: srt[] (with the entries the walk zeroed) and out[] persist between rounds, so a later call with
// resume_k = the position it stopped at goes straight to accepting that seed, whose skip test it had already failed.
SSQ_HD int select_regions(const ssq_opts_t &opt, int l_query, const ChainRec &c, const Seed *cs, const RegCand *cand,
                          u64 *srt /* scratch c.n */, RegCand *out, int &n_out, const uint8_t *have = 0, int resume_k = -1, int *stop_k = 0)
{
	int i, k;
	if (resume_k >= 0) {
		k = resume_k;
		if (have && !have[(u32)srt[k]]) { if (stop_k) *stop_k = k; return (int)(u32)srt[k]; }
		out[n_out++] = cand[(u32)srt[k]];
		--k;
		goto walk;
	}
	for (i = 0; i < c.n; ++i) srt[i] = (u64)(u32)cs[i].len << 32 | (u32)i; // seed score == len
	if (c.n <= 24) { for (i = 1; i < c.n; ++i) { u64 t = srt[i]; for (k = i; k > 0 && srt[k - 1] > t; --k) srt[k] = srt[k - 1]; srt[k] = t; } } // keys are unique: any sort gives the reference order
	else { // heap sort, O(n log n) for the chains of repeat-rich reads
		const int n = c.n;
		for (int st = n / 2 - 1; st >= 0; --st) { int r = st; for (;;) { int ch_ = 2 * r + 1; if (ch_ >= n) break; if (ch_ + 1 < n && srt[ch_ + 1] > srt[ch_]) ++ch_; if (srt[r] >= srt[ch_]) break; u64 t = srt[r]; srt[r] = srt[ch_]; srt[ch_] = t; r = ch_; } }
		for (int e = n - 1; e > 0; --e) { u64 t = srt[0]; srt[0] = srt[e]; srt[e] = t; int r = 0; for (;;) { int ch_ = 2 * r + 1; if (ch_ >= e) break; if (ch_ + 1 < e && srt[ch_ + 1] > srt[ch_]) ++ch_; if (srt[r] >= srt[ch_]) break; u64 t2 = srt[r]; srt[r] = srt[ch_]; srt[ch_] = t2; r = ch_; } }
	}
	k = c.n - 1;
walk:
	for (; k >= 0; --k) {
		const Seed s = cs[(u32)srt[k]];
		for (i = 0; i < n_out; ++i) {
			const RegCand &p = out[i];
			i64 rd; int qd, w, max_gap;
			if (s.rbeg < p.rb || s.rbeg + s.len > p.re || s.qbeg < p.qb || s.qbeg + s.len > p.qe) continue;
			if (s.len - p.seedlen0 > .1 * l_query) continue;
			qd = s.qbeg - p.qb; rd = s.rbeg - p.rb;
			max_gap = cal_max_gap(opt, qd < rd ? qd : (int)rd);
			w = max_gap < p.w ? max_gap : p.w;
			if (qd - rd < w && rd - qd < w) break;
			qd = p.qe - (s.qbeg + s.len); rd = p.re - (s.rbeg + s.len);
			max_gap = cal_max_gap(opt, qd < rd ? qd : (int)rd);
			w = max_gap < p.w ? max_gap : p.w;
			if (qd - rd < w && rd - qd < w) break;
		}
		if (i < n_out) {
			for (i = k + 1; i < c.n; ++i) {
				if (srt[i] == 0) continue;
				const Seed t = cs[(u32)srt[i]];
				if (t.len < s.len * .95) continue;
				if (s.qbeg <= t.qbeg && s.qbeg + s.len - t.qbeg >= s.len >> 2 && t.qbeg - s.qbeg != t.rbeg - s.rbeg) break;
				if (t.qbeg <= s.qbeg && t.qbeg + t.len - s.qbeg >= s.len >> 2 && s.qbeg - t.qbeg != s.rbeg - t.rbeg) break;
			}
			if (i == c.n) { srt[k] = 0; continue; }
		}
		if (have && !have[(u32)srt[k]]) { if (stop_k) *stop_k = k; return (int)(u32)srt[k]; } // this seed's extension has not been computed yet: ask for it
		out[n_out++] = cand[(u32)srt[k]];
	}
	return -1;
}

// Resume point of one read's region selection between extension rounds (all zero = nothing done yet).
struct SelState { i32 c, n_out, kp1; u32 t_rel; }; // chain in progress, regions accepted so far, walk position + 1 (0 = chain not started), its first task
// One round of one read: continue the selection from `st` until it completes (true) or needs an extension that has not been
// computed (false; the seed is flagged in need[], or with force_all every remaining seed of the read).  Pointers are the read's
// own slices: outc[0..n_kept), sorted (seeds of all its chains), cand/srt/out/have/need at its first task.
SSQ_HD bool select_read(const ssq_opts_t &opt, int l_query, int n_kept, const ChainRec *outc, const Seed *sorted, const RegCand *cand, u64 *srt,
                        RegCand *out, const uint8_t *have, uint8_t *need, int force_all, SelState &st)
{
	int c = st.c, n_out = st.n_out, k = st.kp1 - 1;
	u32 t = st.t_rel;
	for (; c < n_kept; ++c, k = -1) {
		const ChainRec ch = outc[c];
		int stop_k = -1;
		const int miss = select_regions(opt, l_query, ch, sorted + ch.seed_start, cand + t, srt + t, out, n_out, have + t, k, &stop_k);
		if (miss >= 0) {
			if (force_all) { u32 e = t; for (int cc = c; cc < n_kept; ++cc) e += (u32)outc[cc].n; for (u32 x = t; x < e; ++x) need[x] = 1; }
			else need[t + miss] = 1;
			st.c = c; st.n_out = n_out; st.kp1 = stop_k + 1; st.t_rel = t;
			return false;
		}
		t += (u32)ch.n;
	}
	st.c = c; st.n_out = n_out; st.kp1 = 0; st.t_rel = t;
	return true;
}
