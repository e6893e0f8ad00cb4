// ssq_bgzf.cuh — the BGZF member encoder (deflate on the device) as SSQ_HD phases.
//
// One member = one payload of at most 0xff00 bytes = one gzip member with the BGZF header (BC extra field, BSIZE), one raw deflate
// block, CRC-32 and ISIZE — the framing of ssq_bgzf_compress (ssq_mem.cu), only the deflate payload differs.  The member is encoded
// by BZ_NT threads (one CTA in ssq_bgzf.cu; host loops over t in tests/hostsim/bgzf_host.cpp) through the phases below, with a
// barrier between phases.  Everything a phase writes is a function of the payload bytes (and level 0 / not 0) alone: the hash table
// keeps the largest position per bucket (atomicMax), histograms and packed bits are sums / ORs, so the result does not depend on
// thread scheduling, launch configuration or how the input was cut into calls.
//
//   load      payload -> shared memory, CRC table, hash table and histograms cleared
//   crc       CRC-32 of 128-byte sub-ranges, each moved to the member's end with the GF(2) shift (zlib's crc32_combine)
//   rounds    BZ_NT positions per round: each position looks up the newest earlier position with the same 4-byte hash (inserted in
//             earlier rounds) and extends the match; then the round's positions are inserted and one thread parses from the
//             last token end through the round, greedy with one step of lazy matching (it visits token starts only)
//   hist      literal/length and distance histograms of the tokens (+ end-of-block)
//   rank      used symbols ordered by (frequency, symbol)
//   plan      one thread: length-limited Huffman codes (15 bits; 7 for the code-length code, code lengths run-length coded with
//             16/17/18), exact bit cost of stored / fixed / dynamic, the cheapest is taken (level 0: stored)
//   pack      token bit lengths, exclusive scan (block-wide), every token ORed into the zeroed output slot at its bit offset
//   finish    gzip header, trailer (CRC-32, ISIZE), member size
#pragma once
#include "ssq_dev.cuh"

#define BZ_PAYLOAD 0xff00u          // bytes of payload per member (65280 + 5 + 26 <= 65536: a stored member always fits BSIZE)
#define BZ_NT 512                   // threads per member = positions per match-finding round
#define BZ_HBITS 14                 // hash table: 16384 buckets of the newest position + 1
#define BZ_MINM 4                   // shortest match the parser takes
#define BZ_SLOT (65536u + 64u)      // output slot per member: member bytes at +6, deflate bits at +24 (8-byte aligned)
#define BZ_SLOT_MEMBER 6u
#define BZ_SLOT_BITS 24u
#define BZ_CRC_SEG 128u             // CRC sub-range per thread (BZ_NT * BZ_CRC_SEG >= BZ_PAYLOAD)

typedef unsigned long long bz_u64;

struct BzSmem {                     // per-member state (shared memory on the device)
	uint8_t in[BZ_PAYLOAD + 8];
	u32 head[1u << BZ_HBITS];
	uint16_t mlen[BZ_NT], mdist[BZ_NT];
	u32 crc_tab[256];
	u32 part[BZ_NT];
	u32 lfreq[288], dfreq[32], cfreq[19];
	uint16_t lsort[288], dsort[32];
	u32 work[288];
	uint8_t llen[288], dlen[32], clen[19];
	uint16_t lrev[288], drev[32], crev[19];
	uint8_t rle[320], rle_x[320];
	u32 n, ntok, next, n_rle, hlit, hdist, hclen, btype, hdr_bits, dbytes, crc;
	int level;
};
static_assert(BZ_NT * BZ_CRC_SEG >= BZ_PAYLOAD, "CRC sub-ranges must cover a payload");

struct BzJob {                      // where one member's bytes come from and go to
	const uint8_t *src; u32 n;
	u32 *tok;                       // scratch: one word per token (<= BZ_PAYLOAD)
	uint8_t *slot;                  // BZ_SLOT bytes
	u32 *size;                      // member size out
};

// ---- primitives: atomics on the device, plain operations in the host loops ----
SSQ_HD void bz_add(u32 *p, u32 v)
{
#ifdef __CUDA_ARCH__
	atomicAdd(p, v);
#else
	*p += v;
#endif
}
SSQ_HD void bz_max(u32 *p, u32 v)
{
#ifdef __CUDA_ARCH__
	atomicMax(p, v);
#else
	if (v > *p) *p = v;
#endif
}
SSQ_HD void bz_or(bz_u64 *p, bz_u64 v)
{
#ifdef __CUDA_ARCH__
	atomicOr(p, v);
#else
	*p |= v;
#endif
}
SSQ_HD int bz_log2(u32 x)
{
#ifdef __CUDA_ARCH__
	return 31 - __clz(x);
#else
	return 31 - __builtin_clz(x);
#endif
}
// nb (<= 57) bits of v at bit offset off of the LSB-first stream in w
SSQ_HD void bz_put(bz_u64 *w, bz_u64 off, bz_u64 v, u32 nb)
{
	const u32 sh = (u32)(off & 63);
	bz_or(w + (off >> 6), v << sh);
	if (sh && sh + nb > 64) bz_or(w + (off >> 6) + 1, v >> (64 - sh));
}
SSQ_HD u32 bz_rev(u32 code, u32 len) { u32 r = 0; for (u32 i = 0; i < len; ++i) { r = (r << 1) | (code & 1); code >>= 1; } return r; }

// ---- CRC-32 (zlib polynomial, reflected) and its GF(2) shift ----
SSQ_HD u32 bz_crc_entry(u32 i) { u32 c = i; for (int k = 0; k < 8; ++k) c = c & 1 ? 0xedb88320u ^ (c >> 1) : c >> 1; return c; }
SSQ_HD u32 bz_multmodp(u32 a, u32 b) // a * b modulo the CRC polynomial
{
	u32 m = 1u << 31, p = 0;
	if (!a) return 0;
	for (;;) {
		if (a & m) { p ^= b; if ((a & (m - 1)) == 0) break; }
		m >>= 1;
		b = b & 1 ? (b >> 1) ^ 0xedb88320u : b >> 1;
	}
	return p;
}
SSQ_HD u32 bz_x8n(u32 n) // x^(8n) modulo the polynomial: appending n zero bytes
{
	u32 p = 1u << 31, sq = 1u << 23; // 1, x^8
	while (n) { if (n & 1) p = bz_multmodp(sq, p); n >>= 1; sq = bz_multmodp(sq, sq); }
	return p;
}

// ---- deflate symbols ----
SSQ_HD void bz_len_sym(u32 len, u32 &sym, u32 &nx, u32 &x) // len 3..258 -> symbol 257..285 + extra bits
{
	const u32 v = len - 3;
	if (len == 258) { sym = 285; nx = 0; x = 0; return; }
	if (v < 8) { sym = 257 + v; nx = 0; x = 0; return; }
	const int b = bz_log2(v);
	sym = 257 + 4 * (b - 1) + ((v >> (b - 2)) & 3); nx = b - 2; x = v & ((1u << (b - 2)) - 1);
}
SSQ_HD void bz_dist_sym(u32 d, u32 &sym, u32 &nx, u32 &x) // distance 1..32768 -> symbol 0..29 + extra bits
{
	const u32 v = d - 1;
	if (v < 4) { sym = v; nx = 0; x = 0; return; }
	const int b = bz_log2(v);
	sym = 2 * b + ((v >> (b - 1)) & 1); nx = b - 1; x = v & ((1u << (b - 1)) - 1);
}
SSQ_HD u32 bz_len_nx(u32 s) { return s < 265 || s == 285 ? 0 : (s - 261) / 4; }
SSQ_HD u32 bz_dist_nx(u32 s) { return s < 4 ? 0 : s / 2 - 1; }
SSQ_HD u32 bz_fixed_len(u32 s) { return s < 144 ? 8 : s < 256 ? 9 : s < 280 ? 7 : 8; }
SSQ_HD u32 bz_hash(const uint8_t *p) { const u32 x = (u32)p[0] | (u32)p[1] << 8 | (u32)p[2] << 16 | (u32)p[3] << 24; return (x * 2654435761u) >> (32 - BZ_HBITS); }

// ---- Huffman code lengths: minimum redundancy (Moffat-Katajainen, in place), then limited to maxlen by moving the overflow up
// the Kraft sum; symbols sorted ascending by (frequency, symbol), so equal inputs give equal codes ----
SSQ_HD void bz_huff(const u32 *freq, const uint16_t *sorted, int n, int maxlen, uint8_t *len, u32 *A)
{
	if (n == 0) return;
	if (n == 1) { len[sorted[0]] = 1; return; }
	for (int i = 0; i < n; ++i) A[i] = freq[sorted[i]];
	int root = 0, leaf = 2, next;
	A[0] += A[1];
	for (next = 1; next < n - 1; ++next) {
		if (leaf >= n || A[root] < A[leaf]) { A[next] = A[root]; A[root++] = (u32)next; } else A[next] = A[leaf++];
		if (leaf >= n || (root < next && A[root] < A[leaf])) { A[next] += A[root]; A[root++] = (u32)next; } else A[next] += A[leaf++];
	}
	A[n - 2] = 0;
	for (next = n - 3; next >= 0; --next) A[next] = A[A[next]] + 1;
	{
		int avbl = 1, used = 0, dpth = 0;
		root = n - 2; next = n - 1;
		while (avbl > 0) {
			while (root >= 0 && (int)A[root] == dpth) { ++used; --root; }
			while (avbl > used) { A[next--] = (u32)dpth; --avbl; }
			avbl = 2 * used; ++dpth; used = 0;
		}
	}
	u32 num[33];
	for (int i = 0; i < 33; ++i) num[i] = 0;
	for (int i = 0; i < n; ++i) ++num[A[i] > 32 ? 32 : A[i]];
	for (int i = maxlen + 1; i <= 32; ++i) { num[maxlen] += num[i]; num[i] = 0; }
	u32 total = 0;
	for (int i = maxlen; i > 0; --i) total += num[i] << (maxlen - i);
	while (total != (1u << maxlen)) {
		--num[maxlen];
		for (int i = maxlen - 1; i > 0; --i) if (num[i]) { --num[i]; num[i + 1] += 2; break; }
		--total;
	}
	for (int i = 1, j = n; i <= maxlen; ++i) for (u32 l = num[i]; l > 0; --l) len[sorted[--j]] = (uint8_t)i;
}
// canonical codes (RFC 1951 3.2.2), stored bit-reversed for LSB-first output
SSQ_HD void bz_canon(const uint8_t *len, int n, uint16_t *rev)
{
	u32 cnt[16], nc[16];
	for (int i = 0; i < 16; ++i) cnt[i] = 0;
	for (int s = 0; s < n; ++s) ++cnt[len[s]];
	cnt[0] = 0;
	u32 code = 0;
	for (int b = 1; b < 16; ++b) { code = (code + cnt[b - 1]) << 1; nc[b] = code; }
	for (int s = 0; s < n; ++s) rev[s] = len[s] ? (uint16_t)bz_rev(nc[len[s]]++, len[s]) : 0;
}

// ================================================================ the phases ====
SSQ_HD void bz_load(BzSmem &S, const BzJob &J, int level, int t)
{
	for (u32 i = t; i < J.n; i += BZ_NT) S.in[i] = J.src[i];
	for (u32 i = J.n + t; i < BZ_PAYLOAD + 8; i += BZ_NT) S.in[i] = 0;
	for (u32 i = t; i < (1u << BZ_HBITS); i += BZ_NT) S.head[i] = 0;
	for (u32 i = t; i < 288; i += BZ_NT) { S.lfreq[i] = 0; S.llen[i] = 0; }
	if (t < 32) { S.dfreq[t] = 0; S.dlen[t] = 0; }
	if (t < 19) { S.cfreq[t] = 0; S.clen[t] = 0; }
	if (t < 256) S.crc_tab[t] = bz_crc_entry((u32)t);
	if (t == 0) { S.n = J.n; S.ntok = 0; S.next = 0; S.level = level; }
}
SSQ_HD void bz_crc(BzSmem &S, int t)
{
	const u32 lo = (u32)t * BZ_CRC_SEG, hi = lo + BZ_CRC_SEG < S.n ? lo + BZ_CRC_SEG : S.n;
	u32 c = 0xffffffffu;
	for (u32 i = lo; i < hi; ++i) c = S.crc_tab[(c ^ S.in[i]) & 0xff] ^ (c >> 8);
	S.part[t] = lo < hi ? bz_multmodp(bz_x8n(S.n - hi), ~c) : 0;
}
// round at `base`, part 1: the match of position base + t against the newest earlier position with the same hash
SSQ_HD void bz_find(BzSmem &S, u32 base, int t)
{
	const u32 p = base + (u32)t;
	u32 L = 0, d = 0;
	if (S.level && p + 4 <= S.n) {
		const u32 c = S.head[bz_hash(S.in + p)];
		if (c && p - (c - 1) <= 32768u) {
			const u32 q = c - 1, lim = S.n - p < 258 ? S.n - p : 258;
			while (L < lim && S.in[q + L] == S.in[p + L]) ++L;
			d = p - q;
		}
	}
	S.mlen[t] = (uint16_t)(L >= BZ_MINM ? L : 0);
	S.mdist[t] = (uint16_t)(L >= BZ_MINM ? d : 0);
}
// part 2: insert the round's positions; one thread turns the round's token starts into tokens
SSQ_HD void bz_insert_parse(BzSmem &S, const BzJob &J, u32 base, int t)
{
	const u32 p = base + (u32)t;
	if (S.level && p + 4 <= S.n) bz_max(&S.head[bz_hash(S.in + p)], p + 1);
	if (t == 0) {
		u32 at = S.next, k = S.ntok;
		const u32 end = base + BZ_NT < S.n ? base + BZ_NT : S.n;
		while (at < end) {
			const u32 L = S.mlen[at - base];
			// lazy by one: a longer match at the next position wins
			if (L && !(at + 1 < end && S.mlen[at + 1 - base] > L)) { J.tok[k++] = 0x80000000u | L << 16 | S.mdist[at - base]; at += L; }
			else J.tok[k++] = S.in[at++];
		}
		S.next = at; S.ntok = k;
	}
}
SSQ_HD void bz_hist(BzSmem &S, const BzJob &J, int t)
{
	u32 s, nx, x;
	for (u32 k = t; k < S.ntok; k += BZ_NT) {
		const u32 w = J.tok[k];
		if (w >> 31) {
			bz_len_sym(w >> 16 & 0x1ff, s, nx, x); bz_add(&S.lfreq[s], 1);
			bz_dist_sym(w & 0xffff, s, nx, x); bz_add(&S.dfreq[s], 1);
		} else bz_add(&S.lfreq[w], 1);
	}
	if (t == 0) bz_add(&S.lfreq[256], 1);
}
SSQ_HD void bz_rank(BzSmem &S, int t)
{
	if (t < 286 && S.lfreq[t]) {
		u32 r = 0; const u32 f = S.lfreq[t];
		for (int j = 0; j < 286; ++j) r += S.lfreq[j] && (S.lfreq[j] < f || (S.lfreq[j] == f && j < t));
		S.lsort[r] = (uint16_t)t;
	}
	if (t >= 288 && t < 288 + 30 && S.dfreq[t - 288]) {
		const int i = t - 288; u32 r = 0; const u32 f = S.dfreq[i];
		for (int j = 0; j < 30; ++j) r += S.dfreq[j] && (S.dfreq[j] < f || (S.dfreq[j] == f && j < i));
		S.dsort[r] = (uint16_t)i;
	}
}
SSQ_HD void bz_rle_emit(BzSmem &S, u32 sym, u32 x) { S.rle[S.n_rle] = (uint8_t)sym; S.rle_x[S.n_rle] = (uint8_t)x; ++S.n_rle; bz_add(&S.cfreq[sym], 1); }
// one thread: trees, costs, the block type, the header length; the CRC of the member
SSQ_HD void bz_plan(BzSmem &S)
{
	u32 crc = 0;
	for (int t = 0; t < BZ_NT; ++t) crc ^= S.part[t];
	S.crc = crc;
	u32 nl = 0, nd = 0;
	for (int s = 0; s < 286; ++s) nl += S.lfreq[s] != 0;
	for (int s = 0; s < 30; ++s) nd += S.dfreq[s] != 0;
	bz_huff(S.lfreq, S.lsort, (int)nl, 15, S.llen, S.work);
	bz_huff(S.dfreq, S.dsort, (int)nd, 15, S.dlen, S.work);
	if (!nd) S.dlen[0] = 1; // a block without matches still declares one distance code
	u32 hlit = 286, hdist = 30;
	while (hlit > 257 && !S.llen[hlit - 1]) --hlit;
	while (hdist > 1 && !S.dlen[hdist - 1]) --hdist;
	// code lengths of both trees as one sequence, run-length coded
	S.n_rle = 0;
	{
		const u32 tot = hlit + hdist;
		u32 i = 0;
		while (i < tot) {
			const u32 v = i < hlit ? S.llen[i] : S.dlen[i - hlit];
			u32 run = 1;
			while (i + run < tot && (i + run < hlit ? S.llen[i + run] : S.dlen[i + run - hlit]) == v) ++run;
			u32 r = run;
			if (v == 0) {
				while (r >= 11) { const u32 k = r < 138 ? r : 138; bz_rle_emit(S, 18, k - 11); r -= k; }
				if (r >= 3) { bz_rle_emit(S, 17, r - 3); r = 0; }
				while (r) { bz_rle_emit(S, 0, 0); --r; }
			} else {
				bz_rle_emit(S, v, 0); --r;
				while (r >= 3) { const u32 k = r < 6 ? r : 6; bz_rle_emit(S, 16, k - 3); r -= k; }
				while (r) { bz_rle_emit(S, v, 0); --r; }
			}
			i += run;
		}
	}
	{ // code-length code: 19 symbols, at most 7 bits
		uint16_t cs[19]; int nc = 0;
		for (int s = 0; s < 19; ++s) if (S.cfreq[s]) {
			int j = nc++;
			while (j > 0 && (S.cfreq[cs[j - 1]] > S.cfreq[s] || (S.cfreq[cs[j - 1]] == S.cfreq[s] && cs[j - 1] > s))) { cs[j] = cs[j - 1]; --j; }
			cs[j] = (uint16_t)s;
		}
		bz_huff(S.cfreq, cs, nc, 7, S.clen, S.work);
		if (nc == 1) S.clen[cs[0] ? 0 : 1] = 1; // inflate takes no incomplete code-length code: a second 1-bit code, never used
	}
	const uint8_t ord[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
	u32 hclen = 19;
	while (hclen > 4 && !S.clen[ord[hclen - 1]]) --hclen;
	S.hlit = hlit; S.hdist = hdist; S.hclen = hclen;
	// exact costs in bits
	bz_u64 hdr = 3 + 14 + 3 * (bz_u64)hclen, fix = 3;
	for (u32 i = 0; i < S.n_rle; ++i) hdr += S.clen[S.rle[i]] + (S.rle[i] == 16 ? 2 : S.rle[i] == 17 ? 3 : S.rle[i] == 18 ? 7 : 0);
	bz_u64 dyn = hdr;
	for (u32 s = 0; s < 286; ++s) if (S.lfreq[s]) {
		const u32 nx = s > 256 ? bz_len_nx(s) : 0;
		dyn += (bz_u64)S.lfreq[s] * (S.llen[s] + nx); fix += (bz_u64)S.lfreq[s] * (bz_fixed_len(s) + nx);
	}
	for (u32 s = 0; s < 30; ++s) if (S.dfreq[s]) { dyn += (bz_u64)S.dfreq[s] * (S.dlen[s] + bz_dist_nx(s)); fix += (bz_u64)S.dfreq[s] * (5 + bz_dist_nx(s)); }
	const bz_u64 stored = 5 + (bz_u64)S.n, dynb = (dyn + 7) / 8, fixb = (fix + 7) / 8;
	if (!S.level || (stored <= dynb && stored <= fixb)) { S.btype = 0; S.dbytes = (u32)stored; S.hdr_bits = 0; }
	else if (fixb <= dynb) {
		S.btype = 1; S.dbytes = (u32)fixb; S.hdr_bits = 3;
		for (u32 s = 0; s < 288; ++s) S.llen[s] = (uint8_t)bz_fixed_len(s);
		for (u32 s = 0; s < 32; ++s) S.dlen[s] = 5;
	} else S.btype = 2, S.dbytes = (u32)dynb, S.hdr_bits = (u32)hdr;
	if (S.btype) { bz_canon(S.llen, 288, S.lrev); bz_canon(S.dlen, 32, S.drev); }
	if (S.btype == 2) bz_canon(S.clen, 19, S.crev);
}
// output slot: zero the words the deflate stream covers (+1 for the trailer bytes)
SSQ_HD void bz_zero(const BzSmem &S, const BzJob &J, int t)
{
	bz_u64 *w = (bz_u64*)(J.slot + BZ_SLOT_BITS);
	const u32 nw = (S.dbytes + 8 + 7) / 8 + 1;
	for (u32 i = t; i < nw; i += BZ_NT) w[i] = 0;
}
// one thread: block header bits (and for stored blocks the 5 header bytes)
SSQ_HD void bz_header(const BzSmem &S, const BzJob &J)
{
	bz_u64 *w = (bz_u64*)(J.slot + BZ_SLOT_BITS);
	if (S.btype == 0) { uint8_t *b = J.slot + BZ_SLOT_BITS; b[0] = 1; b[1] = (uint8_t)S.n; b[2] = (uint8_t)(S.n >> 8); b[3] = (uint8_t)~S.n; b[4] = (uint8_t)(~S.n >> 8); return; }
	bz_put(w, 0, 1 | S.btype << 1, 3);
	if (S.btype == 1) return;
	const uint8_t ord[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
	bz_u64 at = 3;
	bz_put(w, at, S.hlit - 257, 5); at += 5;
	bz_put(w, at, S.hdist - 1, 5); at += 5;
	bz_put(w, at, S.hclen - 4, 4); at += 4;
	for (u32 i = 0; i < S.hclen; ++i) { bz_put(w, at, S.clen[ord[i]], 3); at += 3; }
	for (u32 i = 0; i < S.n_rle; ++i) {
		const u32 s = S.rle[i], nx = s == 16 ? 2 : s == 17 ? 3 : s == 18 ? 7 : 0;
		bz_put(w, at, S.crev[s] | (bz_u64)S.rle_x[i] << S.clen[s], S.clen[s] + nx); at += S.clen[s] + nx;
	}
}
// bits of token k (value LSB-first in *v), 0 past the end
SSQ_HD u32 bz_tok_bits(const BzSmem &S, const BzJob &J, u32 k, bz_u64 *v)
{
	if (k >= S.ntok || S.btype == 0) { *v = 0; return 0; }
	const u32 w = J.tok[k];
	if (!(w >> 31)) { *v = S.lrev[w]; return S.llen[w]; }
	u32 s, nx, x, ds, dnx, dx;
	bz_len_sym(w >> 16 & 0x1ff, s, nx, x);
	bz_dist_sym(w & 0xffff, ds, dnx, dx);
	u32 nb = S.llen[s];
	bz_u64 r = S.lrev[s];
	r |= (bz_u64)x << nb; nb += nx;
	r |= (bz_u64)S.drev[ds] << nb; nb += S.dlen[ds];
	r |= (bz_u64)dx << nb; nb += dnx;
	*v = r;
	return nb;
}
SSQ_HD void bz_stored_copy(const BzSmem &S, const BzJob &J, int t)
{
	if (S.btype) return;
	uint8_t *b = J.slot + BZ_SLOT_BITS + 5;
	for (u32 i = t; i < S.n; i += BZ_NT) b[i] = S.in[i];
}
// one thread, after the tokens: end-of-block at bit `at`, then gzip header and trailer around the deflate bytes
SSQ_HD void bz_eob(const BzSmem &S, const BzJob &J, bz_u64 at)
{
	if (S.btype) bz_put((bz_u64*)(J.slot + BZ_SLOT_BITS), at, S.lrev[256], S.llen[256]);
}
SSQ_HD void bz_finish(const BzSmem &S, const BzJob &J)
{
	uint8_t *h = J.slot + BZ_SLOT_MEMBER, *tr = J.slot + BZ_SLOT_BITS + S.dbytes;
	const u32 size = 18 + S.dbytes + 8, bsize = size - 1;
	const uint8_t hdr[16] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0};
	for (int i = 0; i < 16; ++i) h[i] = hdr[i];
	h[16] = (uint8_t)bsize; h[17] = (uint8_t)(bsize >> 8);
	for (int k = 0; k < 4; ++k) { tr[k] = (uint8_t)(S.crc >> (8 * k)); tr[4 + k] = (uint8_t)(S.n >> (8 * k)); }
	*J.size = size;
}
