// ssq_bai.cuh — the BAI index of a coordinate-sorted BAM file (what `sambamba index` 0.5.9 writes, byte for byte) as SSQ_HD
// phases, plus the host logic that drives them.  The kernels are in ssq_bai.cu; tests/hostsim/bai_host.cpp runs the same phases
// in host loops.
//
//   inflate   the BGZF members in parallel (ssq_gunzip.cuh, gz_bgzf_members): the text and the member table (compressed offset,
//             text offset of every member), from which every virtual offset is made.
//   header    the host reads magic, l_text, n_ref and the reference names from the start of the text: the first record's offset.
//   walk      records are a chain of block_size fields across member borders.  The text after the header is cut into segments of
//             S bytes, one walker each.  Segment 0 starts at the first record; segment i > 0 at its first plausible record start
//             (a sound block_size, refID in range, a printable name ending on its NUL; and so for the 4 records after it).  A
//             walker follows the chain to the first record start at or past its segment's end (its exit).  Segment i's exit must be segment i+1's
//             start; a broken link is walked again from the exit before it, until every link holds (as gz_window repairs chunks).
//             The guess only costs time: the records come from the chain from the first record.
//   records   the walkers go again and write each record's virtual offsets of start and end, refID, pos, reference length
//             (M/D/N/=/X), stored bin and flag.
//   check     the order sambamba requires, and what the device does not reproduce (below), record by record.
//   index     runs of consecutive records in one (reference, bin) are chunks; a stable sort by (reference, bin) puts each bin's
//             runs together in file order; a run merges into the chunk before it when that chunk ends in the BGZF block where the
//             run starts (sambamba: the previous chunk's end and the run's start have the same compressed offset).  The 16 KB
//             linear index takes, for each window, the first record that touches it; windows nothing touches take the value of
//             the window before them (0 at the start).  Per reference, the pseudo-bin 37450 holds the virtual offsets of its
//             first record's start and its last record's end, and its mapped and unmapped counts.
//   serialise the host writes the result: per reference n_bin, the bins in the order sambamba writes them (its bin table is a D
//             associative array, iterated bucket by bucket; bai_aa_order), the pseudo-bin, n_intv and the linear index; then the
//             number of records without a reference.
//
// Rules, each pinned with the reference's sambamba on a fixture (tests/golden/make_bai_golden.py):
//   - the bin is the stored one, not one computed from the CIGAR;
//   - an unmapped record touches the window of its position; a mapped one the windows from its position's to that of
//     (pos + reference length - 1) / 16384, truncated toward zero: a record of reference length 0 touches its position's window
//     unless the position is a nonzero multiple of 16384 (then none; at position 0, window 0);
//   - a virtual offset at a member border is (the next member's offset, 0); the end of the text is (the offset of the empty last
//     member, or the file's length when there is none, 0);
//   - the last reference with records ends where the last record of the file ends, records without a reference included;
//   - empty references are n_bin 0, n_intv 0.
// Refused, with a message (sambamba fails on the first two and writes an index the BAI format cannot hold, or one that differs
// from this description, for the others): records out of coordinate order; a record with a reference and no position; a refID
// below -1 or at or beyond n_ref; a record that reaches past 2^29; a record without a reference before one with a reference; an
// empty BGZF member before the last one; input whose BGZF chain or records do not reach exactly to its end.
#pragma once
#include <algorithm>
#include <string>
#include "ssq_gunzip.cuh"

#define BAI_SEG_DEFAULT (64u << 10)
#define BAI_NONE (~0ull)
#define BAI_LIMIT (1ll << 29)
#define BAI_SHIFT 14
#define BAI_META_BIN 37450u

// one walker: in start (BAI_NONE: guess one in [a, lim)); out exit, count, status
struct BaiSeg { bz_u64 a, lim, start, exit, bad; u32 count, status; };
enum { BAI_S_OK = 0, BAI_S_BAD = 1, BAI_S_NONE = 2 };
struct BaiRec { bz_u64 vbeg, vend; int32_t ref, pos, rlen; uint16_t bin, flag; };
enum { BAI_E_OK = 0, BAI_E_REF = 1, BAI_E_NOPOS = 2, BAI_E_ORDER = 3, BAI_E_NOCOOR = 4, BAI_E_LIMIT = 5 };
struct BaiChunk { bz_u64 beg, end; };
struct BaiBin { int32_t ref; u32 bin, first_run, lo, hi; };  // chunks [lo, hi) of the sorted chunk table

SSQ_HD u32 bai_u32(const uint8_t *t, bz_u64 q) { return t[q] | t[q + 1] << 8 | t[q + 2] << 16 | (u32)t[q + 3] << 24; }
SSQ_HD u32 bai_u16(const uint8_t *t, bz_u64 q) { return t[q] | t[q + 1] << 8; }

// a record at q: 4 + block_size, or 0 when it is not a sound record inside the text
SSQ_HD bz_u64 bai_rec_len(const uint8_t *t, bz_u64 n, bz_u64 q)
{
	if (q + 36 > n) return 0;
	const u32 bs = bai_u32(t, q);
	if (bs < 32 || q + 4 + bs > n) return 0;
	const u32 lrn = t[q + 12], ncig = bai_u16(t, q + 16);
	const int32_t lseq = (int32_t)bai_u32(t, q + 20);
	if (lrn < 1 || lseq < 0 || 32 + lrn + 4ull * ncig + ((bz_u64)lseq + 1) / 2 + (bz_u64)lseq > bs) return 0;
	return 4 + (bz_u64)bs;
}
// one record that looks real: sound, refID in [-1, n_ref), pos >= -1, a name of printable characters ending on its NUL
SSQ_HD bz_u64 bai_looks_real(const uint8_t *t, bz_u64 n, bz_u64 q, int n_ref)
{
	const bz_u64 len = bai_rec_len(t, n, q);
	if (!len) return 0;
	const int32_t ref = (int32_t)bai_u32(t, q + 4), pos = (int32_t)bai_u32(t, q + 8);
	const u32 lrn = t[q + 12];
	if (ref < -1 || ref >= n_ref || pos < -1 || t[q + 36 + lrn - 1] != 0) return 0;
	for (u32 k = 0; k + 1 < lrn; ++k) if (t[q + 36 + k] < '!' || t[q + 36 + k] > '~') return 0;
	return len;
}
// a plausible record start: it and the BAI_GUESS_CHAIN records after it (or as many as there are before the end) look real
#define BAI_GUESS_CHAIN 4
SSQ_HD bool bai_plausible(const uint8_t *t, bz_u64 n, bz_u64 q, int n_ref)
{
	for (int k = 0; k <= BAI_GUESS_CHAIN && q < n; ++k) {
		const bz_u64 len = bai_looks_real(t, n, q, n_ref);
		if (!len) return false;
		q += len;
	}
	return true;
}
// S.start known: follow the chain to the first record start >= S.lim (or the text end)
SSQ_HD void bai_walk(const uint8_t *t, bz_u64 n, BaiSeg &S)
{
	bz_u64 p = S.start; u32 c = 0;
	S.status = BAI_S_OK;
	while (p < S.lim && p < n) {
		const bz_u64 len = bai_rec_len(t, n, p);
		if (!len) { S.status = BAI_S_BAD; S.bad = p; break; }
		p += len; ++c;
	}
	S.exit = p; S.count = c;
}
SSQ_HD void bai_guess_walk(const uint8_t *t, bz_u64 n, int n_ref, BaiSeg &S)
{
	if (S.start == BAI_NONE) {
		bz_u64 q = S.a;
		while (q < S.lim && !bai_plausible(t, n, q, n_ref)) ++q;
		if (q >= S.lim) { S.status = BAI_S_NONE; S.exit = BAI_NONE; S.count = 0; return; }
		S.start = q;
	}
	bai_walk(t, n, S);
}
// virtual offset of text offset x: the member holding byte x; the end of the text: (the next member, or the file's end, 0)
SSQ_HD bz_u64 bai_vo(const GzMember *m, bz_u64 nm, bz_u64 clen, bz_u64 x)
{
	bz_u64 lo = 0, hi = nm; // largest j with toff <= x
	while (hi - lo > 1) { const bz_u64 mid = (lo + hi) / 2; if (m[mid].toff <= x) lo = mid; else hi = mid; }
	const bz_u64 u = x - m[lo].toff;
	if (u >= m[lo].isize && m[lo].isize) return (lo + 1 < nm ? m[lo + 1].coff : clen) << 16;
	return m[lo].coff << 16 | u;
}
// the record at q (of length len) -> its fields
SSQ_HD void bai_rec(const uint8_t *t, bz_u64 q, bz_u64 len, const GzMember *m, bz_u64 nm, bz_u64 clen, BaiRec &r)
{
	r.vbeg = bai_vo(m, nm, clen, q); r.vend = bai_vo(m, nm, clen, q + len);
	r.ref = (int32_t)bai_u32(t, q + 4); r.pos = (int32_t)bai_u32(t, q + 8);
	r.bin = (uint16_t)bai_u16(t, q + 14); r.flag = (uint16_t)bai_u16(t, q + 18);
	const u32 ncig = bai_u16(t, q + 16);
	const bz_u64 c = q + 36 + t[q + 12];
	long long rl = 0;
	for (u32 k = 0; k < ncig; ++k) { const u32 v = bai_u32(t, c + 4ull * k), op = v & 15; if (op == 0 || op == 2 || op == 3 || op == 7 || op == 8) rl += v >> 4; }
	r.rlen = rl > 0x7fffffff ? 0x7fffffff : (int32_t)rl;
}
// the walker again, writing its records from out[0]
SSQ_HD void bai_walk_write(const uint8_t *t, bz_u64 n, const BaiSeg &S, const GzMember *m, bz_u64 nm, bz_u64 clen, BaiRec *out)
{
	bz_u64 p = S.start;
	for (u32 c = 0; c < S.count; ++c) { const bz_u64 len = bai_rec_len(t, n, p); bai_rec(t, p, len, m, nm, clen, out[c]); p += len; }
}
// record i against the one before it: BAI_E_*
SSQ_HD int bai_check(const BaiRec *r, bz_u64 i, int n_ref)
{
	const BaiRec &c = r[i];
	if (c.ref < -1 || c.ref >= n_ref) return BAI_E_REF;
	if (c.ref < 0) return BAI_E_OK;
	if (c.pos < 0) return BAI_E_NOPOS;
	if ((long long)c.pos + ((c.flag & 4) || c.rlen == 0 ? 1 : c.rlen) > BAI_LIMIT) return BAI_E_LIMIT;
	if (i) {
		const BaiRec &p = r[i - 1];
		if (p.ref < 0) return BAI_E_NOCOOR;
		if (c.ref < p.ref || (c.ref == p.ref && c.pos < p.pos)) return BAI_E_ORDER;
	}
	return BAI_E_OK;
}
// linear-index windows [*w0, *w1) the record touches (*w1 also bounds n_intv).  The last window is sambamba's
// (pos + reference length - 1) / 16384 with C's truncating division (so at position 0 a record of reference length 0 still
// touches window 0, where an arithmetic shift would give window -1)
SSQ_HD void bai_windows(const BaiRec &c, long long *w0, long long *w1)
{
	*w0 = c.pos >> BAI_SHIFT;
	const long long last = (long long)c.pos + c.rlen - 1; // >= -1: positions are checked >= 0
	*w1 = (c.flag & 4) ? *w0 + 1 : (last < 0 ? 0 : last >> BAI_SHIFT) + 1;
}
SSQ_HD bool bai_run_start(const BaiRec *r, bz_u64 i) { return !i || r[i].ref != r[i - 1].ref || r[i].bin != r[i - 1].bin; }
SSQ_HD bz_u64 bai_run_key(const BaiRec &c) { return (bz_u64)(u32)c.ref << 16 | c.bin; }
// in (reference, bin, file) order, run j opens a new chunk unless it continues the bin of run j - 1 in the same BGZF block
SSQ_HD bool bai_new_chunk(bz_u64 kprev, bz_u64 vend_prev, bz_u64 k, bz_u64 vbeg) { return kprev != k || (vend_prev >> 16) != (vbeg >> 16); }

// ============================================================================= host logic ====
static inline const char *bai_why(int e)
{
	return e == BAI_E_REF ? "its refID is not a reference of the header" : e == BAI_E_NOPOS ? "it has a reference but no position" :
	       e == BAI_E_ORDER ? "the file is not coordinate-sorted: it comes before the record above it" :
	       e == BAI_E_NOCOOR ? "a record without a reference comes before it" : "it reaches past 2^29, beyond what a BAI index holds";
}

// what the index phase hands the serialiser: per reference, its bins (reference-major, then by bin), chunks, linear index, metadata
struct BaiOut {
	std::vector<BaiBin> bins;
	std::vector<BaiChunk> chunks;
	std::vector<bz_u64> lin;          // all references' linear indexes, back to back
	std::vector<bz_u64> lin_base;     // n_ref + 1
	std::vector<bz_u64> meta;         // 4 per reference: first start, last end, mapped, unmapped
	std::vector<uint8_t> has;         // references with records
	bz_u64 no_coor;
};

struct BaiBackend {
	virtual ~BaiBackend() {}
	virtual int walk(std::vector<BaiSeg> &seg, const std::vector<int> &which, int n_ref) = 0; // seg: host mirror; walks which[]
	virtual int records(const std::vector<BaiSeg> &seg, const std::vector<bz_u64> &base, bz_u64 n_rec) = 0;
	virtual int check(bz_u64 n_rec, int n_ref, bz_u64 *first_bad, bz_u64 *n_pos) = 0;   // first_bad: i << 3 | BAI_E_*, or BAI_NONE
	virtual int index(bz_u64 n_rec, bz_u64 n_pos, int n_ref, BaiOut &out) = 0;
	virtual int rec_at(bz_u64 i, BaiRec *r) = 0;                                         // one record, for a message
	virtual void phase() {}                                                              // the checks are done: the index starts
};

// the walk: segments of seg_bytes from the first record r0 to the text end n; every link made to hold.  0, or SSQ_EFORMAT with a message
static inline int bai_walk_all(BaiBackend &be, int n_ref, bz_u64 r0, bz_u64 n, bz_u64 seg_bytes, std::vector<BaiSeg> &seg, std::vector<bz_u64> &base, bz_u64 *n_rec)
{
	const bz_u64 ns = n > r0 ? (n - r0 + seg_bytes - 1) / seg_bytes : 1;
	seg.assign(ns, BaiSeg());
	std::vector<int> which(ns);
	for (bz_u64 i = 0; i < ns; ++i) {
		BaiSeg &S = seg[i];
		S.a = r0 + i * seg_bytes; S.lim = S.a + seg_bytes < n ? S.a + seg_bytes : n;
		S.start = i ? BAI_NONE : r0; S.exit = BAI_NONE; S.count = 0; S.status = BAI_S_NONE; S.bad = 0;
		which[i] = (int)i;
	}
	int rc;
	if ((rc = be.walk(seg, which, n_ref))) return rc;
	for (;;) {
		bz_u64 k = 0;
		while (k + 1 < ns && seg[k].status == BAI_S_OK && seg[k].exit == seg[k + 1].start) ++k;
		if (seg[k].status == BAI_S_BAD) { ssq_set_error("text byte %llu: not a BAM record (its block_size does not fit)", (unsigned long long)seg[k].bad); return SSQ_EFORMAT; }
		if (k + 1 == ns) break;
		which.clear();
		for (bz_u64 j = k; j + 1 < ns; ++j)
			if (seg[j].status == BAI_S_OK && seg[j].exit != seg[j + 1].start) { seg[j + 1].start = seg[j].exit; which.push_back((int)(j + 1)); }
		if ((rc = be.walk(seg, which, n_ref))) return rc;
	}
	if (seg[ns - 1].exit != n) { ssq_set_error("the last record runs past the end of the text"); return SSQ_EFORMAT; }
	base.assign(ns + 1, 0);
	for (bz_u64 i = 0; i < ns; ++i) base[i + 1] = base[i] + seg[i].count;
	*n_rec = base[ns];
	return SSQ_OK;
}

// the BAM header from a prefix of the text: 0 (*r0 = the first record's offset, *n_ref), 1 = need more text, or SSQ_EFORMAT
static inline int bai_header(const uint8_t *t, bz_u64 have, bz_u64 total, bz_u64 *r0, int *n_ref)
{
	auto need = [&](bz_u64 x) { return x > have; };
	if (need(8)) { if (total < 8 || have == total) { ssq_set_error("not a BAM file: shorter than its header"); return SSQ_EFORMAT; } return 1; }
	if (memcmp(t, "BAM\1", 4)) { ssq_set_error("not a BAM file: no BAM magic"); return SSQ_EFORMAT; }
	const bz_u64 lt = bai_u32(t, 4);
	bz_u64 p = 8 + lt;
	if (p + 4 > total) { ssq_set_error("not a BAM file: the header is truncated"); return SSQ_EFORMAT; }
	if (need(p + 4)) return 1;
	const int32_t nr = (int32_t)bai_u32(t, p);
	if (nr < 0) { ssq_set_error("not a BAM file: n_ref < 0"); return SSQ_EFORMAT; }
	p += 4;
	for (int32_t i = 0; i < nr; ++i) {
		if (p + 4 > total) { ssq_set_error("not a BAM file: the reference table is truncated"); return SSQ_EFORMAT; }
		if (need(p + 4)) return 1;
		p += 8 + (bz_u64)bai_u32(t, p);
		if (p > total) { ssq_set_error("not a BAM file: the reference table is truncated"); return SSQ_EFORMAT; }
	}
	*r0 = p; *n_ref = nr;
	return 0;
}

// the order sambamba 0.5.9 writes one reference's bins in: its D associative array (druntime's chained hash table: 4 buckets,
// hash of a uint = its value, new keys at the tail of their bucket, rehashed to the next size of a prime list when it holds more
// than 4 keys per bucket, the old keys moved last to first; iterated bucket by bucket).  keys: the bins in the order their first chunks were made
// (the same table keyed by strings orders the merged header's read-group and program IDs, ssq_merge.cuh)
template <class K>
static inline void bai_aa_order(const std::vector<K> &keys, std::vector<int> &order)
{
	static const bz_u64 primes[] = {31, 97, 389, 1543, 6151, 24593, 98317, 393241, 1572869};
	std::vector<std::vector<int>> bk(4);
	for (size_t i = 0; i < keys.size(); ++i) {
		bk[keys[i] % bk.size()].push_back((int)i);
		if (i + 1 > bk.size() * 4) {
			size_t p = 0;
			while (p + 1 < sizeof primes / sizeof *primes && i + 1 > primes[p]) ++p;
			std::vector<std::vector<int>> nb(primes[p]);
			for (size_t q = bk.size(); q--;) for (size_t x = bk[q].size(); x--;) nb[keys[bk[q][x]] % nb.size()].push_back(bk[q][x]);
			bk.swap(nb);
		}
	}
	order.clear();
	for (auto &b : bk) for (int e : b) order.push_back(e);
}

static inline void bai_put32(std::string &s, u32 v) { s.append((const char*)&v, 4); }
static inline void bai_put64(std::string &s, bz_u64 v) { s.append((const char*)&v, 8); }
static inline void bai_serialise(int n_ref, const BaiOut &o, std::string &s)
{
	s.assign("BAI\1", 4);
	bai_put32(s, (u32)n_ref);
	size_t b = 0;
	std::vector<u32> keys; std::vector<int> order; std::vector<const BaiBin*> ins;
	for (int r = 0; r < n_ref; ++r) {
		const size_t b0 = b;
		while (b < o.bins.size() && o.bins[b].ref == r) ++b;
		if (!o.has[r]) { bai_put32(s, 0); bai_put32(s, 0); continue; }
		ins.clear();
		for (size_t k = b0; k < b; ++k) ins.push_back(&o.bins[k]);
		std::sort(ins.begin(), ins.end(), [](const BaiBin *x, const BaiBin *y) { return x->first_run < y->first_run; });
		keys.clear();
		for (auto *x : ins) keys.push_back(x->bin);
		bai_aa_order(keys, order);
		bai_put32(s, (u32)(ins.size() + 1));
		for (int e : order) {
			const BaiBin &B = *ins[e];
			bai_put32(s, B.bin); bai_put32(s, B.hi - B.lo);
			for (u32 c = B.lo; c < B.hi; ++c) { bai_put64(s, o.chunks[c].beg); bai_put64(s, o.chunks[c].end); }
		}
		bai_put32(s, BAI_META_BIN); bai_put32(s, 2);
		for (int k = 0; k < 4; ++k) bai_put64(s, o.meta[4 * r + k]);
		bai_put32(s, (u32)(o.lin_base[r + 1] - o.lin_base[r]));
		for (bz_u64 w = o.lin_base[r]; w < o.lin_base[r + 1]; ++w) bai_put64(s, o.lin[w]);
	}
	bai_put64(s, o.no_coor);
}

// after the inflate: the whole index of the text [0, n) (members m of a file of clen bytes).  fetch(x, buf) copies the text's first
// x bytes to buf.  0, or SSQ_EFORMAT with a message
template <class Fetch>
static inline int bai_from_text(BaiBackend &be, Fetch fetch, bz_u64 n, const std::vector<GzMember> &m, bz_u64 seg_bytes, std::string &bai)
{
	for (size_t j = 0; j + 1 < m.size(); ++j)
		if (!m[j].isize) { ssq_set_error("an empty BGZF member at compressed byte %llu is not the last one", (unsigned long long)m[j].coff); return SSQ_EFORMAT; }
	bz_u64 r0 = 0; int n_ref = 0, rc;
	std::vector<uint8_t> h;
	for (bz_u64 want = 1 << 16;; want *= 4) {
		const bz_u64 k = want < n ? want : n;
		h.resize(k);
		if ((rc = fetch(k, h.data()))) return rc;
		const int r = bai_header(h.data(), k, n, &r0, &n_ref);
		if (r == 0) break;
		if (r != 1) return r;
	}
	std::vector<BaiSeg> seg; std::vector<bz_u64> base;
	bz_u64 n_rec = 0;
	if ((rc = bai_walk_all(be, n_ref, r0, n, seg_bytes, seg, base, &n_rec))) return rc;
	if ((rc = be.records(seg, base, n_rec))) return rc;
	bz_u64 bad = BAI_NONE, n_pos = 0;
	if ((rc = be.check(n_rec, n_ref, &bad, &n_pos))) return rc;
	if (bad != BAI_NONE) {
		BaiRec r;
		if ((rc = be.rec_at(bad >> 3, &r))) return rc;
		ssq_set_error("record %llu (refID %d, pos %d, at virtual offset %llu/%llu): %s", (unsigned long long)(bad >> 3), r.ref, r.pos,
		              (unsigned long long)(r.vbeg >> 16), (unsigned long long)(r.vbeg & 0xffff), bai_why((int)(bad & 7)));
		return SSQ_EFORMAT;
	}
	be.phase();
	BaiOut o;
	if ((rc = be.index(n_rec, n_pos, n_ref, o))) return rc;
	o.no_coor = n_rec - n_pos;
	bai_serialise(n_ref, o, bai);
	return SSQ_OK;
}
