// ssq_merge.cuh — `sambamba merge out.bam in1.bam in2.bam ...` (0.5.9) of coordinate-sorted BAM files: the records in the order
// sambamba's merge gives them and its merged header, as SSQ_HD phases plus the host logic that drives them.  The kernels are in
// ssq_merge.cu; tests/hostsim/merge_host.cpp runs the same phases in host loops.  The inputs stream through windows, so files
// larger than device memory merge.
//
//   header   each input's header is read on the host (zlib, its first members); the merged header follows sambamba's rules below.
//   window   per input, the host cuts a window of whole BGZF members from the file (walking the BSIZE fields, at most
//            window_bytes of compressed bytes, at least one member).  The device inflates it (ssq_gunzip_inflate_bgzf_dev) behind
//            the bytes carried from the input's last window: the record the window end cut, or the rest of the header.
//   records  the BAI builder's walker (ssq_bai.cuh) finds the record starts, segment by segment; the chain ends at the first
//            record the text does not hold whole, which is carried into the next window.
//   keys     8 bytes per record (refID with -1 last, pos, reverse strand: sambamba's sort key), and each input's own order is
//            checked: (refID, pos) must not fall.  The keys go to the host.
//   order    the host runs sambamba's heap (below) over the keys alone, up to the first step that needs a key from an input whose
//            window is used up and whose file is not.  The records so far are gathered; that input's next window is read; the
//            heap goes on where it stopped.
//   gather   the output positions (input << 48 | record) go to the device; a scan of the record sizes in output order, then a
//            warp per record copies it into the output buffer, which is compressed on the device or handed back to the host.
//
// Rules, each pinned with the reference's sambamba on a fixture (tests/golden/make_merge_golden.py):
//   - order: D's NWayUnion over a BinaryHeap of the inputs.  The inputs without records are removed "unstably" (a hole is filled
//     from the back, after empty inputs at the back are dropped); the heap is a max-heap under comp(a, b) = key(b) < key(a),
//     built by down(i) for i = n/2-1 .. 0; each step takes the root's front, swaps the root with element n-1, n -= 1, down(0),
//     pops the front of element n, drops it if it is empty, else n += 1 and sifts it up.  Equal keys from different inputs
//     come out in the order this gives, not in input order.
//   - header: @HD VN:1.3 SO:coordinate; the @SQ lines; the @RG lines, then the @PG lines, each the union of the inputs' lines
//     (identical lines once) in the iteration order of a D associative array keyed by ID (hash h = h * 11 + byte; bai_aa_order),
//     keys entered by file in argument order and by line within a file; the @CO lines in argument order, duplicates kept.  Tags
//     in sambamba's order (reorder_tags).
// Refused (SSQ_EFORMAT or SSQ_EDATA, the file named; sambamba does other things or something the fixtures do not pin): fewer than
// two inputs; an input that is not BGZF or does not inflate; a header without @HD SO:coordinate; @HD lines, @SQ dictionaries or
// reference tables that differ; an @RG / @PG ID carried by two different lines; a header line that is not @HD / @SQ / @RG / @PG /
// @CO; a record whose refID is not a reference of the header; records out of (refID, pos) order within an input; a record cut
// by the end of its file; a record that is not one (its block_size does not fit).
#pragma once
#include <errno.h>
#include <stdio.h>
#include <string.h>
#include <chrono>
#include <string>
#include <vector>
#include <zlib.h>
#include "ssq_bai.cuh"
#include "ssq_samhdr.h"

#define MG_WINDOW_DEFAULT (32ull << 20)
#define MG_IDX_BITS 48
#define MG_IDX_MASK ((1ull << MG_IDX_BITS) - 1)
#define MG_MAX_RECORD (1u << 30)
enum { MG_E_OK = 0, MG_E_REF = 1, MG_E_ORDER = 2 };

// the merge key of the record at q (the sort key of the sambamba shim): refID << 34 | (pos + 1) << 1 | reverse; no reference: ~0
SSQ_HD bz_u64 mg_key(const uint8_t *t, bz_u64 q)
{
	const int32_t ref = (int32_t)bai_u32(t, q + 4), pos = (int32_t)bai_u32(t, q + 8);
	return ref < 0 ? ~0ull : ((bz_u64)(u32)ref << 34 | (bz_u64)(u32)(pos + 1) << 1 | ((bai_u16(t, q + 18) >> 4) & 1));
}
// record i of a window (offsets roff): *key, and MG_E_*.  Strand is not an order: only (refID, pos) may not fall
SSQ_HD int mg_check(const uint8_t *t, const bz_u64 *roff, bz_u64 i, int n_ref, bz_u64 *key)
{
	const int32_t ref = (int32_t)bai_u32(t, roff[i] + 4);
	*key = mg_key(t, roff[i]);
	if (ref < -1 || ref >= n_ref) return MG_E_REF;
	if (i && mg_key(t, roff[i - 1]) >> 1 > *key >> 1) return MG_E_ORDER;
	return MG_E_OK;
}
// a walker's records -> their text offsets from roff[0]
SSQ_HD void mg_walk_write(const uint8_t *t, bz_u64 n, const BaiSeg &S, bz_u64 *roff)
{
	bz_u64 p = S.start;
	for (u32 c = 0; c < S.count; ++c) { roff[c] = p; p += bai_rec_len(t, n, p); }
}

// ============================================================================= host logic ====
// one input on the host: its file, compressed bytes read ahead, header, and the state of its window
struct MgInput {
	std::string path;
	FILE *fp = 0;
	std::vector<uint8_t> c;           // compressed bytes [c_at, c_n) not yet in a window
	bz_u64 c_at = 0, c_n = 0, c_off = 0; // c_off: file offset of c[0]
	bool c_eof = false;
	std::string text, refs;           // header text (to its first NUL) and reference table (n_ref and entries, as stored)
	bz_u64 r0 = 0; int n_ref = 0;     // text offset of the first record
	bz_u64 skip = 0, tl = 0, chain_end = 0; // header bytes still to skip; text in the window buffer; where its records end
	std::vector<bz_u64> keys;         // the window's records
	bz_u64 next = 0, before = 0, last_key = 0; // next record; records of the earlier windows; key of the last record read
	bool done = false;                // no window follows
	~MgInput() { if (fp) fclose(fp); }
};

// more compressed bytes: 0, or SSQ_EIO
static inline int mg_read_more(MgInput &in)
{
	if (in.c_at) { memmove(in.c.data(), in.c.data() + in.c_at, in.c_n - in.c_at); in.c_n -= in.c_at; in.c_off += in.c_at; in.c_at = 0; }
	if (in.c.size() < in.c_n + (1u << 20)) in.c.resize(in.c.size() * 2 > in.c_n + (1u << 20) ? in.c.size() * 2 : in.c_n + (1u << 20));
	const size_t k = fread(in.c.data() + in.c_n, 1, in.c.size() - in.c_n, in.fp);
	if (!k) { if (ferror(in.fp)) { ssq_set_error("%s: read error", in.path.c_str()); return SSQ_EIO; } in.c_eof = true; }
	in.c_n += k;
	return SSQ_OK;
}
// the member at c[at] whole in the buffer: 0 (*cs, *is), 1 = the file ends at `at`, or SSQ_EDATA / SSQ_EIO with a message
static inline int mg_member(MgInput &in, bz_u64 &at, u32 *cs, u32 *is)
{
	for (;;) {
		if (at == in.c_n && in.c_eof) return 1;
		const int r = at < in.c_n ? gz_bgzf_member(in.c.data(), in.c_n, at, cs, is) : GZ_B_TRUNC;
		if (r == GZ_B_OK) return 0;
		if (r != GZ_B_TRUNC || in.c_eof) { ssq_set_error("%s is not BGZF: %s at compressed byte %llu", in.path.c_str(), gz_bgzf_why(r), (unsigned long long)(in.c_off + at)); return SSQ_EDATA; }
		const bz_u64 sh = in.c_at;
		int rc;
		if ((rc = mg_read_more(in))) return rc;
		at -= sh;
	}
}
// the next window of whole members: [*w0, *w0 + *wn) of in.c and its members (offsets from the window); 1 = the file has ended
static inline int mg_window(MgInput &in, bz_u64 window_bytes, bz_u64 *w0, bz_u64 *wn, std::vector<GzMember> &m)
{
	m.clear();
	bz_u64 at = in.c_at, t = 0;
	int rc;
	for (;;) {
		u32 cs, is;
		if ((rc = mg_member(in, at, &cs, &is)) == 1) break;
		if (rc) return rc;
		const bz_u64 w = in.c_at; // the buffer may have moved: offsets from the window's start
		if (!m.empty() && at + cs - w > window_bytes) break;
		m.push_back({at - w, t, cs, is});
		t += is; at += cs;
	}
	if (m.empty()) return 1;
	*w0 = in.c_at; *wn = at - in.c_at;
	in.c_at = at;
	return SSQ_OK;
}

// the BAM header of input `in` (from its first members, inflated here with zlib; the window path reads them again)
static inline int mg_read_header(MgInput &in)
{
	std::vector<uint8_t> t;
	bz_u64 at = 0;
	int rc;
	for (;;) {
		u32 cs, is;
		if ((rc = mg_member(in, at, &cs, &is)) < 0) return rc;
		if (rc == 0) {
			const bz_u64 h = 12 + (in.c[at + 10] | in.c[at + 11] << 8);
			const size_t old = t.size();
			t.resize(old + is);
			z_stream zs; memset(&zs, 0, sizeof zs);
			inflateInit2(&zs, -15);
			zs.next_in = in.c.data() + at + h; zs.avail_in = (uInt)(cs - h - 8); zs.next_out = t.data() + old; zs.avail_out = is;
			const int zr = inflate(&zs, Z_FINISH);
			inflateEnd(&zs);
			if (zr != Z_STREAM_END || zs.total_out != is) { ssq_set_error("%s: corrupt BGZF member at compressed byte %llu", in.path.c_str(), (unsigned long long)(in.c_off + at)); return SSQ_EDATA; }
			at += cs;
		}
		const int r = bai_header(t.data(), t.size(), rc == 1 ? t.size() : ~0ull >> 1, &in.r0, &in.n_ref);
		if (r == 0 && in.r0 <= t.size()) break; // (bai_header does not wait for the last reference name)
		if (r != 0 && r != 1) { const std::string e = ssq_last_error(); ssq_set_error("%s: %s", in.path.c_str(), e.c_str()); return SSQ_EFORMAT; }
		if (rc == 1) { ssq_set_error("%s: not a BAM file: the header is truncated", in.path.c_str()); return SSQ_EFORMAT; }
	}
	const u32 lt = bai_u32(t.data(), 4);
	in.text.assign((const char*)t.data() + 8, strnlen((const char*)t.data() + 8, lt));
	in.refs.assign((const char*)t.data() + 8 + lt, in.r0 - 8 - lt);
	in.skip = in.r0;
	return SSQ_OK;
}

// the merged header text (sambamba's rules, head of this file): 0, or SSQ_EFORMAT naming the files
static inline int mg_merge_header(const std::vector<MgInput*> &in, std::string &out)
{
	struct Tab { std::vector<std::string> id, line; std::vector<bz_u64> hash; };
	Tab tab[2]; // @RG, @PG
	std::string hd0, sq0, co;
	for (size_t f = 0; f < in.size(); ++f) {
		const std::string &t = in[f]->text;
		const char *name = in[f]->path.c_str();
		std::string hd, sq;
		for (size_t p = 0; p < t.size();) {
			size_t e = t.find('\n', p);
			if (e == std::string::npos) e = t.size();
			const std::string line = t.substr(p, e - p);
			p = e + 1;
			if (line.empty()) continue;
			const std::string ty = line.substr(0, 3);
			if (ty == "@HD") hd += line + "\n";
			else if (ty == "@SQ") reorder_tags(line, sq);
			else if (ty == "@CO") co += line + "\n";
			else if (ty == "@RG" || ty == "@PG") {
				Tab &T = tab[ty == "@PG"];
				std::string r; reorder_tags(line, r); r.pop_back();
				const size_t a = r.find("\tID:");
				if (a == std::string::npos) { ssq_set_error("%s: an %s line without ID", name, ty.c_str()); return SSQ_EFORMAT; }
				const size_t b = r.find('\t', a + 4);
				const std::string id = r.substr(a + 4, b == std::string::npos ? std::string::npos : b - a - 4);
				size_t k = 0;
				while (k < T.id.size() && T.id[k] != id) ++k;
				if (k == T.id.size()) {
					bz_u64 h = 0;
					for (unsigned char ch : id) h = h * 11 + ch;
					T.id.push_back(id); T.line.push_back(r); T.hash.push_back(h);
				} else if (T.line[k] != r) { ssq_set_error("%s: %s ID %s is carried by two different lines (sambamba renames one)", name, ty.c_str(), id.c_str()); return SSQ_EFORMAT; }
			} else { ssq_set_error("%s: header line %s is not merged here", name, ty.c_str()); return SSQ_EFORMAT; }
		}
		if (hd.find("\tSO:coordinate") == std::string::npos) { ssq_set_error("%s: its header does not say SO:coordinate", name); return SSQ_EFORMAT; }
		if (!f) { hd0 = hd; sq0 = sq; continue; }
		if (hd != hd0) { ssq_set_error("the @HD lines of %s and %s differ", in[0]->path.c_str(), name); return SSQ_EFORMAT; }
		if (sq != sq0 || in[f]->refs != in[0]->refs) { ssq_set_error("the @SQ dictionaries of %s and %s differ", in[0]->path.c_str(), name); return SSQ_EFORMAT; }
	}
	out = "@HD\tVN:1.3\tSO:coordinate\n" + sq0;
	std::vector<int> order;
	for (const Tab &T : tab) { bai_aa_order(T.hash, order); for (int k : order) out += T.line[k] + "\n"; }
	out += co;
	return SSQ_OK;
}

// open the inputs and read their headers; the merged header text
static inline int mg_open(const char *const *paths, int n, std::vector<MgInput> &in, std::string &text)
{
	if (n < 2) { ssq_set_error("merge needs at least two inputs"); return SSQ_EINVAL; }
	in.clear(); in.resize(n);
	std::vector<MgInput*> p;
	int rc;
	for (int k = 0; k < n; ++k) {
		in[k].path = paths[k];
		if (!(in[k].fp = fopen(paths[k], "rb"))) { ssq_set_error("cannot open %s: %s", paths[k], strerror(errno)); return SSQ_EIO; }
		if ((rc = mg_read_header(in[k]))) return rc;
		p.push_back(&in[k]);
	}
	return mg_merge_header(p, text);
}

// "BAM\1", l_text, the merged text, the reference table of the first input
static inline std::string mg_bam_header(const std::string &text, const MgInput &first)
{
	std::string o("BAM\1", 4);
	const u32 l = (u32)text.size();
	o.append((const char*)&l, 4); o += text; o += first.refs;
	return o;
}

struct MergeBackend {
	virtual ~MergeBackend() {}
	// input k's next text buffer: the current one's [from, from + keep), then the members m of the compressed window c[0, clen)
	// inflated (SSQ_EDATA: *err_at = the failing member's offset in c)
	virtual int fill(int k, bz_u64 from, bz_u64 keep, const uint8_t *c, bz_u64 clen, const std::vector<GzMember> &m, bz_u64 *err_at) = 0;
	virtual int peek(int k, bz_u64 at, void *buf, u32 len) = 0;                             // text bytes of input k to the host
	virtual int walk(int k, std::vector<BaiSeg> &seg, const std::vector<int> &which, int n_ref) = 0;
	// the walkers' record offsets, then the keys (to keys) and the first failing record (i << 3 | MG_E_*, or BAI_NONE)
	virtual int records(int k, const std::vector<BaiSeg> &seg, const std::vector<bz_u64> &base, bz_u64 n_rec, int n_ref, std::vector<bz_u64> &keys, bz_u64 *bad) = 0;
	// the records at the output positions (k << MG_IDX_BITS | i), in that order, to the output
	virtual int gather(const std::vector<bz_u64> &order, bz_u64 bytes_max) = 0;
};

// the record chain of input k's text [r0, n), segment by segment; it ends at the first record the text does not hold whole
// (*end).  0, or SSQ_EFORMAT with a message
static inline int mg_walk_all(MergeBackend &be, MgInput &in, int k, bz_u64 r0, bz_u64 n, bz_u64 seg_bytes, std::vector<BaiSeg> &seg, std::vector<bz_u64> &base, bz_u64 *n_rec, bz_u64 *end)
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
	if ((rc = be.walk(k, seg, which, in.n_ref))) return rc;
	bz_u64 last = ns - 1;
	for (;;) {
		bz_u64 j = 0;
		while (j + 1 < ns && seg[j].status == BAI_S_OK && seg[j].exit == seg[j + 1].start) ++j;
		if (seg[j].status == BAI_S_BAD) { // the first broken link: a record cut by the window's end, or not a record
			const bz_u64 p = seg[j].bad;
			uint8_t b[4];
			if (p + 4 <= n) {
				if ((rc = be.peek(k, p, b, 4))) return rc;
				const u32 bs = bai_u32(b, 0);
				if (bs >= MG_MAX_RECORD || p + 4 + bs <= n) {
					bz_u64 i = 0;
					for (bz_u64 q = 0; q <= j; ++q) i += seg[q].count;
					ssq_set_error("%s: record %llu is not a BAM record (its block_size does not fit)", in.path.c_str(), (unsigned long long)(in.before + i));
					return SSQ_EFORMAT;
				}
			}
			seg[j].exit = p; last = j;
			for (bz_u64 q = j + 1; q < ns; ++q) seg[q].count = 0;
			break;
		}
		if (j + 1 == ns) break;
		which.clear();
		for (bz_u64 q = j; q + 1 < ns; ++q)
			if (seg[q].status == BAI_S_OK && seg[q].exit != seg[q + 1].start) { seg[q + 1].start = seg[q].exit; which.push_back((int)(q + 1)); }
		if ((rc = be.walk(k, seg, which, in.n_ref))) return rc;
	}
	base.assign(ns + 1, 0);
	for (bz_u64 i = 0; i < ns; ++i) base[i + 1] = base[i] + seg[i].count;
	*n_rec = base[ns]; *end = seg[last].exit;
	return SSQ_OK;
}

// input k's window is used up: read windows until one holds a whole record or the file ends (in.done)
static inline int mg_refill(MergeBackend &be, MgInput &in, int k, bz_u64 window_bytes, bz_u64 seg_bytes)
{
	bz_u64 from = in.chain_end, keep = in.tl - in.chain_end;
	std::vector<GzMember> m; std::vector<BaiSeg> seg; std::vector<bz_u64> base;
	in.before += in.keys.size();
	in.keys.clear(); in.next = 0;
	for (;;) {
		bz_u64 w0 = 0, wn = 0, err_at = 0;
		int rc = mg_window(in, window_bytes, &w0, &wn, m);
		if (rc == 1) {
			in.done = true;
			if (keep || in.skip) { ssq_set_error("%s: record %llu runs past the end of the file", in.path.c_str(), (unsigned long long)in.before); return SSQ_EFORMAT; }
			return SSQ_OK;
		}
		if (rc) return rc;
		if ((rc = be.fill(k, from, keep, in.c.data() + w0, wn, m, &err_at))) {
			if (rc == SSQ_EDATA) ssq_set_error("%s: corrupt BGZF member at compressed byte %llu", in.path.c_str(), (unsigned long long)(in.c_off + w0 + err_at));
			return rc;
		}
		in.tl = keep + m.back().toff + m.back().isize;
		bz_u64 s = 0;
		if (in.skip) { s = in.skip < in.tl ? in.skip : in.tl; in.skip -= s; }
		if (in.skip) { from = in.tl; keep = 0; in.chain_end = in.tl; continue; }
		bz_u64 n_rec = 0, end = s;
		if (s < in.tl && (rc = mg_walk_all(be, in, k, s, in.tl, seg_bytes, seg, base, &n_rec, &end))) return rc;
		in.chain_end = end;
		if (!n_rec) { from = s; keep = in.tl - s; continue; }
		bz_u64 bad = BAI_NONE;
		if ((rc = be.records(k, seg, base, n_rec, in.n_ref, in.keys, &bad))) return rc;
		if (bad == BAI_NONE && in.before && in.keys[0] >> 1 < in.last_key >> 1) bad = 0 << 3 | MG_E_ORDER;
		if (bad != BAI_NONE) {
			const bz_u64 i = bad >> 3, key = in.keys[i];
			if ((bad & 7) == MG_E_REF) ssq_set_error("%s: record %llu: its refID is not a reference of the header", in.path.c_str(), (unsigned long long)(in.before + i));
			else ssq_set_error("%s: record %llu (refID %d, pos %d) comes before the record above it: the file is not coordinate-sorted", in.path.c_str(),
			                   (unsigned long long)(in.before + i), key == ~0ull ? -1 : (int)(key >> 34), key == ~0ull ? -1 : (int)((key >> 1 & 0xffffffffu) - 1));
			return SSQ_EFORMAT;
		}
		in.last_key = in.keys.back();
		return SSQ_OK;
	}
}

// sambamba's heap over the inputs (head of this file); positions hold input numbers, keys are their fronts
struct MgHeap {
	std::vector<int> h;
	const std::vector<MgInput> *in;
	bz_u64 key(int p) const { const MgInput &x = (*in)[h[p]]; return x.keys[x.next]; }
	bool comp(int a, int b) const { return key(b) < key(a); }
	void down(int i)
	{
		const int n = (int)h.size();
		for (;;) {
			const int l = 2 * i + 1, r = l + 1;
			if (r == n) { if (comp(i, l)) std::swap(h[i], h[l]); return; }
			if (r > n) return;
			const int g = comp(i, l) ? (comp(l, r) ? r : l) : (comp(i, r) ? r : i);
			if (g == i) return;
			std::swap(h[i], h[g]); i = g;
		}
	}
	void up(int c) { while (c > 0) { const int p = (c - 1) / 2; if (!comp(p, c)) return; std::swap(h[p], h[c]); c = p; } }
};

typedef std::chrono::steady_clock MgClock;
static inline double mg_since(MgClock::time_point t) { return std::chrono::duration<double, std::milli>(MgClock::now() - t).count(); }

// the whole merge after mg_open: every record through be.gather in sambamba's order.  ms[0] windows (read, inflate, walk, keys),
// ms[1] the host heap, ms[2] gathers (with what the backend does with the output), all host clocks around synchronised work
static inline int mg_run(MergeBackend &be, std::vector<MgInput> &in, bz_u64 window_bytes, bz_u64 seg_bytes, bz_u64 *n_out, double ms[3])
{
	int rc;
	MgClock::time_point t = MgClock::now();
	for (size_t k = 0; k < in.size(); ++k) if ((rc = mg_refill(be, in[k], (int)k, window_bytes, seg_bytes))) return rc;
	ms[0] += mg_since(t);
	t = MgClock::now();
	MgHeap H; H.in = &in;
	for (size_t k = 0; k < in.size(); ++k) H.h.push_back((int)k);
	for (size_t i = 0; i < H.h.size();) { // "unstable" removal of the inputs without records
		if (!in[H.h[i]].keys.empty()) { ++i; continue; }
		while (!H.h.empty() && in[H.h.back()].keys.empty()) H.h.pop_back();
		if (i >= H.h.size()) break;
		H.h[i] = H.h.back(); H.h.pop_back(); ++i;
	}
	for (int i = (int)H.h.size() / 2 - 1; i >= 0; --i) H.down(i);
	std::vector<bz_u64> order;
	*n_out = 0;
	auto flush = [&]() {
		bz_u64 mx = 0;
		for (const MgInput &x : in) mx += x.tl;
		ms[1] += mg_since(t);
		const MgClock::time_point g = MgClock::now();
		const int r = order.empty() ? 0 : be.gather(order, mx);
		*n_out += order.size(); order.clear();
		ms[2] += mg_since(g);
		t = MgClock::now();
		return r;
	};
	while (!H.h.empty()) {
		const int r = H.h[0];
		order.push_back((bz_u64)r << MG_IDX_BITS | in[r].next);
		std::swap(H.h[0], H.h.back());
		const int x = H.h.back();
		H.h.pop_back(); H.down(0);
		MgInput &X = in[x];
		if (++X.next == X.keys.size() && !X.done) { // its window is used up: what is gathered so far goes out, its next window comes in
			if ((rc = flush())) return rc;
			const MgClock::time_point w = MgClock::now();
			if ((rc = mg_refill(be, X, x, window_bytes, seg_bytes))) return rc;
			ms[0] += mg_since(w);
			t = MgClock::now();
		}
		if (X.next < X.keys.size()) { H.h.push_back(x); H.up((int)H.h.size() - 1); }
	}
	return flush();
}
