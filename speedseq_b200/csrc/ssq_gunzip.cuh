// ssq_gunzip.cuh — chunk-parallel gzip decoding (RFC 1951 deflate inside RFC 1952 gzip members) as SSQ_HD phases, plus the host
// logic that drives them.  The kernels are in ssq_gunzip.cu; tests/hostsim/gunzip_host.cpp runs the same phases in host loops.
//
// One deflate stream is decoded in windows of compressed bytes.  A window starts at a known position (GzPos: a bit offset plus
// what sits there — a gzip header, a block start, or a point inside a block whose header is at `hdr`) with the last <= 32 KB of
// text before it as context.  Per window:
//   sync      the window is cut into chunks of C compressed bytes; for every chunk i > 0 the lanes of a warp test the chunk's bit
//             offsets in order and keep the first one where a dynamic-Huffman block header is valid, its block decodes to EOB with
//             valid symbols and distances <= 32768, and the next block header is plausible (or the block is final).  A chunk
//             without one is merged into the chunk before it.
//   decode    one thread per chunk decodes from its start to the first block start at or past the next chunk's start (e_i), into
//             a slot of 16-bit symbols: a byte is itself, a reference before the chunk start is a placeholder 256 + p naming the
//             context byte p of the 32 KB before the chunk (copies of placeholders stay placeholders).  All block types and
//             member boundaries are decoded; a full slot or event list stops the chunk at a resumable position (between
//             symbols, inside a block if need be), so every chunk makes progress whatever the block sizes.
//   link      chunk 0 starts at a true position, so a chunk whose links i -> i+1 (e_i == start_{i+1}) all hold back to chunk 0
//             is exact.  Every broken link is repaired by decoding chunk i+1 again from e_i, until every link holds; each round
//             the exact prefix grows by at least one chunk.
//   resolve   chunk outputs are laid out by a prefix sum behind the context; one CTA resolves the placeholders of each chunk's
//             last 32 KB in chunk order (the next chunk's context), then every other symbol is resolved in one parallel pass.
//   crc       CRC-32 of fixed-size pieces of each member's text, combined on the host with the GF(2) shift (bz_multmodp, bz_x8n)
//             and checked with ISIZE against the trailer; the running CRC and length of a member carry across windows.
//   carry     the window ends where its last exact chunk stopped; the next one starts there with the last 32 KB of text.
// End of stream is zlib gzread's: concatenated members are one stream, bytes after a member that do not start with 1f 8b are
// ignored, an empty input is an empty output.  Anything else that does not decode is an error at a compressed offset.
#pragma once
#include <string.h>
#include <vector>
#include "ssq_bgzf.cuh"

#define GZ_CTX 32768u             // deflate window: the context a chunk may reference
#define GZ_SLOT (1u << 19)        // symbols per chunk slot (FASTQ: a 32 KB chunk plus the block it ends in, with room to spare)
#define GZ_MAXCH 1024             // chunks per window: slots 1 GB, text buffer 512 MB
#define GZ_EVCAP 16               // member ends recorded per chunk decode
#define GZ_CHUNK_DEFAULT (32u << 10)
#define GZ_SLACK (1u << 20)       // input past the window the last chunk may read to finish its block
#define GZ_CRC_PIECE 16384u       // text bytes per CRC piece
#define GZ_LFB 9                  // bits of the first-level literal/length table
#define GZ_DFB 7                  // bits of the first-level distance table
#define GZ_NONE (~0ull)

// what sits at a position
enum { GZ_M_FIRST = 0, GZ_M_NEXT = 1, GZ_M_BLOCK = 2, GZ_M_IN = 3, GZ_M_TRAILER = 4 };
// how a chunk decode ended
enum { GZ_S_OK = 0, GZ_S_FULL = 1, GZ_S_INPUT = 2, GZ_S_EOS = 3, GZ_S_BAD = 4 };

struct GzPos { bz_u64 bit, hdr; u32 mode; }; // hdr: the block header of an M_IN position (M_IN at hdr == the block start)

struct GzChunk {
	GzPos start;                  // in: where to decode from
	bz_u64 stop;                  // in: stop at the first block start >= stop
	GzPos end;                    // out: where it stopped
	u32 len, status, n_ev;        // out: symbols, GZ_S_*, member ends
	u32 min_ph;                   // out: smallest placeholder index before the chunk's first member start (GZ_CTX if none)
	bz_u64 bad;                   // out: bit offset of the error (GZ_S_BAD)
};
struct GzEvent { u32 out, crc, isize, pad; bz_u64 at; }; // a member ended after `out` symbols; trailer at compressed byte `at`

struct GzIn { const uint8_t *p; bz_u64 n; int final; }; // compressed bytes the window may read

// a decoder's Huffman tables: first-level tables (sym << 4 | len, 0 = longer code or none) + canonical counts/symbols
struct GzTab {
	uint16_t lfast[1 << GZ_LFB], dfast[1 << GZ_DFB];
	uint16_t lcnt[16], lsym[288], dcnt[16], dsym[32];
	uint8_t lens[320];
};

// ---- bit reader: LSB-first; bytes past the input read as zero and mark `over` ----
struct GzBits {
	const uint8_t *p; bz_u64 n, nb; bz_u64 buf; u32 cnt;
	SSQ_HD void seek(bz_u64 bit) { nb = bit >> 3; buf = 0; cnt = 0; fill(); u32 k = (u32)(bit & 7); buf >>= k; cnt -= k; }
	SSQ_HD void fill() { while (cnt <= 56) { buf |= (bz_u64)(nb < n ? p[nb] : 0) << cnt; ++nb; cnt += 8; } }
	SSQ_HD bz_u64 pos() const { return nb * 8 - cnt; }
	SSQ_HD bool over() const { return pos() > n * 8; }
	SSQ_HD u32 peek(u32 k) { if (cnt < k) fill(); return (u32)(buf & ((1ull << k) - 1)); }
	SSQ_HD void drop(u32 k) { buf >>= k; cnt -= k; }
	SSQ_HD u32 get(u32 k) { if (!k) return 0; u32 v = peek(k); drop(k); return v; }
};

// canonical code from lengths: counts + symbols in code order; returns the unused code space (0 = complete, < 0 = over-subscribed)
SSQ_HD int gz_canon(const uint8_t *len, int n, uint16_t *cnt, uint16_t *sym)
{
	for (int i = 0; i < 16; ++i) cnt[i] = 0;
	for (int s = 0; s < n; ++s) ++cnt[len[s]];
	int left = 1;
	for (int l = 1; l < 16; ++l) { left <<= 1; left -= cnt[l]; if (left < 0) return left; }
	uint16_t off[16]; off[1] = 0;
	for (int l = 1; l < 15; ++l) off[l + 1] = off[l] + cnt[l];
	for (int s = 0; s < n; ++s) if (len[s]) sym[off[len[s]]++] = (uint16_t)s;
	return left;
}
SSQ_HD void gz_fast(const uint8_t *len, int n, int fb, uint16_t *fast)
{
	for (int i = 0; i < (1 << fb); ++i) fast[i] = 0;
	u32 cnt[16], next[16], code = 0;
	for (int i = 0; i < 16; ++i) cnt[i] = 0;
	for (int s = 0; s < n; ++s) ++cnt[len[s]];
	cnt[0] = 0;
	for (int b = 1; b < 16; ++b) { code = (code + cnt[b - 1]) << 1; next[b] = code; }
	for (int s = 0; s < n; ++s) {
		const u32 l = len[s];
		if (!l) continue;
		const u32 c = next[l]++;
		if ((int)l > fb) continue;
		for (u32 r = bz_rev(c, l); r < (1u << fb); r += 1u << l) fast[r] = (uint16_t)(s << 4 | l);
	}
}
// one symbol: first-level table, then bit by bit; -1 = no such code
SSQ_HD int gz_sym(GzBits &B, const uint16_t *fast, int fb, const uint16_t *cnt, const uint16_t *sym)
{
	const u32 e = fast[B.peek(fb)];
	if (e) { B.drop(e & 15); return e >> 4; }
	const u32 bits = B.peek(15);
	int code = 0, first = 0, index = 0;
	for (int l = 1; l < 16; ++l) {
		code |= (bits >> (l - 1)) & 1;
		const int c = cnt[l];
		if (code - c < first) { B.drop(l); return sym[index + (code - first)]; }
		index += c; first += c; first <<= 1; code <<= 1;
	}
	return -1;
}
SSQ_HD u32 gz_len_base(u32 s) { const u32 i = s - 257; return i < 8 ? 3 + i : s == 285 ? 258 : 3 + ((4 + ((i - 8) & 3)) << ((i - 4) / 4)); }
SSQ_HD u32 gz_dist_base(u32 s) { return s < 4 ? 1 + s : 1 + ((2 + (s & 1)) << (s / 2 - 1)); }

// the header of the block at B (after BFINAL/BTYPE = 2): tables into T.  strict (sync search): the literal/length code must be
// complete; otherwise zlib's rules (an incomplete code only when its longest length is 1).  Returns 0, or -1 invalid, -2 input
SSQ_HD int gz_dyn_header(GzBits &B, GzTab &T, bool strict)
{
	const u32 hlit = B.get(5) + 257, hdist = B.get(5) + 1, hclen = B.get(4) + 4;
	if (hlit > 286 || hdist > 30) return -1;
	const uint8_t ord[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
	uint8_t cl[19];
	for (int i = 0; i < 19; ++i) cl[i] = 0;
	for (u32 i = 0; i < hclen; ++i) cl[ord[i]] = (uint8_t)B.get(3);
	if (B.over()) return -2;
	if (gz_canon(cl, 19, T.lcnt, T.lsym) != 0) return -1; // the code-length code must be complete
	for (int i = 0; i < 8; ++i) T.lfast[i] = 0; // (no fast table for it: bit by bit)
	u32 i = 0;
	while (i < hlit + hdist) {
		const int s = gz_sym(B, T.lfast, 0, T.lcnt, T.lsym);
		if (s < 0) return B.over() ? -2 : -1;
		if (s < 16) { T.lens[i++] = (uint8_t)s; continue; }
		u32 rep, v = 0;
		if (s == 16) { if (!i) return -1; v = T.lens[i - 1]; rep = 3 + B.get(2); }
		else if (s == 17) rep = 3 + B.get(3);
		else rep = 11 + B.get(7);
		if (i + rep > hlit + hdist) return -1;
		while (rep--) T.lens[i++] = (uint8_t)v;
	}
	if (B.over()) return -2;
	if (!T.lens[256]) return -1;
	// zlib takes an incomplete code only when it is one code of length 1, and an empty distance code
	const int ll = gz_canon(T.lens, (int)hlit, T.lcnt, T.lsym);
	if (ll < 0 || (ll > 0 && (strict || !(T.lcnt[1] == 1 && hlit - T.lcnt[0] == 1)))) return -1;
	const int dl = gz_canon(T.lens + hlit, (int)hdist, T.dcnt, T.dsym);
	if (dl < 0 || (dl > 0 && !(T.dcnt[1] == 1 && hdist - T.dcnt[0] == 1) && T.dcnt[0] != hdist)) return -1;
	gz_fast(T.lens, (int)hlit, GZ_LFB, T.lfast);
	gz_fast(T.lens + hlit, (int)hdist, GZ_DFB, T.dfast);
	return 0;
}
SSQ_HD void gz_fixed(GzTab &T)
{
	for (int s = 0; s < 288; ++s) T.lens[s] = (uint8_t)bz_fixed_len((u32)s);
	for (int s = 0; s < 30; ++s) T.lens[288 + s] = 5;
	gz_canon(T.lens, 288, T.lcnt, T.lsym);
	gz_canon(T.lens + 288, 30, T.dcnt, T.dsym);
	gz_fast(T.lens, 288, GZ_LFB, T.lfast);
	gz_fast(T.lens + 288, 30, GZ_DFB, T.dfast);
}

// ---- sync search: is `bit` the start of a dynamic block that decodes to its end, followed by a plausible header? ----
SSQ_HD bool gz_try_sync(const GzIn &I, GzTab &T, bz_u64 bit)
{
	GzBits B; B.p = I.p; B.n = I.n; B.seek(bit);
	const u32 h = B.get(3);
	if ((h >> 1) != 2) return false;
	if (gz_dyn_header(B, T, true)) return false;
	u32 produced = 0; // a distance may reach 32768 bytes before the block
	for (;;) {
		const int s = gz_sym(B, T.lfast, GZ_LFB, T.lcnt, T.lsym);
		if (s < 0 || s > 285 || B.over()) return false;
		if (s < 256) { ++produced; continue; }
		if (s == 256) break;
		const u32 len = gz_len_base((u32)s) + B.get(bz_len_nx((u32)s));
		const int d = gz_sym(B, T.dfast, GZ_DFB, T.dcnt, T.dsym);
		if (d < 0 || d > 29) return false;
		const u32 dist = gz_dist_base((u32)d) + B.get(bz_dist_nx((u32)d));
		if (dist > GZ_CTX + produced) return false;
		produced += len;
	}
	if (B.over()) return false;
	if (h & 1) return true;
	const u32 nh = B.get(3);
	if (B.over()) return false;
	if ((nh >> 1) == 3) return false;
	if ((nh >> 1) == 2) { const u32 a = B.get(5), b = B.get(5); return a <= 29 && b <= 29 && !B.over(); }
	if ((nh >> 1) == 0) {
		const bz_u64 q = (B.pos() + 7) >> 3;
		if (q + 4 > I.n) return false;
		return (u32)(I.p[q] | I.p[q + 1] << 8) == (u32)(~(I.p[q + 2] | I.p[q + 3] << 8) & 0xffff);
	}
	return true;
}
// lanes of a warp (host: lane loop) test bit offsets lo + lane, lo + lane + 32, ...: the first valid one below hi, or GZ_NONE
SSQ_HD bool gz_sync_lane(const GzIn &I, GzTab &T, bz_u64 lo, bz_u64 hi, u32 round, int lane, bz_u64 *cand)
{
	const bz_u64 b = lo + (bz_u64)round * 32 + (bz_u64)lane;
	*cand = b;
	return b < hi && gz_try_sync(I, T, b);
}

// ---- one chunk decode ----
SSQ_HD u32 gz_rd8(const GzIn &I, bz_u64 byte) { return byte < I.n ? I.p[byte] : 0; }
// a gzip member header at byte q: its length (> 0), 0 when the input ends in it, -1 when invalid
SSQ_HD long long gz_member_header(const GzIn &I, bz_u64 q)
{
	if (q + 10 > I.n) return 0;
	if (I.p[q] != 0x1f || I.p[q + 1] != 0x8b) return -1;
	const u32 flg = I.p[q + 3];
	if (I.p[q + 2] != 8 || (flg & 0xe0)) return -1;
	bz_u64 at = q + 10;
	if (flg & 4) { if (at + 2 > I.n) return 0; at += 2 + (I.p[at] | I.p[at + 1] << 8); }
	for (u32 f = 8; f <= 16; f <<= 1) if (flg & f) { while (at < I.n && I.p[at]) ++at; if (at >= I.n) return 0; ++at; }
	if (flg & 2) {
		if (at + 2 > I.n) return 0;
		u32 c = 0xffffffffu;
		for (bz_u64 k = q; k < at; ++k) c = bz_crc_entry((c ^ I.p[k]) & 0xff) ^ (c >> 8);
		if ((~c & 0xffff) != (u32)(I.p[at] | I.p[at + 1] << 8)) return -1;
		at += 2;
	}
	if (at > I.n) return 0;
	return (long long)(at - q);
}

// decodes chunk C from C.start (see the header comment); slot: GZ_SLOT symbols, ev: GZ_EVCAP events
SSQ_HD void gz_decode(const GzIn &I, GzTab &T, GzChunk &C, uint16_t *slot, GzEvent *ev)
{
	GzBits B; B.p = I.p; B.n = I.n;
	u32 o = 0, mode = C.start.mode, n_ev = 0, min_ph = GZ_CTX;
	int mstart = -(int)GZ_CTX - 1; // output offset of the current member's start; below -GZ_CTX: before the chunk, unknown
	bz_u64 bit = C.start.bit, hdr = C.start.hdr, left = 0; // left: bytes still to copy of a stored block
	u32 btype = 0, bfinal = 0;
	C.status = GZ_S_BAD; C.bad = bit;
#define GZ_END(st) do { C.status = (st); goto done; } while (0)
#define GZ_FAIL(at) do { C.bad = (at); C.status = GZ_S_BAD; goto done; } while (0)
	if (mode == GZ_M_IN) { // resume inside the block whose header is at hdr
		B.seek(hdr);
		const u32 h = B.get(3);
		bfinal = h & 1; btype = h >> 1;
		if (btype == 2) { if (gz_dyn_header(B, T, false)) GZ_FAIL(hdr); }
		else if (btype == 1) gz_fixed(T);
		else {
			const bz_u64 q = (B.pos() + 7) >> 3, len = gz_rd8(I, q) | gz_rd8(I, q + 1) << 8;
			left = len - ((bit >> 3) - (q + 4));
		}
		B.seek(bit);
	}
	for (;;) {
		if (mode == GZ_M_FIRST || mode == GZ_M_NEXT) {
			const bz_u64 q = bit >> 3;
			if (mode == GZ_M_NEXT || q < I.n) {
				const bool magic = q + 2 <= I.n && I.p[q] == 0x1f && I.p[q + 1] == 0x8b;
				if (!magic && mode == GZ_M_NEXT) {
					if (q + 2 > I.n && !I.final) GZ_END(GZ_S_INPUT);
					GZ_END(GZ_S_EOS); // nothing, or bytes that are not a member: the stream ends
				}
			} else if (I.final) GZ_END(GZ_S_EOS); // empty input
			else GZ_END(GZ_S_INPUT);
			const long long h = gz_member_header(I, q);
			if (h < 0) GZ_FAIL(bit);
			if (h == 0) { if (I.final) GZ_FAIL(bit); GZ_END(GZ_S_INPUT); }
			bit = (q + (bz_u64)h) * 8; mode = GZ_M_BLOCK; mstart = (int)o;
			continue;
		}
		if (mode == GZ_M_TRAILER) {
			const bz_u64 q = bit >> 3;
			if (q + 8 > I.n) { if (I.final) GZ_FAIL(bit); GZ_END(GZ_S_INPUT); }
			GzEvent &E = ev[n_ev++];
			E.out = o; E.at = q;
			E.crc = I.p[q] | I.p[q + 1] << 8 | I.p[q + 2] << 16 | (u32)I.p[q + 3] << 24;
			E.isize = I.p[q + 4] | I.p[q + 5] << 8 | I.p[q + 6] << 16 | (u32)I.p[q + 7] << 24;
			bit = (q + 8) * 8; mode = GZ_M_NEXT; mstart = (int)o;
			if (n_ev == GZ_EVCAP) GZ_END(GZ_S_FULL);
			continue;
		}
		if (mode == GZ_M_BLOCK) {
			if (bit >= C.stop) GZ_END(GZ_S_OK);
			B.seek(bit);
			hdr = bit;
			const u32 h = B.get(3);
			if (B.over()) { if (I.final) GZ_FAIL(bit); GZ_END(GZ_S_INPUT); }
			bfinal = h & 1; btype = h >> 1;
			if (btype == 3) GZ_FAIL(bit);
			if (btype == 2) {
				const int r = gz_dyn_header(B, T, false);
				if (r == -2 || (r == 0 && B.over())) { if (I.final) GZ_FAIL(bit); GZ_END(GZ_S_INPUT); }
				if (r) GZ_FAIL(bit);
			} else if (btype == 1) gz_fixed(T);
			else {
				const bz_u64 q = (B.pos() + 7) >> 3;
				if (q + 4 > I.n) { if (I.final) GZ_FAIL(bit); GZ_END(GZ_S_INPUT); }
				const u32 len = I.p[q] | I.p[q + 1] << 8, nlen = I.p[q + 2] | I.p[q + 3] << 8;
				if (len != (~nlen & 0xffff)) GZ_FAIL(bit);
				left = len;
				B.seek((q + 4) * 8);
			}
			mode = GZ_M_IN;
		}
		// inside a block: B is at the next symbol (or stored byte)
		if (btype == 0) {
			bz_u64 q = B.pos() >> 3;
			while (left) {
				if (q >= I.n) { bit = q * 8; if (I.final) GZ_FAIL(bit); GZ_END(GZ_S_INPUT); }
				if (o == GZ_SLOT) { bit = q * 8; GZ_END(GZ_S_FULL); }
				slot[o++] = I.p[q++]; --left;
			}
			bit = q * 8;
		} else {
			for (;;) {
				bit = B.pos();
				const int s = gz_sym(B, T.lfast, GZ_LFB, T.lcnt, T.lsym);
				if (B.over()) { if (I.final) GZ_FAIL(bit); GZ_END(GZ_S_INPUT); }
				if (s < 0 || s > 285) GZ_FAIL(bit);
				if (s < 256) {
					if (o == GZ_SLOT) GZ_END(GZ_S_FULL);
					slot[o++] = (uint16_t)s;
					continue;
				}
				if (s == 256) break;
				const u32 len = gz_len_base((u32)s) + B.get(bz_len_nx((u32)s));
				const int d = gz_sym(B, T.dfast, GZ_DFB, T.dcnt, T.dsym);
				if (d < 0 || d > 29) { if (B.over()) { if (I.final) GZ_FAIL(bit); GZ_END(GZ_S_INPUT); } GZ_FAIL(bit); }
				const u32 dist = gz_dist_base((u32)d) + B.get(bz_dist_nx((u32)d));
				if (B.over()) { if (I.final) GZ_FAIL(bit); GZ_END(GZ_S_INPUT); }
				const int src = (int)o - (int)dist;
				if (src < mstart || src < -(int)GZ_CTX) GZ_FAIL(bit); // reaches before the member (or the deflate window)
				if (o + len > GZ_SLOT) GZ_END(GZ_S_FULL);
				for (u32 k = 0; k < len; ++k, ++o) {
					const int j = src + (int)k;
					if (j >= 0) slot[o] = slot[j];
					else { const u32 p = (u32)(j + (int)GZ_CTX); slot[o] = (uint16_t)(256 + p); if (p < min_ph) min_ph = p; }
				}
			}
			bit = B.pos();
		}
		mode = bfinal ? GZ_M_TRAILER : GZ_M_BLOCK;
		if (bfinal) bit = (bit + 7) & ~7ull;
	}
done:
#undef GZ_END
#undef GZ_FAIL
	C.end.bit = bit; C.end.hdr = mode == GZ_M_IN ? hdr : bit; C.end.mode = mode;
	C.len = o; C.n_ev = n_ev; C.min_ph = min_ph;
}

// ---- resolve: symbols of chunk i (at text offset off) -> bytes; wout = [32 KB context][text] ----
SSQ_HD void gz_resolve_range(const uint16_t *slot, bz_u64 off, u32 lo, u32 hi, uint8_t *wout, u32 t, u32 nt)
{
	for (u32 o = lo + t; o < hi; o += nt) {
		const u32 v = slot[o];
		wout[GZ_CTX + off + o] = v < 256 ? (uint8_t)v : wout[off + (v - 256)];
	}
}
// ---- CRC-32 of one piece (zlib convention) ----
SSQ_HD u32 gz_crc_piece(const uint32_t *tab, const uint8_t *p, u32 n)
{
	u32 c = 0xffffffffu;
	for (u32 i = 0; i < n; ++i) c = tab[(c ^ p[i]) & 0xff] ^ (c >> 8);
	return ~c;
}

// =============================================================== host logic: one window ====
// Backend: where the phases run (the device in ssq_gunzip.cu, host loops in tests/hostsim/gunzip_host.cpp).  Chunk records and
// events are mirrored on the host between phases.
struct GzBackend {
	virtual ~GzBackend() {}
	virtual int sync(const GzIn &I, int n, bz_u64 lo, bz_u64 cbits, bz_u64 wend, bz_u64 *s) = 0;   // s[1..n-1]
	virtual int decode(const GzIn &I, const std::vector<int> &which, GzChunk *ch, GzEvent *ev) = 0; // ch/ev: host mirrors, all chunks
	virtual int resolve(int n, const u32 *len, const bz_u64 *off) = 0;                              // chunk k of the chain -> text
	virtual int crc(const std::vector<bz_u64> &off, const std::vector<u32> &len, std::vector<u32> &out) = 0;
};

struct GzState {                  // what carries from window to window
	GzPos pos;                    // where the next window starts (positions relative to the current input)
	u32 crc, isize;               // running CRC-32 and length of the current member
	long long mstart;             // text offset of the current member's start, relative to the next window's text
	bz_u64 total;                 // text so far
	int eos;
	int64_t stats[4];             // chunks decoded, chunks started at a searched sync, chunks re-decoded, windows
};
static inline void gz_state_init(GzState &S)
{
	memset(&S, 0, sizeof S);
	S.pos.bit = 0; S.pos.hdr = 0; S.pos.mode = GZ_M_FIRST;
}

// one window over I from S.pos: on success the text is in the backend's [context][text] buffer, *text = its length, S carries.
// Returns 0, or SSQ_EDATA with *err_at = compressed byte offset (relative to I)
static inline int gz_window(GzBackend &be, GzState &S, const GzIn &I, bz_u64 chunk_bytes, std::vector<GzChunk> &ch, std::vector<GzEvent> &ev,
                            bz_u64 *text, bz_u64 *err_at)
{
	const bz_u64 cbits = chunk_bytes * 8, lo = S.pos.bit, inbits = I.n * 8;
	bz_u64 wend = lo + cbits * GZ_MAXCH;
	if (wend > inbits) wend = inbits;
	int n = wend > lo ? (int)((wend - lo + cbits - 1) / cbits) : 1;
	if (n < 1) n = 1;
	std::vector<bz_u64> s(n, GZ_NONE);
	int rc;
	if (n > 1 && (rc = be.sync(I, n, lo, cbits, wend, s.data()))) return rc;
	// the chain: chunk 0 at the carry, then every chunk with a sync point
	std::vector<bz_u64> starts(1, lo);
	for (int i = 1; i < n; ++i) if (s[i] != GZ_NONE) starts.push_back(s[i]);
	const int m = (int)starts.size();
	ch.assign(m, GzChunk());
	ev.assign((size_t)m * GZ_EVCAP, GzEvent());
	std::vector<int> which(m);
	for (int k = 0; k < m; ++k) {
		GzChunk &c = ch[k];
		if (k == 0) c.start = S.pos; else { c.start.bit = c.start.hdr = starts[k]; c.start.mode = GZ_M_BLOCK; }
		c.stop = k + 1 < m ? starts[k + 1] : wend;
		if (k + 1 == m && wend == inbits) c.stop = GZ_NONE; // the last chunk runs to the end of the input
		which[k] = k;
	}
	S.stats[0] += m; S.stats[1] += m - 1; S.stats[3] += 1;
	if ((rc = be.decode(I, which, ch.data(), ev.data()))) return rc;
	auto linked = [&](int k) { const GzPos &a = ch[k].end, &b = ch[k + 1].start; return a.bit == b.bit && a.hdr == b.hdr && a.mode == b.mode; };
	int last;
	for (;;) {
		int k = 0;
		while (k + 1 < m && (ch[k].status == GZ_S_OK || ch[k].status == GZ_S_FULL) && linked(k)) ++k;
		if (k + 1 == m || ch[k].status == GZ_S_BAD || ch[k].status == GZ_S_EOS || ch[k].status == GZ_S_INPUT) { last = k; break; }
		which.clear();
		for (int j = k; j + 1 < m; ++j)
			if ((ch[j].status == GZ_S_OK || ch[j].status == GZ_S_FULL) && !linked(j)) { ch[j + 1].start = ch[j].end; which.push_back(j + 1); }
		S.stats[2] += (int64_t)which.size();
		if ((rc = be.decode(I, which, ch.data(), ev.data()))) return rc;
	}
	if (ch[last].status == GZ_S_BAD) { *err_at = ch[last].bad >> 3; return SSQ_EDATA; }
	// layout, references across chunks into earlier members, CRC pieces
	std::vector<u32> len(last + 1);
	std::vector<bz_u64> off(last + 1);
	std::vector<bz_u64> poff; std::vector<u32> plen;
	std::vector<int> pmember;     // piece -> index of the member end it belongs to (-1: still open)
	struct End { u32 crc, isize; bz_u64 at, out; };
	std::vector<End> ends;
	bz_u64 at = 0;
	long long mstart = S.mstart;
	bz_u64 seg = 0;               // start of the current member's text in this window
	auto pieces = [&](bz_u64 a, bz_u64 b, int member) { for (bz_u64 x = a; x < b; x += GZ_CRC_PIECE) { poff.push_back(x); plen.push_back((u32)(b - x < GZ_CRC_PIECE ? b - x : GZ_CRC_PIECE)); pmember.push_back(member); } };
	for (int k = 0; k <= last; ++k) {
		const GzChunk &c = ch[k];
		len[k] = c.len; off[k] = at;
		if (c.min_ph < GZ_CTX && (long long)at - (long long)GZ_CTX + (long long)c.min_ph < mstart) { *err_at = c.start.bit >> 3; return SSQ_EDATA; }
		for (u32 e = 0; e < c.n_ev; ++e) {
			const GzEvent &E = ev[(size_t)k * GZ_EVCAP + e];
			pieces(seg, at + E.out, (int)ends.size());
			ends.push_back({E.crc, E.isize, E.at, at + E.out});
			seg = at + E.out; mstart = (long long)seg;
		}
		at += c.len;
	}
	pieces(seg, at, -1);
	if ((rc = be.resolve(last + 1, len.data(), off.data()))) return rc;
	std::vector<u32> pc;
	if ((rc = be.crc(poff, plen, pc))) return rc;
	size_t p = 0;
	for (size_t e = 0; e <= ends.size(); ++e) {
		for (; p < poff.size() && pmember[p] == (e < ends.size() ? (int)e : -1); ++p) { S.crc = bz_multmodp(bz_x8n(plen[p]), S.crc) ^ pc[p]; S.isize += plen[p]; }
		if (e == ends.size()) break;
		if (S.crc != ends[e].crc || S.isize != ends[e].isize) { *err_at = ends[e].at; return SSQ_EDATA; }
		S.crc = 0; S.isize = 0;
	}
	S.pos = ch[last].end;
	S.eos = ch[last].status == GZ_S_EOS;
	S.mstart = mstart - (long long)at;
	S.total += at;
	*text = at;
	return SSQ_OK;
}
// input bytes before a position that no later window reads
static inline bz_u64 gz_consumed(const GzPos &p) { return (p.mode == GZ_M_IN ? p.hdr : p.bit) >> 3; }
static inline void gz_rebase(GzPos &p, bz_u64 bytes) { p.bit -= bytes * 8; p.hdr -= bytes * 8; }

// a whole stream in p[0, n): windows until the end of the stream; emit(text) takes each window's text out of the backend
template <class Emit>
static inline int gz_run(GzBackend &be, GzState &S, const uint8_t *p, bz_u64 n, bz_u64 chunk_bytes, Emit emit, bz_u64 *err_at)
{
	std::vector<GzChunk> ch; std::vector<GzEvent> ev;
	bz_u64 base = 0;
	while (!S.eos) {
		GzIn I; I.p = p + base; I.n = n - base; I.final = 1;
		bz_u64 text = 0, at = 0;
		const GzPos before = S.pos;
		int rc = gz_window(be, S, I, chunk_bytes, ch, ev, &text, &at);
		if (rc == SSQ_EDATA) *err_at = base + at;
		if (rc) return rc;
		if ((rc = emit(text))) return rc;
		if (!S.eos && !text && S.pos.bit == before.bit && S.pos.mode == before.mode) { *err_at = base + (S.pos.bit >> 3); return SSQ_EDATA; }
		const bz_u64 c = gz_consumed(S.pos);
		gz_rebase(S.pos, c); base += c;
	}
	return SSQ_OK;
}
