// ssq_sbtext.cuh — samblaster's stage over name-grouped SAM text (the `samblaster` shim's unfused input) as SSQ_HD routines:
// csrc/ssq_sbtext.cu runs them as kernels (a thread per line, a thread per QNAME block), tests/hostsim/sbtext_host.cpp runs the
// same routines in plain loops.  The decisions themselves are the sb_* routines of ssq_dev3.cuh that the fused stage uses; what
// is here is reading them their inputs from the text and writing the three streams back as text.
//   sbt_parse_line   tab offsets, FLAG, POS, CIGAR (ops as sb_geometry takes them), RNAME -> contig id, MC:Z / MQ:i present
//   sbt_block        primary lines (samblaster's rule: the last of each kind, 0x900 lines skipped), signature, discordant and
//                    splitter marks, the mate line whose CIGAR / MAPQ go into MC:Z / MQ:i
//   sbt_line_text    one line's bytes in each of the three streams (W = false: sizes only)
// Lines the device refuses (the call returns SSQ_EFORMAT and consumes nothing, so the caller runs its host code over them):
// fewer than 11 fields, a NUL byte, FLAG not 1-9 digits, POS not 1-18 digits, a CIGAR other than `*` or (1-9 digits, one of
// MIDNSHP=X)+ with every length below 2^28, an RNAME other than `*` that no @SQ line names, a QNAME block of more than
// SBT_MAX_BLOCK lines, and a primary line that a signature needs whose RNAME is `*` while FLAG says it is mapped.
#pragma once
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <string>
#include <vector>
#include "ssq_dev3.cuh"

#define SBT_MAX_BLOCK 256 // lines per QNAME block the device takes
#define SBT_STR_(x) #x
#define SBT_STR(x) SBT_STR_(x)

enum { SBT_OK = 0, SBT_E_FIELDS, SBT_E_NUL, SBT_E_FLAG, SBT_E_POS, SBT_E_CIGAR, SBT_E_RNAME, SBT_E_BLOCK, SBT_E_NOREF };

struct SbtLine {
	u32 beg, end;            // the line in the text, without its '\n'
	u32 qend, fend;          // end of QNAME, end of FLAG (both at a tab)
	u32 mq_beg, cig_beg, cig_end; // MAPQ field = [mq_beg, cig_beg - 1), CIGAR field = [cig_beg, cig_end); ops at ops[cig_beg / 2 ..)
	i32 flag, rid, n_cig;    // rid: first @SQ with that SN, -1 for `*`
	i64 pos1;                // the POS field
	i32 mate;                // line whose CIGAR / MAPQ fields MC:Z / MQ:i copy, -1 none (set per block)
	u32 blk;                 // block of the line (set per block)
	uint8_t has_mc, has_mq, err, mark; // mark: 1 splitter, 2 discordant (set per block)
};

// @SQ names: open addressing over FNV-1a; a slot holds the first contig id with that name, -1 empty
struct SbtCtg { const char *names; const u32 *name_off; const i32 *slot; u32 mask; };
SSQ_HD u32 sbt_hash(const char *s, u32 n) { u32 h = 2166136261u; for (u32 i = 0; i < n; ++i) { h ^= (uint8_t)s[i]; h *= 16777619u; } return h; }
SSQ_HD bool sbt_eq(const char *a, u32 na, const char *b, u32 nb) { if (na != nb) return false; for (u32 i = 0; i < na; ++i) if (a[i] != b[i]) return false; return true; }
SSQ_HD int sbt_find(const SbtCtg &C, const char *s, u32 n) // contig id, -1 absent
{
	for (u32 h = sbt_hash(s, n) & C.mask;; h = (h + 1) & C.mask) {
		const int id = C.slot[h];
		if (id < 0) return -1;
		if (sbt_eq(C.names + C.name_off[id], C.name_off[id + 1] - C.name_off[id], s, n)) return id;
	}
}

// digits only, at least one, at most maxd; false otherwise
SSQ_HD bool sbt_digits(const char *t, u32 a, u32 b, int maxd, i64 *v)
{
	if (b <= a || b - a > (u32)maxd) return false;
	i64 x = 0;
	for (u32 i = a; i < b; ++i) { const char c = t[i]; if (c < '0' || c > '9') return false; x = x * 10 + (c - '0'); }
	*v = x;
	return true;
}
// CIGAR text -> ops in the encoding sb_geometry takes (M = X: 0, I 1, D N 2, S 3, H 4; P leaves no op); false if not fully consumed
SSQ_HD bool sbt_cigar(const char *t, u32 a, u32 b, u32 *ops, i32 *n_ops)
{
	*n_ops = 0;
	if (b == a + 1 && t[a] == '*') return true;
	if (b <= a) return false;
	int n = 0;
	for (u32 i = a; i < b;) {
		u32 len = 0; int nd = 0;
		while (i < b && t[i] >= '0' && t[i] <= '9' && nd < 10) { len = len * 10 + (u32)(t[i] - '0'); ++i; ++nd; }
		if (nd == 0 || nd > 9 || i >= b || len >= (1u << 28)) return false;
		int op;
		switch (t[i]) {
		case 'M': case '=': case 'X': op = 0; break;
		case 'I': op = 1; break;
		case 'D': case 'N': op = 2; break;
		case 'S': op = 3; break;
		case 'H': op = 4; break;
		case 'P': op = -1; break;
		default: return false;
		}
		++i;
		if (op >= 0) ops[n++] = len << 4 | (u32)op;
	}
	*n_ops = n;
	return true;
}

// one line [beg, end) of the text
SSQ_HD void sbt_parse_line(const char *t, u32 beg, u32 end, const SbtCtg &C, u32 *ops, SbtLine &L)
{
	L.beg = beg; L.end = end; L.qend = L.fend = L.mq_beg = L.cig_beg = L.cig_end = beg;
	L.flag = 0; L.rid = -1; L.n_cig = 0; L.pos1 = 0; L.mate = -1; L.blk = 0; L.has_mc = L.has_mq = 0; L.err = SBT_OK; L.mark = 0;
	int f = 0, err = SBT_OK;
	u32 fs = beg;
	for (u32 i = beg;; ++i) {
		if (i < end && t[i] == 0 && !err) err = SBT_E_NUL;
		if (i < end && t[i] != '\t') continue;
		const u32 fe = i; // field f = [fs, fe)
		i64 v;
		switch (f) {
		case 0: L.qend = fe; break;
		case 1: L.fend = fe; if (sbt_digits(t, fs, fe, 9, &v)) L.flag = (i32)v; else if (!err) err = SBT_E_FLAG; break;
		case 2:
			if (fe == fs + 1 && t[fs] == '*') L.rid = -1;
			else if ((L.rid = sbt_find(C, t + fs, fe - fs)) < 0 && !err) err = SBT_E_RNAME;
			break;
		case 3: if (sbt_digits(t, fs, fe, 18, &v)) L.pos1 = v; else if (!err) err = SBT_E_POS; break;
		case 4: L.mq_beg = fs; break;
		case 5: L.cig_beg = fs; L.cig_end = fe; if (!sbt_cigar(t, fs, fe, ops + fs / 2, &L.n_cig) && !err) err = SBT_E_CIGAR; break;
		default:
			if (f >= 11 && fe - fs >= 5 && t[fs + 2] == ':' && t[fs + 4] == ':') {
				if (t[fs] == 'M' && t[fs + 1] == 'C' && t[fs + 3] == 'Z') L.has_mc = 1;
				if (t[fs] == 'M' && t[fs + 1] == 'Q' && t[fs + 3] == 'i') L.has_mq = 1;
			}
		}
		++f; fs = i + 1;
		if (i >= end) break;
	}
	if (f < 11) err = SBT_E_FIELDS;
	if (err) L.n_cig = 0;
	L.err = (uint8_t)err;
}
// does line i start a QNAME block (its QNAME differs from line i - 1's)?
SSQ_HD bool sbt_block_start(const char *t, const SbtLine *L, u32 i)
{
	if (i == 0) return true;
	const SbtLine &a = L[i - 1], &b = L[i];
	return !sbt_eq(t + a.beg, a.qend - a.beg, t + b.beg, b.qend - b.beg);
}

SSQ_HD SbLine sbt_sbline(const SbtLine &l, const u32 *ops) { SbLine s; s.flag = l.flag; s.rid = l.rid; s.shown = true; s.cig = ops + l.cig_beg / 2; s.n_cig = l.n_cig; s.pos1 = l.pos1; return s; }
SSQ_HD bool sbt_mapped_needs_ref(const SbtLine &l) { return !(l.flag & 0x4) && l.rid < 0; }

// block blk = lines [b0, b1): its signature (k1, k2, valid), and per line the block, the mate line and the marks.  Returns an
// SBT_E_* code when the device does not take the block (nothing is written to the signature then)
SSQ_HD int sbt_block(const SbOpts &o, const i64 *sb_off, const u32 *ops, SbtLine *L, u32 b0, u32 b1, u32 blk, u64 *k1, u64 *k2, uint8_t *valid)
{
	*k1 = *k2 = 0; *valid = 0;
	if (b1 - b0 > SBT_MAX_BLOCK) return SBT_E_BLOCK;
	int first = -1, second = -1;
	for (u32 i = b0; i < b1; ++i) {
		L[i].blk = blk; L[i].mate = -1; L[i].mark = 0;
		const int f = L[i].flag;
		if (f & 0x900) continue;
		if (!(f & 0x1)) second = (int)i;
		else if (f & 0x40) first = (int)i;
		else if (f & 0x80) second = (int)i;
	}
	bool ok = false, disc = false;
	if (first >= 0 && second >= 0) {
		for (u32 i = b0; i < b1; ++i) {
			if ((L[i].flag & 0xC0) == 0x40) L[i].mate = second;
			else if ((L[i].flag & 0xC0) == 0x80) L[i].mate = first;
		}
		const SbtLine &F = L[first], &S = L[second];
		if (!((F.flag & 0x4) && (S.flag & 0x4)) && (sbt_mapped_needs_ref(F) || sbt_mapped_needs_ref(S))) return SBT_E_NOREF;
		ok = sb_pair_signature(sbt_sbline(F, ops), sbt_sbline(S, ops), sb_off, k1, k2, &disc);
		if (disc) { L[first].mark |= 2; L[second].mark |= 2; }
	} else if (first >= 0 || second >= 0) {
		const SbtLine &only = L[first >= 0 ? first : second];
		if (sbt_mapped_needs_ref(only)) return SBT_E_NOREF;
		ok = sb_lone_signature(sbt_sbline(only, ops), sb_off, k1, k2);
	}
	*valid = ok ? 1 : 0;
	if (o.want_split) for (int side = 0x40; side <= 0x80; side += 0x40) {
		SbSplitLine sl[64]; u32 at[64];
		int count = 0;
		for (u32 i = b0; i < b1; ++i) {
			const int f = L[i].flag;
			if ((f & 0xC0) != side || (f & 0x100) || (f & 0x4)) continue;
			if (count < 64) {
				sl[count].g = sb_geometry(ops + L[i].cig_beg / 2, L[i].n_cig, true, L[i].pos1, (f & 0x10) != 0);
				sl[count].flag = f; sl[count].rid = L[i].rid; at[count] = i;
			}
			++count;
		}
		const u64 m = count <= 64 ? sb_splitters(o, sl, count) : 0;
		for (int k = 0; k < count && k < 64; ++k) if (m >> k & 1) L[at[k]].mark |= 1;
	}
	return SBT_OK;
}

// one record: QNAME (+ _suffix), FLAG re-printed, the rest of the line verbatim, MC:Z / MQ:i from the mate line when absent
template <bool W>
SSQ_HD void sbt_record(Sink<W> &s, const char *t, const SbtLine *L, u32 i, int flag, char suffix, bool tags)
{
	const SbtLine &l = L[i];
	sputs(s, t + l.beg, (int)(l.qend - l.beg));
	if (suffix) { sput(s, '_'); sput(s, suffix); }
	sput(s, '\t');
	sputn(s, flag);
	sputs(s, t + l.fend, (int)(l.end - l.fend));
	if (tags && l.mate >= 0) {
		const SbtLine &m = L[l.mate];
		if (!l.has_mc) { sputs(s, "\tMC:Z:", 6); sputs(s, t + m.cig_beg, (int)(m.cig_end - m.cig_beg)); }
		if (!l.has_mq) { sputs(s, "\tMQ:i:", 6); sputs(s, t + m.mq_beg, (int)(m.cig_beg - 1 - m.mq_beg)); }
	}
	sput(s, '\n');
}
// line i in the three streams (0 main, 1 splitters, 2 discordants); dup = its block is a duplicate
template <bool W>
SSQ_HD void sbt_line_text(const SbOpts &o, const char *t, const SbtLine *L, u32 i, bool dup, Sink<W> out[3])
{
	const SbtLine &l = L[i];
	const int flag = l.flag | (dup ? 0x400 : 0);
	const bool tags = o.addMateTags != 0;
	if (!(o.removeDups && dup)) sbt_record(out[0], t, L, i, flag, 0, tags);
	if (o.want_disc && (l.mark & 2) && !(o.excludeDups && dup)) sbt_record(out[2], t, L, i, flag, 0, tags);
	if (o.want_split && (l.mark & 1) && !(o.excludeDups && dup)) sbt_record(out[1], t, L, i, flag, (flag & 0x1) ? ((flag & 0x40) ? '1' : '2') : 0, tags);
}

// ---- host side, shared by the device driver and the host restatement ----
SSQ_HD SbOpts sbt_opts(const ssq_sb_opts_t &s)
{
	SbOpts o;
	o.enabled = 1; o.excludeDups = s.exclude_dups; o.addMateTags = s.add_mate_tags; o.maxSplitCount = s.max_split_count; o.minNonOverlap = s.min_non_overlap;
	o.minIndelSize = s.min_indel_size; o.maxUnmappedBases = s.max_unmapped_bases; o.removeDups = s.remove_dups; o.want_split = s.want_split; o.want_disc = s.want_disc;
	return o;
}
// the @SQ lines of a header as samblaster reads them: SN = the bytes after the first "\tSN:" up to a tab or newline (at most
// 1023), padded offset += LN + 2 * 500 + 1 for every @SQ line that has both, names looked up first occurrence first
struct SbtHeader { std::vector<char> names; std::vector<u32> name_off; std::vector<i64> off; std::vector<i32> slot; u32 mask; };
static inline const char *sbt_memstr(const char *a, const char *b, const char *pat)
{
	const size_t n = strlen(pat);
	for (const char *p = a; p + n <= b; ++p) if (!memcmp(p, pat, n)) return p;
	return 0;
}
static inline void sbt_parse_header(const char *h, size_t n, SbtHeader &H)
{
	i64 total = 0;
	H.name_off.assign(1, 0);
	for (size_t a = 0; a < n;) {
		size_t b = a;
		while (b < n && h[b] != '\n') ++b;
		const char *l = h + a, *le = h + b;
		if (b - a >= 4 && !memcmp(l, "@SQ\t", 4)) {
			const char *p = sbt_memstr(l, le, "\tSN:"), *q = sbt_memstr(l, le, "\tLN:");
			if (p && q) {
				const char *s = p + 4, *e = s;
				while (e < le && *e != '\t' && e - s < 1023) ++e;
				H.names.insert(H.names.end(), s, e);
				H.name_off.push_back((u32)H.names.size());
				H.off.push_back(total);
				total += atoll(std::string(q + 4, le).c_str()) + 2 * SB_PAD + 1;
			}
		}
		a = b + 1;
	}
	const u32 nc = (u32)H.off.size();
	u32 cap = 16;
	while (cap < 2 * nc) cap <<= 1;
	H.mask = cap - 1;
	H.slot.assign(cap, -1);
	for (u32 i = 0; i < nc; ++i) {
		const char *s = H.names.data() + H.name_off[i]; const u32 len = H.name_off[i + 1] - H.name_off[i];
		for (u32 k = sbt_hash(s, len) & H.mask;; k = (k + 1) & H.mask) {
			const int id = H.slot[k];
			if (id < 0) { H.slot[k] = (i32)i; break; }
			if (sbt_eq(H.names.data() + H.name_off[id], H.name_off[id + 1] - H.name_off[id], s, len)) break; // first SN wins
		}
	}
	if (H.names.empty()) H.names.push_back(0);
	if (H.off.empty()) H.off.push_back(0);
}
// how many blocks a call takes: the last block waits for more text unless final (the next line may continue it), max_blocks
// (0 = no limit) caps the count.  The call then consumes the text up to the first line of block `take`, or all of it when final
// and every block was taken
static inline u64 sbt_take(u64 n_blocks, int final, u64 max_blocks)
{
	u64 take = final ? n_blocks : (n_blocks ? n_blocks - 1 : 0);
	if (max_blocks && take > max_blocks) take = max_blocks;
	return take;
}
static inline const char *sbt_err_text(int code)
{
	switch (code) {
	case SBT_E_FIELDS: return "fewer than 11 fields";
	case SBT_E_NUL: return "a NUL byte";
	case SBT_E_FLAG: return "FLAG is not 1-9 digits";
	case SBT_E_POS: return "POS is not 1-18 digits";
	case SBT_E_CIGAR: return "a CIGAR the device parser does not take";
	case SBT_E_RNAME: return "an RNAME that is not in @SQ";
	case SBT_E_BLOCK: return "a QNAME block of more than " SBT_STR(SBT_MAX_BLOCK) " lines";
	case SBT_E_NOREF: return "a mapped primary line with RNAME '*'";
	}
	return "?";
}
// the SSQ_EFORMAT message: line numbers count from 1 at the start of the call's text
static inline void sbt_refusal(char *buf, size_t cap, u64 line, u64 byte, int code, const char *text, size_t len)
{
	size_t n = 0;
	while (n < 60 && byte + n < len && text[byte + n] != '\n' && text[byte + n] != 0) ++n;
	snprintf(buf, cap, "SAM text the device does not take: line %llu (byte %llu): %s: '%.*s%s'", (unsigned long long)line + 1, (unsigned long long)byte,
	         sbt_err_text(code), (int)n, text + byte, n == 60 ? "..." : "");
}
