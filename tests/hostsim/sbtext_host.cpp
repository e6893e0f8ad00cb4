// sbtext_host.cpp — TEST-ONLY: ssq_sbtext_run (speedseq_b200/csrc/ssq_sbtext.cu) run on the host.  The same SSQ_HD routines of
// ssq_sbtext.cuh in the order the kernels run them, each kernel as a plain loop over its thread indices; the line and block
// selects are the loops they compute, and the dup-set is "first signature seen wins" over a std::set.  Same contract as the device
// call: whole QNAME blocks, the last one held back unless final, SSQ_EFORMAT with nothing consumed for lines the device refuses.
#include <set>
#include <string>
#include <utility>
#include "../../speedseq_b200/csrc/ssq_sbtext.cuh"

struct HsSbt {
	SbtHeader H; SbOpts o;
	std::set<std::pair<u64, u64> > seen;
	std::string out[3];
};
static char hs_err[512];

extern "C" void *hs_sbt_create(const char *hdr, size_t n, const ssq_sb_opts_t *sb)
{
	HsSbt *s = new HsSbt();
	sbt_parse_header(hdr, n, s->H);
	s->o = sbt_opts(*sb);
	return s;
}
extern "C" void hs_sbt_free(void *h) { delete (HsSbt*)h; }
extern "C" const char *hs_sbt_error(void) { return hs_err; }

extern "C" int hs_sbt_run(void *h, const char *t, size_t len, int final, uint64_t max_blocks, size_t *used, ssq_sbtext_out_t *out)
{
	HsSbt &S = *(HsSbt*)h;
	*used = 0;
	memset(out, 0, sizeof *out);
	if (len >= 0x7fffffffull) return SSQ_EINVAL;
	// lines: a flag per byte, select
	std::vector<u32> beg, end;
	u32 at = 0;
	for (u32 i = 0; i < (u32)len; ++i) if (t[i] == '\n') { beg.push_back(at); end.push_back(i); at = i + 1; }
	if (final && at < (u32)len) { beg.push_back(at); end.push_back((u32)len); }
	const u64 n_lines = beg.size();
	// fields, a thread per line
	std::vector<u32> ops(len / 2 + 1);
	std::vector<SbtLine> L(n_lines + 1);
	SbtCtg C; C.names = S.H.names.data(); C.name_off = S.H.name_off.data(); C.slot = S.H.slot.data(); C.mask = S.H.mask;
	for (u64 i = 0; i < n_lines; ++i) sbt_parse_line(t, beg[i], end[i], C, ops.data(), L[i]);
	// blocks
	std::vector<u32> bstart;
	for (u64 i = 0; i < n_lines; ++i) if (sbt_block_start(t, L.data(), (u32)i)) bstart.push_back((u32)i);
	const u64 n_blocks = bstart.size(), take = sbt_take(n_blocks, final, max_blocks), lines = take < n_blocks ? bstart[take] : n_lines;
	bstart.push_back((u32)n_lines);
	// a thread per block, then the first refused line
	std::vector<u64> k1(take), k2(take);
	std::vector<uint8_t> valid(take), dup(take);
	u64 first_err = ~0ull;
	for (u64 b = 0; b < take; ++b) {
		const int e = sbt_block(S.o, S.H.off.data(), ops.data(), L.data(), bstart[b], bstart[b + 1], (u32)b, &k1[b], &k2[b], &valid[b]);
		if (e && ((u64)bstart[b] << 8 | e) < first_err) first_err = (u64)bstart[b] << 8 | e;
	}
	for (u64 i = 0; i < lines; ++i) if (L[i].err && (i << 8 | L[i].err) < first_err) first_err = i << 8 | L[i].err;
	if (first_err != ~0ull) {
		sbt_refusal(hs_err, sizeof hs_err, first_err >> 8, beg[first_err >> 8], (int)(first_err & 0xff), t, len);
		return SSQ_EFORMAT;
	}
	// duplicates, in block order
	for (u64 b = 0; b < take; ++b) {
		dup[b] = 0;
		if (valid[b] && !S.seen.insert(std::make_pair(k1[b], k2[b])).second) dup[b] = 1;
		out->n_dup += dup[b];
	}
	// sizes, offsets (the scan), bytes
	for (int k = 0; k < 3; ++k) S.out[k].clear();
	std::vector<u64> off[3];
	for (int k = 0; k < 3; ++k) off[k].assign(lines + 1, 0);
	for (u64 i = 0; i < lines; ++i) {
		Sink<false> o[3];
		for (int k = 0; k < 3; ++k) { o[k].p = 0; o[k].n = 0; }
		sbt_line_text(S.o, t, L.data(), (u32)i, dup[L[i].blk] != 0, o);
		for (int k = 0; k < 3; ++k) off[k][i + 1] = off[k][i] + o[k].n;
		out->n_split_lines += o[1].n != 0; out->n_disc_lines += o[2].n != 0;
	}
	for (int k = 0; k < 3; ++k) S.out[k].resize(off[k][lines]);
	for (u64 i = 0; i < lines; ++i) {
		Sink<true> o[3];
		for (int k = 0; k < 3; ++k) { o[k].p = &S.out[k][0] + off[k][i]; o[k].n = 0; }
		sbt_line_text(S.o, t, L.data(), (u32)i, dup[L[i].blk] != 0, o);
	}
	for (int k = 0; k < 3; ++k) { out->text[k] = S.out[k].data(); out->len[k] = S.out[k].size(); }
	out->n_ids = take;
	*used = take < n_blocks ? beg[lines] : (final ? len : 0);
	return SSQ_OK;
}
