// bgzf_host.cpp — TEST-ONLY: the BGZF member encoder of speedseq_b200/csrc/ssq_bgzf.cu run on the host.  Every member goes
// through the SSQ_HD phases of ssq_bgzf.cuh in the order the kernel runs them, each phase as a loop over the BZ_NT thread indices
// (a barrier between phases = the end of a loop).  The block-wide exclusive scan of the token bit lengths is restated as the plain
// prefix sum it computes.  Output = what ssq_bgzf_deflate returns for the same input and level, byte for byte.
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../speedseq_b200/csrc/ssq_bgzf.cuh"

static void encode_member(BzSmem &S, const BzJob &J, int level)
{
	for (int t = 0; t < BZ_NT; ++t) bz_load(S, J, level, t);
	for (int t = 0; t < BZ_NT; ++t) bz_crc(S, t);
	for (u32 base = 0; base < S.n; base += BZ_NT) {
		for (int t = 0; t < BZ_NT; ++t) bz_find(S, base, t);
		for (int t = 0; t < BZ_NT; ++t) bz_insert_parse(S, J, base, t);
	}
	for (int t = 0; t < BZ_NT; ++t) bz_hist(S, J, t);
	for (int t = 0; t < BZ_NT; ++t) bz_rank(S, t);
	bz_plan(S);
	for (int t = 0; t < BZ_NT; ++t) bz_zero(S, J, t);
	bz_header(S, J);
	for (int t = 0; t < BZ_NT; ++t) bz_stored_copy(S, J, t);
	bz_u64 run = S.hdr_bits;
	for (u32 c = 0; c < S.ntok; c += BZ_NT) {
		bz_u64 v[BZ_NT]; u32 nb[BZ_NT];
		for (int t = 0; t < BZ_NT; ++t) nb[t] = bz_tok_bits(S, J, c + t, &v[t]);
		for (int t = 0; t < BZ_NT; ++t) { if (nb[t]) bz_put((bz_u64*)(J.slot + BZ_SLOT_BITS), run, v[t], nb[t]); run += nb[t]; }
	}
	bz_eob(S, J, run);
	bz_finish(S, J);
}

extern "C" int hostsim_bgzf(const void *in, size_t n, int level, int with_eof, void **out, size_t *out_len)
{
	static const unsigned char eof_blk[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};
	const size_t n_blk = (n + BZ_PAYLOAD - 1) / BZ_PAYLOAD;
	std::vector<bz_u64> slot(BZ_SLOT / 8);
	std::vector<u32> tok(BZ_PAYLOAD);
	BzSmem *S = new BzSmem;
	unsigned char *o = (unsigned char*)malloc(n_blk * 65536 + 28 + 1);
	size_t at = 0;
	for (size_t b = 0; b < n_blk; ++b) {
		u32 size = 0;
		BzJob J;
		J.src = (const uint8_t*)in + b * BZ_PAYLOAD; J.n = (u32)(b + 1 < n_blk ? BZ_PAYLOAD : n - b * BZ_PAYLOAD);
		J.tok = tok.data(); J.slot = (uint8_t*)slot.data(); J.size = &size;
		encode_member(*S, J, level);
		memcpy(o + at, J.slot + BZ_SLOT_MEMBER, size);
		at += size;
	}
	delete S;
	if (with_eof) { memcpy(o + at, eof_blk, 28); at += 28; }
	*out = o; *out_len = at;
	return 0;
}
extern "C" void hostsim_free(void *p) { free(p); }
