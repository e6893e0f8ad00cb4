// seed_sector_host.cpp — TEST-ONLY: the paired rank query of the seeding (ScalarFm::occ4_pair in speedseq_b200/csrc/ssq_dev.cuh)
// compiled for the host and compared with two single queries (ScalarFm::occ4) on the re-blocked 32-byte rank structure of an
// oracle-built index.  Built into a temporary directory by tests/test_seed_sector_cpu.py; not part of libssq.so.
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../speedseq_b200/csrc/ssq_dev.cuh"
extern "C" {
#include "../../oracle/ssqo.h"
}

// the 64-row, 32-byte blocks k_reblock32 (ssq_index.cu) derives from the on-disk 128-row, 64-byte blocks
static void reblock32(const ssqo_idx_t *o, std::vector<u32> &out)
{
	const u64 n = o->bwt.seq_len, nb = (n + 63) / 64 + 1;
	out.assign(nb * 8, 0);
	for (u64 b = 0; b < nb; ++b) {
		const u32 *src = o->bwt.bwt + ((b >> 1) << 4);
		const u64 *c64 = (const u64*)src;
		u32 add[4] = {0, 0, 0, 0};
		if (b & 1) for (int i = 0; i < 64; ++i) ++add[src[8 + (i >> 4)] >> ((~i & 15) << 1) & 3];
		const bool have = ((b >> 1) << 7) < n + 128; // within the stored blocks (incl. the final count block)
		for (int c = 0; c < 4; ++c) out[b * 8 + c] = have ? (u32)(c64[c] + add[c]) : 0;
		for (int w = 0; w < 4; ++w) out[b * 8 + 4 + w] = (((b >> 1) << 7) + (b & 1) * 64 + w * 16 < n) ? src[8 + (b & 1) * 4 + w] : 0;
	}
}

// Every pair of rows (k0 - 1, k1) with k0 in [lo, hi) and k0 <= k1 < k0 + span (the row before an interval [k0, k1] and its last
// row; k0 = 0: no row before it), with the index's primary row moved to `primary`: the '$' row shifts every later row by one, so
// its place in its block decides which block each row falls in.  Returns the number of pairs whose counts differ from two single
// queries; n_one / n_two: pairs answered from one / two sectors.
extern "C" long long seed_sector_pair_check(const void *oidx, unsigned long long primary, unsigned long long lo, unsigned long long hi, int span,
                                            unsigned long long *n_one, unsigned long long *n_two)
{
	const ssqo_idx_t *o = (const ssqo_idx_t*)oidx;
	std::vector<u32> b32;
	reblock32(o, b32);
	DevIndex ix;
	memset(&ix, 0, sizeof ix);
	ix.bwt = o->bwt.bwt; ix.bwt32 = b32.data(); ix.seq_len = o->bwt.seq_len; ix.primary = primary;
	memcpy(ix.L2, o->bwt.L2, sizeof ix.L2);
	ScalarFm fm(ix);
	long long bad = 0;
	*n_one = *n_two = 0;
	for (u64 k0 = lo; k0 < hi; ++k0)
		for (u64 k1 = k0; k1 < k0 + (u64)span && k1 < ix.seq_len; ++k1) {
			u32 a[4], b[4], c[4], d[4];
			const u32 k0r = k0 == 0 ? (u32)-1 : (u32)(k0 - 1);
			fm.occ4(k0r, a); fm.occ4((u32)k1, b);
			const u32 before = fm.n_blk;
			fm.occ4_pair(k0r, (u32)k1, c, d);
			(fm.n_blk - before == 1 ? *n_one : *n_two) += 1;
			for (int t = 0; t < 4; ++t) bad += a[t] != c[t] || b[t] != d[t];
		}
	return bad;
}
