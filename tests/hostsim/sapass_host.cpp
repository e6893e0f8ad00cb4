// sapass_host.cpp — TEST-ONLY: the multi-pass suffix sort of speedseq_b200/csrc/ssq_sapass.cuh run on the host.  sp_build (the
// pass and chunk planners, the round loop, the finalisation ranges) runs unchanged against a backend whose "device" memory is
// host memory: every SSQ_HD body as a loop over its elements, std::stable_sort in place of the radix sort, plain loops in place
// of the scans.  Output files and stats (peak bytes apart from the sort's scratch) = what ssq_index_build_ex gives with path 2
// and the same working budget.  Also checks that every open member of round h has i + h <= n.
#include <stdarg.h>
#include <stdlib.h>
#include <stdio.h>
#include <algorithm>
#include <utility>
static int g_violation;
#define SP_ASSERT(c) do { if (!(c)) g_violation = 1; } while (0)
#include "../../speedseq_b200/csrc/ssq_sapass.cuh"

static char g_err[512];
void ssq_set_error(const char *fmt, ...)
{
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(g_err, sizeof g_err, fmt, ap);
	va_end(ap);
}

struct SpHost {
	u64 cur = 0, peak = 0;
	int need(SpBuf &b, u64 bytes)
	{
		if (bytes <= b.cap) return 0;
		release(b);
		if (!(b.p = malloc(bytes))) { ssq_set_error("host restatement: out of memory"); return SSQ_ENOMEM; }
		b.cap = bytes; cur += bytes;
		if (cur > peak) peak = cur;
		return 0;
	}
	void release(SpBuf &b) { if (b.p) { free(b.p); cur -= b.cap; } b.p = 0; b.cap = 0; }
	int put(void *d, const void *h, u64 bytes) { memcpy(d, h, bytes); return 0; }
	int get(void *h, const void *d, u64 bytes) { memcpy(h, d, bytes); return 0; }
	int zero(void *d, u64 bytes) { memset(d, 0, bytes); return 0; }
	template <class F> int each(u64 n, const F &f) { for (u64 j = 0; j < n; ++j) f(j); return 0; }
	int sort(u64 *&k, u64 *&v, u64 *&, u64 *&, u64 m, int bits)
	{
		const u64 mask = bits >= 64 ? ~0ull : (1ull << bits) - 1;
		std::vector<std::pair<u64, u64> > a(m);
		for (u64 j = 0; j < m; ++j) a[j] = std::make_pair(k[j] & mask, v[j]);
		std::stable_sort(a.begin(), a.end(), [](const std::pair<u64, u64> &x, const std::pair<u64, u64> &y) { return x.first < y.first; });
		for (u64 j = 0; j < m; ++j) { k[j] = a[j].first; v[j] = a[j].second; }
		return 0;
	}
	int max_scan(u64 *a, u64 m) { for (u64 j = 1; j < m; ++j) if (a[j] < a[j - 1]) a[j] = a[j - 1]; return 0; }
	int excl_sum(u64 *a, u64 m) { u64 s = 0; for (u64 j = 0; j < m; ++j) { const u64 x = a[j]; a[j] = s; s += x; } return 0; }
};

// PREFIX.bwt / PREFIX.sa from the 2-bit forward text pac (l_pac bases) with a working budget of work bytes (chunk_work: the
// rounds' chunks, 0 = work); stats as
// ssq_index_build_stats_t.  Returns 0, an SSQ_E* code (message: hostsim_error), or 99 when the i + h <= n invariant broke.
extern "C" int hostsim_sapass(const uint8_t *pac, size_t pac_bytes, int64_t l_pac, const char *prefix, uint64_t work, uint64_t chunk_work, ssq_index_build_stats_t *st)
{
	std::vector<uint8_t> p(pac, pac + pac_bytes);
	p.resize((size_t)(l_pac >> 2) + 2, 0);
	SpHost be;
	g_violation = 0;
	g_err[0] = 0;
	st->path = 2;
	const int rc = sp_build(be, p.data(), p.size(), l_pac, prefix, work, st, chunk_work);
	return rc ? rc : g_violation ? 99 : 0;
}
extern "C" const char *hostsim_error(void) { return g_err; }
