// gunzip_host.cpp — TEST-ONLY: the chunk-parallel gzip decoder of speedseq_b200/csrc/ssq_gunzip.cu run on the host.  The window
// logic of ssq_gunzip.cuh (gz_window, gz_run) drives the same SSQ_HD phases the kernels run, each as a host loop: the sync search
// as a loop over 32 lanes per round, one chunk decode after the other, the in-order tail pass and then the rest of the resolve,
// the CRC pieces.  Output and stats = what ssq_gunzip_inflate_dev returns for the same input and chunk size.
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../speedseq_b200/csrc/ssq_gunzip.cuh"

struct HostBackend : GzBackend {
	std::vector<uint16_t> slots;
	std::vector<uint8_t> wout;
	std::vector<u32> crc_tab;
	GzTab T;
	HostBackend() : wout(GZ_CTX), crc_tab(256) { for (u32 i = 0; i < 256; ++i) crc_tab[i] = bz_crc_entry(i); }
	int sync(const GzIn &I, int n, bz_u64 lo, bz_u64 cbits, bz_u64 wend, bz_u64 *s) override
	{
		for (int i = 1; i < n; ++i) {
			const bz_u64 a = lo + (bz_u64)i * cbits, b = a + cbits < wend ? a + cbits : wend;
			s[i] = GZ_NONE;
			for (u32 r = 0; s[i] == GZ_NONE && a + (bz_u64)r * 32 < b; ++r)
				for (int lane = 0; lane < 32; ++lane) { bz_u64 c; if (gz_sync_lane(I, T, a, b, r, lane, &c)) { s[i] = c; break; } }
		}
		return 0;
	}
	int decode(const GzIn &I, const std::vector<int> &which, GzChunk *ch, GzEvent *ev) override
	{
		if (slots.size() < (size_t)(which.empty() ? 0 : which.back() + 1) * GZ_SLOT) slots.resize((size_t)(which.back() + 1) * GZ_SLOT);
		for (int k : which) gz_decode(I, T, ch[k], slots.data() + (size_t)k * GZ_SLOT, ev + (size_t)k * GZ_EVCAP);
		return 0;
	}
	int resolve(int n, const u32 *len, const bz_u64 *off) override
	{
		bz_u64 tot = 0;
		for (int k = 0; k < n; ++k) tot += len[k];
		if (wout.size() < GZ_CTX + tot) wout.resize(GZ_CTX + tot);
		for (int k = 0; k < n; ++k) gz_resolve_range(slots.data() + (size_t)k * GZ_SLOT, off[k], len[k] > GZ_CTX ? len[k] - GZ_CTX : 0, len[k], wout.data(), 0, 1);
		for (int k = 0; k < n; ++k) gz_resolve_range(slots.data() + (size_t)k * GZ_SLOT, off[k], 0, len[k] > GZ_CTX ? len[k] - GZ_CTX : 0, wout.data(), 0, 1);
		return 0;
	}
	int crc(const std::vector<bz_u64> &off, const std::vector<u32> &len, std::vector<u32> &out) override
	{
		out.resize(off.size());
		for (size_t i = 0; i < off.size(); ++i) out[i] = gz_crc_piece(crc_tab.data(), wout.data() + GZ_CTX + off[i], len[i]);
		return 0;
	}
};

// the whole stream in[0, n) (final) with chunks of chunk_bytes: 0, or SSQ_EDATA with *err_at; stats as ssq_gunzip_stats
extern "C" int hostsim_gunzip(const void *in, size_t n, size_t chunk_bytes, void **out, size_t *out_len, int64_t *stats, size_t *err_at)
{
	HostBackend *be = new HostBackend;
	GzState S; gz_state_init(S);
	std::vector<uint8_t> o;
	auto emit = [&](bz_u64 text) {
		o.insert(o.end(), be->wout.begin() + GZ_CTX, be->wout.begin() + GZ_CTX + text);
		std::vector<uint8_t> ctx(be->wout.begin() + text, be->wout.begin() + text + GZ_CTX); // the last 32 KB of [context][text]
		memcpy(be->wout.data(), ctx.data(), GZ_CTX);
		return 0;
	};
	bz_u64 at = 0;
	const int rc = gz_run(*be, S, (const uint8_t*)in, n, chunk_bytes ? chunk_bytes : GZ_CHUNK_DEFAULT, emit, &at);
	delete be;
	memcpy(stats, S.stats, sizeof S.stats);
	*err_at = (size_t)at;
	*out_len = o.size();
	*out = malloc(o.size() + 1);
	memcpy(*out, o.data(), o.size());
	return rc;
}
extern "C" void hostsim_free(void *p) { free(p); }
