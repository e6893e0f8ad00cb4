// merge_host.cpp — TEST-ONLY: the BAM merge of speedseq_b200/csrc/ssq_merge.cu run on the host.  The host logic of ssq_merge.cuh
// (windows, header, walk links, sambamba's heap: mg_run) drives the same SSQ_HD phases the kernels run, each as a host loop: the
// members of a window decode one after the other (bai_host.cpp's HostBgzf: the phases of ssq_gunzip.cuh), the walkers, the
// record offsets, the keys and checks, the gather.  Output = the uncompressed file ssq_merge_run hands its sink without z.
#include "bai_host.cpp"
#include "../../speedseq_b200/csrc/ssq_merge.cuh"

extern "C" const char *ssq_last_error(void) { return g_err; }

struct HostMerge : MergeBackend {
	struct In { std::vector<uint8_t> text[2]; int cur = 0; std::vector<bz_u64> roff; };
	std::vector<In> in;
	std::string *out;
	const uint8_t *text(int k) { return in[k].text[in[k].cur].data(); }
	int fill(int k, bz_u64 from, bz_u64 keep, const uint8_t *c, bz_u64 clen, const std::vector<GzMember> &m, bz_u64 *err_at) override
	{
		In &I = in[k];
		std::vector<uint8_t> &dst = I.text[1 - I.cur], w(m.back().toff + m.back().isize);
		HostBgzf hz; hz.in = c; hz.out = &w;
		if (gz_bgzf_members(hz, m, err_at)) return SSQ_EDATA;
		dst.resize(keep + w.size());
		if (keep) memcpy(dst.data(), I.text[I.cur].data() + from, keep);
		if (!w.empty()) memcpy(dst.data() + keep, w.data(), w.size());
		I.cur = 1 - I.cur;
		return 0;
	}
	int peek(int k, bz_u64 at, void *buf, u32 len) override { memcpy(buf, text(k) + at, len); return 0; }
	int walk(int k, std::vector<BaiSeg> &seg, const std::vector<int> &which, int n_ref) override
	{
		for (int i : which) bai_guess_walk(text(k), seg.back().lim, n_ref, seg[i]);
		return 0;
	}
	int records(int k, const std::vector<BaiSeg> &seg, const std::vector<bz_u64> &base, bz_u64 n_rec, int n_ref, std::vector<bz_u64> &keys, bz_u64 *bad) override
	{
		std::vector<bz_u64> &r = in[k].roff;
		r.resize(n_rec); keys.resize(n_rec);
		for (size_t i = 0; i < seg.size(); ++i) mg_walk_write(text(k), seg.back().lim, seg[i], r.data() + base[i]);
		*bad = BAI_NONE;
		for (bz_u64 i = 0; i < n_rec; ++i) { const int e = mg_check(text(k), r.data(), i, n_ref, &keys[i]); if (e && *bad == BAI_NONE) *bad = i << 3 | (bz_u64)e; }
		return 0;
	}
	int gather(const std::vector<bz_u64> &order, bz_u64) override
	{
		for (bz_u64 o : order) {
			const int k = (int)(o >> MG_IDX_BITS);
			const uint8_t *p = text(k) + in[k].roff[o & MG_IDX_MASK];
			out->append((const char*)p, 4 + bai_u32(p, 0));
		}
		return 0;
	}
};

// the merge of paths[0, n) with windows of `window` compressed bytes and walker segments of seg bytes (0: the defaults):
// 0 (*out: the uncompressed merged file, free with hostsim_merge_free), or an SSQ_E* code with the message in err
extern "C" int hostsim_merge(const char *const *paths, int n, size_t window, size_t seg, void **out, size_t *out_len, char *err, size_t err_cap)
{
	*out = 0; *out_len = 0; g_err[0] = 0;
	std::vector<MgInput> in;
	std::string text, body;
	int rc = mg_open(paths, n, in, text);
	if (!rc) {
		body = mg_bam_header(text, in[0]);
		HostMerge be; be.in.resize(n); be.out = &body;
		double ms[3] = {0, 0, 0};
		bz_u64 n_rec = 0;
		rc = mg_run(be, in, window ? window : MG_WINDOW_DEFAULT, seg ? seg : BAI_SEG_DEFAULT, &n_rec, ms);
	}
	snprintf(err, err_cap, "%s", g_err);
	if (rc) return rc;
	*out = malloc(body.size());
	memcpy(*out, body.data(), body.size());
	*out_len = body.size();
	return 0;
}
extern "C" void hostsim_merge_free(void *p) { free(p); }
