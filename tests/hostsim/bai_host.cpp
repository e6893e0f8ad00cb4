// bai_host.cpp — TEST-ONLY: the BAI builder of speedseq_b200/csrc/ssq_bai.cu run on the host.  The host logic of ssq_bai.cuh and
// ssq_gunzip.cuh (gz_bgzf_chain, gz_bgzf_members, bai_from_text) drives the same SSQ_HD phases the kernels run, each as a host
// loop: the member decodes one after the other, the CRC pieces, the walkers, the record writes and checks; the device's radix sort
// and scans are a stable sort and running sums here.  Output = what ssq_bai_build returns for the same input and segment size.
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "../../include/ssq.h"
static char g_err[512];
static void ssq_set_error(const char *fmt, ...) { va_list ap; va_start(ap, fmt); vsnprintf(g_err, sizeof g_err, fmt, ap); va_end(ap); }
#include "../../speedseq_b200/csrc/ssq_bai.cuh"

struct HostBgzf : GzBgzfBackend {
	const uint8_t *in; std::vector<uint8_t> *out;
	std::vector<uint16_t> slots; std::vector<u32> crc_tab; GzTab T;
	HostBgzf() : crc_tab(256) { for (u32 i = 0; i < 256; ++i) crc_tab[i] = bz_crc_entry(i); }
	int decode(const GzMember *m, int k, GzChunk *ch, GzEvent *ev) override
	{
		slots.resize((size_t)k * GZ_SLOT);
		for (int i = 0; i < k; ++i) { GzIn I; I.p = in + m[i].coff; I.n = m[i].csize; I.final = 1; gz_decode(I, T, ch[i], slots.data() + (size_t)i * GZ_SLOT, ev + (size_t)i * GZ_EVCAP); }
		return 0;
	}
	int emit(const GzMember *m, int k) override
	{
		for (int i = 0; i < k; ++i) gz_bgzf_emit(slots.data() + (size_t)i * GZ_SLOT, m[i].isize, out->data() + m[i].toff, 0, 1);
		return 0;
	}
	int crc(const std::vector<bz_u64> &off, const std::vector<u32> &len, std::vector<u32> &o) override
	{
		o.resize(off.size());
		for (size_t i = 0; i < off.size(); ++i) o[i] = gz_crc_piece(crc_tab.data(), out->data() + off[i], len[i]);
		return 0;
	}
};

struct HostBai : BaiBackend {
	const uint8_t *t; bz_u64 n, clen;
	const std::vector<GzMember> *m;
	std::vector<BaiRec> rec;
	int walk(std::vector<BaiSeg> &seg, const std::vector<int> &which, int nr) override { for (int i : which) bai_guess_walk(t, n, nr, seg[i]); return 0; }
	int records(const std::vector<BaiSeg> &seg, const std::vector<bz_u64> &base, bz_u64 n_rec) override
	{
		rec.resize(n_rec);
		for (size_t i = 0; i < seg.size(); ++i) bai_walk_write(t, n, seg[i], m->data(), m->size(), clen, rec.data() + base[i]);
		return 0;
	}
	int check(bz_u64 n_rec, int nr, bz_u64 *first_bad, bz_u64 *n_pos) override
	{
		*first_bad = BAI_NONE; *n_pos = 0;
		for (bz_u64 i = 0; i < n_rec; ++i) {
			const int e = bai_check(rec.data(), i, nr);
			if (e && *first_bad == BAI_NONE) *first_bad = i << 3 | (bz_u64)e;
			if (rec[i].ref >= 0) *n_pos = i + 1;
		}
		return 0;
	}
	int rec_at(bz_u64 i, BaiRec *r) override { *r = rec[i]; return 0; }
	int index(bz_u64 n_rec, bz_u64 P, int nr, BaiOut &o) override
	{
		const BaiRec *r = rec.data();
		// runs in file order, then stably by (reference, bin)
		std::vector<bz_u64> first;
		for (bz_u64 i = 0; i < P; ++i) if (bai_run_start(r, i)) first.push_back(i);
		const size_t nrun = first.size();
		std::vector<bz_u64> key(nrun), vb(nrun), ve(nrun);
		for (size_t j = 0; j < nrun; ++j) { key[j] = bai_run_key(r[first[j]]); vb[j] = r[first[j]].vbeg; ve[j] = r[(j + 1 < nrun ? first[j + 1] : P) - 1].vend; }
		std::vector<u32> ord(nrun);
		for (size_t j = 0; j < nrun; ++j) ord[j] = (u32)j;
		std::stable_sort(ord.begin(), ord.end(), [&](u32 a, u32 b) { return key[a] < key[b]; });
		for (size_t j = 0; j < nrun; ++j) {
			const u32 x = ord[j];
			const bool nb = !j || key[ord[j - 1]] != key[x];
			if (!j || bai_new_chunk(key[ord[j - 1]], ve[ord[j - 1]], key[x], vb[x])) o.chunks.push_back({vb[x], ve[x]});
			else o.chunks.back().end = ve[x];
			if (nb) { if (!o.bins.empty()) o.bins.back().hi = (u32)o.chunks.size() - 1; o.bins.push_back({(int32_t)(key[x] >> 16), (u32)(key[x] & 0xffff), x, (u32)o.chunks.size() - 1, 0}); }
		}
		if (!o.bins.empty()) o.bins.back().hi = (u32)o.chunks.size();
		// linear index and metadata
		o.has.assign(nr, 0); o.meta.assign(4 * (size_t)nr, 0); o.lin_base.assign(nr + 1, 0);
		std::vector<bz_u64> nint(nr, 0);
		for (bz_u64 i = 0; i < P; ++i) { long long w0, w1; bai_windows(r[i], &w0, &w1); if (w1 > (long long)nint[r[i].ref]) nint[r[i].ref] = (bz_u64)w1; }
		for (int k = 0; k < nr; ++k) o.lin_base[k + 1] = o.lin_base[k] + nint[k];
		o.lin.assign(o.lin_base[nr], BAI_NONE);
		for (bz_u64 i = 0; i < P; ++i) {
			long long w0, w1; bai_windows(r[i], &w0, &w1);
			for (long long w = w0; w < w1; ++w) { bz_u64 &x = o.lin[o.lin_base[r[i].ref] + w]; if (r[i].vbeg < x) x = r[i].vbeg; }
			const int k = r[i].ref;
			if (!i || r[i - 1].ref != k) { o.has[k] = 1; o.meta[4 * k] = r[i].vbeg; }
			if (i + 1 == P) o.meta[4 * k + 1] = r[n_rec - 1].vend; else if (r[i + 1].ref != k) o.meta[4 * k + 1] = r[i].vend;
			++o.meta[4 * k + ((r[i].flag & 4) ? 3 : 2)];
		}
		for (int k = 0; k < nr; ++k) { bz_u64 prev = 0; for (bz_u64 w = o.lin_base[k]; w < o.lin_base[k + 1]; ++w) { if (o.lin[w] == BAI_NONE) o.lin[w] = prev; prev = o.lin[w]; } }
		return 0;
	}
};

// the index of the BGZF file in[0, n) with walker segments of seg bytes (0: default): 0, or an SSQ_E* code with the message in err
extern "C" int hostsim_bai(const void *in, size_t n, size_t seg, void **out, size_t *out_len, char *err, size_t err_cap)
{
	*out = 0; *out_len = 0; g_err[0] = 0;
	const uint8_t *p = (const uint8_t*)in;
	std::vector<GzMember> m(n / 20 + 1);
	bz_u64 nm = 0, at = 0;
	int rc = gz_bgzf_chain(p, n, m.data(), m.size(), &nm, &at);
	m.resize(nm);
	std::vector<uint8_t> text;
	std::string bai;
	if (rc) { ssq_set_error("not BGZF: %s at compressed byte %llu", gz_bgzf_why(rc), (unsigned long long)at); rc = SSQ_EDATA; }
	else if (!nm) { ssq_set_error("not a BAM file: no BGZF member"); rc = SSQ_EFORMAT; }
	if (!rc) {
		text.resize(m.back().toff + m.back().isize);
		HostBgzf hz; hz.in = p; hz.out = &text;
		if ((rc = gz_bgzf_members(hz, m, &at))) ssq_set_error("corrupt BGZF member at compressed byte %llu", (unsigned long long)at);
	}
	if (!rc) {
		HostBai hb; hb.t = text.data(); hb.n = text.size(); hb.clen = n; hb.m = &m;
		auto fetch = [&](bz_u64 k, uint8_t *b) { memcpy(b, text.data(), k); return 0; };
		rc = bai_from_text(hb, fetch, text.size(), m, seg ? seg : BAI_SEG_DEFAULT, bai);
	}
	snprintf(err, err_cap, "%s", g_err);
	if (rc) return rc;
	*out = malloc(bai.size());
	memcpy(*out, bai.data(), bai.size());
	*out_len = bai.size();
	return 0;
}
extern "C" void hostsim_bai_free(void *p) { free(p); }
