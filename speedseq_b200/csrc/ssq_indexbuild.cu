// ssq_indexbuild.cu — `bwa index` on the GPU: FASTA -> PREFIX.{amb,ann,pac,bwt,sa}.
//
// Reference call site: `$BWA index $REF` at speedseq/bin/speedseq:389 (and :1925); the five files must be
// byte-identical to what upstream bwa writes — pinned by the reference's goldens
// speedseq/example/data/human_g1k_v37_20_42220611-42542245.fasta.{amb,ann,pac,bwt,sa} (tests/test_gpu_index.py).
// Upstream routines replaced (not vendored in the reference tree): bns_fasta2bntseq, bwt_pac2bwt/bwt_bwtgen,
// bwt_bwtupdate_core, bwt_cal_sa.
//
// Design: the text T = forward + reverse-complement strand never leaves its 2-bit packing; the suffix array of T$ is built
// by the multi-pass device sort of ssq_sapass.cuh (5 B of HBM per suffix for the rank array + a working budget sized from the
// device's free memory, fewer than 2^40 suffixes: whole GRCh37 has 6.2 G), and BWT symbols, the occ checkpoints every 128
// symbols and the SA samples every 32 rows are written in the reference's layout.  Without a device or the memory for it, the
// suffix array is built on the host — induced sorting with 64-bit indices (ssq_sais.h), BWT / occ checkpoints / SA samples by
// host threads — and
// written in the same layout; no GPU is touched on that path (SSQ_INDEX_HOST=1 forces it for any size: the CPU tests pin it on
// the reference's goldens).  FASTA parsing and the lrand48() replacement of ambiguous bases are inherently sequential (the
// random stream is consumed in file order) and run on the host.
#include <cuda_runtime.h>
#include <cub/cub.cuh>
#include <zlib.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <ctype.h>
#include <string>
#include <vector>
#include <thread>
#include "ssq_host.h"
#include "ssq_sais.h"
#include "ssq_sapass.cuh"

// ---------------------------------------------------------------------------- host: FASTA ----
struct FaContig { std::string name, anno; i64 offset; i32 len, n_ambs; };
struct FaHole { i64 offset; i32 len; char amb; };

static inline int nt4(int c)
{
	switch (c) { case 'A': case 'a': return 0; case 'C': case 'c': return 1; case 'G': case 'g': return 2; case 'T': case 't': return 3; }
	return 4;
}

// streams the FASTA once: header line = name up to the first blank + optional comment; every non-blank residue
// character is one base; ambiguity codes become lrand48()&3 (seed 11) and are logged as holes, runs of the same
// letter merged
static int parse_fasta(const char *fn, std::vector<FaContig> &ctg, std::vector<FaHole> &holes, std::vector<uint8_t> &pac, i64 &l_pac)
{
	gzFile fp = strcmp(fn, "-") ? gzopen(fn, "r") : gzdopen(0, "r");
	if (!fp) return SSQ_EIO;
	std::vector<char> buf(1 << 20);
	bool in_header = false, at_line_start = true, name_done = false;
	int last = 0, n;
	FaContig *cur = 0;
	l_pac = 0;
	srand48(11);
	while ((n = gzread(fp, buf.data(), (unsigned)buf.size())) > 0) {
		for (int i = 0; i < n; ++i) {
			const int c = (unsigned char)buf[i];
			if (in_header) {
				if (c == '\n') { in_header = false; at_line_start = true; if (!cur->anno.empty() && cur->anno.back() == '\r') cur->anno.pop_back(); if (cur->anno.empty() && !cur->name.empty() && cur->name.back() == '\r') cur->name.pop_back(); }
				else if (!name_done) { if (isspace(c)) name_done = true; else cur->name.push_back((char)c); }
				else cur->anno.push_back((char)c);
				continue;
			}
			if (c == '\n') { at_line_start = true; continue; }
			if (at_line_start && c == '>') {
				ctg.push_back(FaContig());
				cur = &ctg.back();
				cur->offset = l_pac; cur->len = 0; cur->n_ambs = 0;
				in_header = true; name_done = false; last = 0;
				continue;
			}
			at_line_start = false;
			if (!cur || isspace(c)) continue;
			int b = nt4(c);
			if (b >= 4) {
				if (last == c) ++holes.back().len;
				else { FaHole h; h.offset = l_pac; h.len = 1; h.amb = (char)c; holes.push_back(h); ++cur->n_ambs; }
				b = (int)(lrand48() & 3);
			}
			last = c;
			if ((size_t)(l_pac >> 2) >= pac.size()) pac.resize(pac.size() ? pac.size() * 2 : (1 << 20), 0);
			pac[l_pac >> 2] |= (uint8_t)(b << ((~l_pac & 3) << 1));
			++l_pac; ++cur->len;
		}
	}
	gzclose(fp);
	return ctg.empty() || l_pac == 0 ? SSQ_EIO : SSQ_OK;
}

static int write_text_files(const char *prefix, const std::vector<FaContig> &ctg, const std::vector<FaHole> &holes, const std::vector<uint8_t> &pac, i64 l_pac)
{
	std::string p(prefix);
	FILE *fp = fopen((p + ".ann").c_str(), "w");
	if (!fp) return SSQ_EIO;
	fprintf(fp, "%lld %d %u\n", (long long)l_pac, (int)ctg.size(), 11u);
	for (size_t i = 0; i < ctg.size(); ++i) {
		fprintf(fp, "0 %s %s\n", ctg[i].name.c_str(), ctg[i].anno.empty() ? "(null)" : ctg[i].anno.c_str());
		fprintf(fp, "%lld %d %d\n", (long long)ctg[i].offset, ctg[i].len, ctg[i].n_ambs);
	}
	fclose(fp);
	if (!(fp = fopen((p + ".amb").c_str(), "w"))) return SSQ_EIO;
	fprintf(fp, "%lld %d %u\n", (long long)l_pac, (int)ctg.size(), (unsigned)holes.size());
	for (size_t i = 0; i < holes.size(); ++i) fprintf(fp, "%lld %d %c\n", (long long)holes[i].offset, holes[i].len, holes[i].amb);
	fclose(fp);
	if (!(fp = fopen((p + ".pac").c_str(), "wb"))) return SSQ_EIO;
	fwrite(pac.data(), 1, (size_t)((l_pac >> 2) + ((l_pac & 3) ? 1 : 0)), fp);
	uint8_t ct = 0;
	if (l_pac % 4 == 0) fwrite(&ct, 1, 1, fp);
	ct = (uint8_t)(l_pac % 4);
	fwrite(&ct, 1, 1, fp);
	fclose(fp);
	return SSQ_OK;
}

// ------------------------------------------------------------------------------ kernels ----
// one thread per element of [0, n) (grid-stride past 2^30 threads); f is one of the SSQ_HD bodies of ssq_sapass.cuh
template <class F> __global__ void k_sp_each(u64 n, F f)
{
	for (u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x; j < n; j += (u64)gridDim.x * blockDim.x) f(j);
}
template <class F> static cudaError_t sp_launch(u64 n, const F &f)
{
	if (!n) return cudaSuccess;
	const u64 g = (n + 255) / 256;
	k_sp_each<<<(unsigned)(g < (1u << 22) ? g : (1u << 22)), 256>>>(n, f);
	return cudaGetLastError();
}

// ------------------------------------------------------------------------- host path ----
// PREFIX.bwt / PREFIX.sa from the 2-bit forward strand with everything on the host; bits: width of a suffix-array entry (32, 40, 64)
template <class SAP>
static int build_bwt_sa_host_impl(const char *prefix, const std::vector<uint8_t> &pac, i64 l_pac, std::vector<uint8_t> &s, SAP SA);
static int build_bwt_sa_host(const char *prefix, const std::vector<uint8_t> &pac, i64 l_pac, int bits)
{
	const u64 n1 = 2 * (u64)l_pac + 1;
	std::vector<uint8_t> s, raw;
	try { s.resize(n1); raw.resize(n1 * (size_t)(bits / 8) + 8); }
	catch (...) { ssq_set_error("not enough host memory for the suffix array of %llu symbols (%llu GB)", (unsigned long long)(n1 - 1), (unsigned long long)((n1 * (size_t)(bits / 8 + 1)) >> 30)); return SSQ_ENOMEM; }
	if (bits == 32) return build_bwt_sa_host_impl(prefix, pac, l_pac, s, (int32_t*)raw.data());
	if (bits == 64) return build_bwt_sa_host_impl(prefix, pac, l_pac, s, (int64_t*)raw.data());
	ssq_p40 v; v.p = raw.data();
	return build_bwt_sa_host_impl(prefix, pac, l_pac, s, v);
}
template <class SAP>
static int build_bwt_sa_host_impl(const char *prefix, const std::vector<uint8_t> &pac, i64 l_pac, std::vector<uint8_t> &s, SAP SA)
{
	const u64 n = 2 * (u64)l_pac, n1 = n + 1;
	std::vector<u32> out, cnt;
	int n_thr = (int)std::thread::hardware_concurrency();
	if (n_thr < 1) n_thr = 1;
	if (n_thr > 64) n_thr = 64;
	auto par = [&](u64 total, auto fn) { // fn(lo, hi) over [0, total) in n_thr contiguous pieces
		std::vector<std::thread> th;
		const u64 per = (total + n_thr - 1) / n_thr;
		for (int t = 0; t < n_thr; ++t) { const u64 lo = per * t, hi = lo + per < total ? lo + per : total; if (lo < hi) th.emplace_back(fn, lo, hi); }
		for (auto &x : th) x.join();
	};
	// T$ over {0: '$', 1..4: A C G T}: forward strand then its reverse complement (sp_sym on the device paths)
	par(n, [&](u64 lo, u64 hi) {
		for (u64 i = lo; i < hi; ++i) {
			const bool fw = i < (u64)l_pac;
			const u64 p = fw ? i : n - 1 - i;
			const int b = pac[p >> 2] >> ((~p & 3) << 1) & 3;
			s[i] = (uint8_t)(1 + (fw ? b : 3 - b));
		}
	});
	s[n] = 0;
	ssq_sais(s.data(), SA, (int64_t)n1, (int64_t)5);
	u64 primary = 0;
	{
		std::vector<u64> found(n_thr + 1, ~0ull);
		std::vector<std::thread> th;
		const u64 per = (n1 + n_thr - 1) / n_thr;
		for (int t = 0; t < n_thr; ++t) th.emplace_back([&, t]() { const u64 lo = per * t, hi = lo + per < n1 ? lo + per : n1; for (u64 r = lo; r < hi; ++r) if ((i64)SA[(i64)r] == 0) found[t] = r; });
		for (auto &x : th) x.join();
		for (int t = 0; t < n_thr; ++t) if (found[t] != ~0ull) primary = found[t];
	}
	// interleaved occ/BWT: block b at words [16b, 16b+16) = u64 occ[4] then 8 words of 16 symbols (MSB first); totals after the last word
	const u64 n_blk = (n + 127) / 128, raw_words = (n + 15) / 16, total_words = raw_words + (n_blk + 1) * 8;
	try { out.assign(total_words, 0); cnt.assign((n_blk + 1) * 4, 0); } catch (...) { ssq_set_error("not enough host memory for the BWT"); return SSQ_ENOMEM; }
	par(n_blk, [&](u64 lo, u64 hi) {
		for (u64 b = lo; b < hi; ++b) {
			u32 c[4] = {0, 0, 0, 0};
			for (u32 w = 0; w < 8; ++w) {
				const u64 j0 = b * 128 + (u64)w * 16;
				if (j0 >= n) break;
				u32 v = 0;
				for (u32 k = 0; k < 16; ++k) {
					const u64 j = j0 + k;
					u32 sym = 0;
					if (j < n) { const u64 r = j + (j >= primary); sym = (u32)s[(u64)(i64)SA[(i64)r] - 1] - 1; ++c[sym]; }
					v = v << 2 | sym;
				}
				out[b * 16 + 8 + w] = v;
			}
			for (int k = 0; k < 4; ++k) cnt[b * 4 + k] = c[k];
		}
	});
	u64 run[4] = {0, 0, 0, 0};
	for (u64 b = 0; b <= n_blk; ++b) { // checkpoints: counts before the block; the last one (totals) sits 8 words before the end
		u32 *o = b < n_blk ? &out[b * 16] : &out[total_words - 8];
		for (int k = 0; k < 4; ++k) { o[2 * k] = (u32)run[k]; o[2 * k + 1] = (u32)(run[k] >> 32); if (b < n_blk) run[k] += cnt[b * 4 + k]; }
	}
	u64 L2[5] = {0, run[0], run[0] + run[1], run[0] + run[1] + run[2], run[0] + run[1] + run[2] + run[3]};
	std::string p(prefix);
	FILE *fp = fopen((p + ".bwt").c_str(), "wb");
	if (!fp) { ssq_set_error("cannot write %s.bwt", prefix); return SSQ_EIO; }
	fwrite(&primary, 8, 1, fp); fwrite(L2 + 1, 8, 4, fp); fwrite(out.data(), 4, out.size(), fp);
	if (fclose(fp)) { ssq_set_error("cannot write %s.bwt", prefix); return SSQ_EIO; }
	std::vector<u32>().swap(out); std::vector<u32>().swap(cnt);
	const u64 n_sa = (n + 32) / 32, sa_intv = 32, seq_len = n;
	std::vector<u64> smp(n_sa ? n_sa - 1 : 0);
	for (u64 k = 1; k < n_sa; ++k) smp[k - 1] = (u64)(i64)SA[(i64)(k * 32)];
	if (!(fp = fopen((p + ".sa").c_str(), "wb"))) { ssq_set_error("cannot write %s.sa", prefix); return SSQ_EIO; }
	fwrite(&primary, 8, 1, fp); fwrite(L2 + 1, 8, 4, fp); fwrite(&sa_intv, 8, 1, fp); fwrite(&seq_len, 8, 1, fp); fwrite(smp.data(), 8, smp.size(), fp);
	if (fclose(fp)) { ssq_set_error("cannot write %s.sa", prefix); return SSQ_EIO; }
	return SSQ_OK;
}

// -------------------------------------------------------------------- multi-pass device path ----
// the backend sp_build (ssq_sapass.cuh) runs on: kernels over the SSQ_HD bodies, CUB for sorts and scans
struct SpDevice {
	u64 cur = 0, peak = 0;
	SpBuf tmp = {0, 0};
	~SpDevice() { release(tmp); }
	int ck(cudaError_t e) { if (e == cudaSuccess) return 0; ssq_set_error("multi-pass index build: %s", cudaGetErrorString(e)); return SSQ_ECUDA; }
	int need(SpBuf &b, u64 bytes)
	{
		if (bytes <= b.cap) return 0;
		release(b);
		if (cudaMalloc(&b.p, bytes) != cudaSuccess) {
			cudaGetLastError();
			size_t fr = 0, tot = 0;
			cudaMemGetInfo(&fr, &tot);
			b.p = 0;
			ssq_set_error("multi-pass index build: cannot allocate %.3f GB of device memory (this build holds %.3f GB, %.3f GB free)", bytes / 1e9, cur / 1e9, fr / 1e9);
			return SSQ_ENOMEM;
		}
		b.cap = bytes; cur += bytes;
		if (cur > peak) peak = cur;
		return 0;
	}
	void release(SpBuf &b) { if (b.p) { cudaFree(b.p); cur -= b.cap; } b.p = 0; b.cap = 0; }
	int put(void *d, const void *h, u64 bytes) { return ck(cudaMemcpy(d, h, bytes, cudaMemcpyHostToDevice)); }
	int get(void *h, const void *d, u64 bytes) { return ck(cudaMemcpy(h, d, bytes, cudaMemcpyDeviceToHost)); }
	int zero(void *d, u64 bytes) { return ck(cudaMemset(d, 0, bytes)); }
	template <class F> int each(u64 n, const F &f) { return ck(sp_launch(n, f)); }
	int sort(u64 *&k, u64 *&v, u64 *&k2, u64 *&v2, u64 m, int bits)
	{
		cub::DoubleBuffer<u64> kb(k, k2), vb(v, v2);
		size_t tb = 0;
		int rc;
		if ((rc = ck(cub::DeviceRadixSort::SortPairs(0, tb, kb, vb, (int)m, 0, bits)))) return rc;
		if ((rc = need(tmp, tb + 1))) return rc;
		if ((rc = ck(cub::DeviceRadixSort::SortPairs(tmp.p, tb, kb, vb, (int)m, 0, bits)))) return rc;
		k = kb.Current(); k2 = kb.Alternate(); v = vb.Current(); v2 = vb.Alternate();
		return 0;
	}
	int max_scan(u64 *a, u64 m)
	{
		size_t tb = 0;
		int rc;
		if ((rc = ck(cub::DeviceScan::InclusiveScan(0, tb, a, a, cub::Max(), (int)m)))) return rc;
		if ((rc = need(tmp, tb + 1))) return rc;
		return ck(cub::DeviceScan::InclusiveScan(tmp.p, tb, a, a, cub::Max(), (int)m));
	}
	int excl_sum(u64 *a, u64 m)
	{
		size_t tb = 0;
		int rc;
		if ((rc = ck(cub::DeviceScan::ExclusiveSum(0, tb, a, a, (int)m)))) return rc;
		if ((rc = need(tmp, tb + 1))) return rc;
		return ck(cub::DeviceScan::ExclusiveSum(tmp.p, tb, a, a, (int)m));
	}
};

// -------------------------------------------------------------------------------- driver ----
#define SP_MARGIN(fr) ((u64)(1ull << 30) + (u64)(fr) / 32) // device memory left to other users of the card
// the least working budget the automatic choice takes the device with: 256 MB, and at least enough for 32 first-sort passes
static u64 sp_min_work(u64 n1) { const u64 w = n1 * SP_PASS_ROW_BYTES / 32; return w > (256ull << 20) ? w : (256ull << 20); }

extern "C" int ssq_index_build_ex(const char *fasta, const char *prefix, int device, const ssq_index_build_opts_t *opt, ssq_index_build_stats_t *st)
{
	if (!fasta) return SSQ_EINVAL;
	if (!prefix) prefix = fasta;
	ssq_index_build_stats_t st0;
	if (!st) st = &st0;
	memset(st, 0, sizeof *st);
	const int want = opt ? opt->path : 0;
	if (want != 0 && want != 2 && want != 3) { ssq_set_error("index build path %d: 0 auto, 2 device (multi-pass) sort, 3 host", want); return SSQ_EINVAL; }
	int rc;
	std::vector<FaContig> ctg; std::vector<FaHole> holes; std::vector<uint8_t> pac;
	i64 l_pac = 0;
	if ((rc = parse_fasta(fasta, ctg, holes, pac, l_pac))) { ssq_set_error("cannot read any sequence from %s", fasta); return rc; }
	pac.resize((size_t)(l_pac >> 2) + 2, 0);
	const u64 n1 = 2 * (u64)l_pac + 1;
	const bool small = n1 < 0x7fffffffull; // 32-bit suffix-array entries suffice on the host path
	const u64 fixed = 5 * n1 + pac.size() + SP_NBUCKET * 8 + 64; // rank planes, text, bucket counts
	const char *force = getenv("SSQ_INDEX_HOST"); // 1: host path with the narrowest entry type that fits, 40 / 64: with 40- / 64-bit entries
	int path = want;
	u64 work = opt ? opt->work_bytes : 0;
	char why[256] = "";
	if (want == 0 && force && atoi(force)) path = 3;
	if (path == 2 && n1 >= SP_MAX_N1) { ssq_set_error("%llu suffixes: the device sort holds fewer than 2^40", (unsigned long long)n1); return SSQ_EINVAL; }
	if (path != 3) {
		if ((rc = ssq_use_device(device))) {
			if (path != 0 || small) return rc;
			path = 3; // a reference past 2^31 suffixes and no usable device: the host path, no GPU needed
			snprintf(why, sizeof why, "no usable CUDA device");
		} else {
			size_t fr = 0, tot = 0;
			cudaError_t e = cudaMemGetInfo(&fr, &tot);
			if (e != cudaSuccess) { ssq_set_error("cudaMemGetInfo: %s", cudaGetErrorString(e)); return SSQ_ECUDA; }
			const u64 avail = (u64)fr > SP_MARGIN(fr) ? (u64)fr - SP_MARGIN(fr) : 0;
			if (!work) work = avail > fixed ? avail - fixed : 0;
			if (path == 0) {
				if (n1 < SP_MAX_N1 && work >= sp_min_work(n1)) path = 2;
				else {
					path = 3;
					snprintf(why, sizeof why, "%.1f GB of device memory free; the device sort needs %.1f GB for its rank array and text + %.1f GB to work in",
					         fr / 1e9, (fixed + SP_MARGIN(fr)) / 1e9, sp_min_work(n1) / 1e9);
				}
			} else if (!work) {
				ssq_set_error("device index build: %.1f GB of device memory free, %.1f GB needed for the rank array and text before any working space",
				              fr / 1e9, (fixed + SP_MARGIN(fr)) / 1e9);
				return SSQ_ENOMEM;
			}
		}
	}
	st->path = path;
	if ((rc = write_text_files(prefix, ctg, holes, pac, l_pac))) { ssq_set_error("cannot write %s.{ann,amb,pac}", prefix); return rc; }
	if (path == 2) {
		SpDevice be;
		return sp_build(be, pac.data(), pac.size(), l_pac, prefix, work, st);
	}
	const int f = force ? atoi(force) : 0; // entry width: what was asked for, else 32 bits while they suffice, else 40 (5 bytes per suffix)
	rc = build_bwt_sa_host(prefix, pac, l_pac, f == 64 ? 64 : (f == 40 || !small) ? 40 : 32);
	if (!rc) ssq_set_error("%s", why); // why the automatic choice took the host path (empty when it was asked for)
	return rc;
}

extern "C" int ssq_index_build(const char *fasta, const char *prefix, int device)
{
	return ssq_index_build_ex(fasta, prefix, device, 0, 0);
}
