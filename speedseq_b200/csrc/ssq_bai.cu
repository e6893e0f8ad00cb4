// ssq_bai.cu — the BAI builder on the device: the phases of ssq_bai.cuh as kernels, driven by bai_from_text.
//   inflate  ssq_gunzip_inflate_bgzf_dev (ssq_gunzip.cu): one thread per member, the text at its final place, the member table.
//   walk     a thread per segment (guess, then follow the chain); broken links walked again, round by round.
//   records  a thread per segment writes its records at the segment's place (running sum of the counts on the host).
//   check    a thread per record; the first failing record by atomicMin, the records with a reference by atomicMax.
//   index    run starts -> cub::DeviceSelect; per run its key and chunk; cub::DeviceRadixSort (stable) by (reference, bin);
//            chunk and bin starts -> cub::DeviceScan; chunks and bins written by a thread per run; linear index by atomicMin of
//            start offsets over each record's windows, then one thread per reference fills the untouched windows; metadata by a
//            thread per record (first and last of its reference), mapped / unmapped counts warp-aggregated.
// Host work: the header, the link check, the running sum of segment counts, the bin order of sambamba's hash table and the bytes.
// C-ABI: ssq_bai_create / ssq_bai_build / ssq_bai_times / ssq_bai_stream / ssq_bai_free (include/ssq.h).
#include <stdlib.h>
#include <string.h>
#include <vector>
#include <cub/cub.cuh>
#include "ssq_host.h"
#include "ssq_bai.cuh"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { ssq_set_error("%s:%d: %s", __FILE__, __LINE__, cudaGetErrorString(e_)); return SSQ_ECUDA; } } while (0)

__global__ void __launch_bounds__(128) k_bai_walk(const uint8_t *t, bz_u64 n, int n_ref, BaiSeg *seg, const int *which, int nw)
{
	for (int w = blockIdx.x * blockDim.x + threadIdx.x; w < nw; w += gridDim.x * blockDim.x) bai_guess_walk(t, n, n_ref, seg[which[w]]);
}
__global__ void __launch_bounds__(128) k_bai_records(const uint8_t *t, bz_u64 n, const BaiSeg *seg, const bz_u64 *base, int ns, const GzMember *m, bz_u64 nm, bz_u64 clen, BaiRec *rec)
{
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < ns; i += gridDim.x * blockDim.x) bai_walk_write(t, n, seg[i], m, nm, clen, rec + base[i]);
}
__global__ void __launch_bounds__(256) k_bai_check(const BaiRec *rec, bz_u64 n, int n_ref, unsigned long long *res)
{
	for (bz_u64 i = blockIdx.x * (bz_u64)blockDim.x + threadIdx.x; i < n; i += (bz_u64)gridDim.x * blockDim.x) {
		const int e = bai_check(rec, i, n_ref);
		if (e) atomicMin(&res[0], (unsigned long long)(i << 3 | (bz_u64)e));
		if (rec[i].ref >= 0) atomicMax(&res[1], (unsigned long long)(i + 1));
	}
}
__global__ void __launch_bounds__(256) k_bai_run_flags(const BaiRec *rec, bz_u64 P, uint8_t *flag)
{
	for (bz_u64 i = blockIdx.x * (bz_u64)blockDim.x + threadIdx.x; i < P; i += (bz_u64)gridDim.x * blockDim.x) flag[i] = bai_run_start(rec, i);
}
// run j: key, chunk (start of its first record, end of its last)
__global__ void __launch_bounds__(256) k_bai_runs(const BaiRec *rec, bz_u64 P, const u32 *first, const int *nrun_p, bz_u64 *key, u32 *val, BaiChunk *ch)
{
	const int nrun = *nrun_p;
	for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nrun; j += gridDim.x * blockDim.x) {
		const bz_u64 f = first[j], l = (j + 1 < nrun ? first[j + 1] : P) - 1;
		key[j] = bai_run_key(rec[f]); val[j] = (u32)j;
		ch[j].beg = rec[f].vbeg; ch[j].end = rec[l].vend;
	}
}
// in sorted order: does run j open a chunk, a bin
__global__ void __launch_bounds__(256) k_bai_opens(const bz_u64 *key, const u32 *val, const BaiChunk *ch, const int *nrun_p, u32 *newc, u32 *newb)
{
	const int nrun = *nrun_p;
	for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nrun; j += gridDim.x * blockDim.x) {
		newb[j] = !j || key[j - 1] != key[j];
		newc[j] = !j || bai_new_chunk(key[j - 1], ch[val[j - 1]].end, key[j], ch[val[j]].beg);
	}
}
__global__ void __launch_bounds__(256) k_bai_chunks(const bz_u64 *key, const u32 *val, const BaiChunk *ch, const int *nrun_p, const u32 *newc, const u32 *newb,
                                                  const u32 *cidx, const u32 *bidx, BaiChunk *out, BaiBin *bins)
{
	const int nrun = *nrun_p;
	for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nrun; j += gridDim.x * blockDim.x) {
		const u32 c = cidx[j] - 1, b = bidx[j] - 1; // inclusive sums: run j belongs to chunk c and bin b
		const bool lastc = j + 1 == nrun || newc[j + 1], lastb = j + 1 == nrun || newb[j + 1];
		if (newc[j]) out[c].beg = ch[val[j]].beg;
		if (lastc) out[c].end = ch[val[j]].end;
		if (newb[j]) { bins[b].ref = (int32_t)(key[j] >> 16); bins[b].bin = (u32)(key[j] & 0xffff); bins[b].first_run = val[j]; bins[b].lo = c; }
		if (lastb) bins[b].hi = c + 1;
	}
}
__global__ void __launch_bounds__(256) k_bai_nint(const BaiRec *rec, bz_u64 P, u32 *nint)
{
	for (bz_u64 i = blockIdx.x * (bz_u64)blockDim.x + threadIdx.x; i < P; i += (bz_u64)gridDim.x * blockDim.x) {
		long long w0, w1; bai_windows(rec[i], &w0, &w1);
		if (w1 > 0) atomicMax(&nint[rec[i].ref], (u32)w1);
	}
}
__global__ void __launch_bounds__(256) k_bai_lin(const BaiRec *rec, bz_u64 P, const bz_u64 *lbase, unsigned long long *lin)
{
	for (bz_u64 i = blockIdx.x * (bz_u64)blockDim.x + threadIdx.x; i < P; i += (bz_u64)gridDim.x * blockDim.x) {
		long long w0, w1; bai_windows(rec[i], &w0, &w1);
		for (long long w = w0; w < w1; ++w) atomicMin(&lin[lbase[rec[i].ref] + w], (unsigned long long)rec[i].vbeg);
	}
}
__global__ void k_bai_lin_fill(const bz_u64 *lbase, int n_ref, bz_u64 *lin)
{
	for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < n_ref; r += gridDim.x * blockDim.x) {
		bz_u64 prev = 0;
		for (bz_u64 w = lbase[r]; w < lbase[r + 1]; ++w) { if (lin[w] == BAI_NONE) lin[w] = prev; prev = lin[w]; }
	}
}
// metadata: meta[4r] first start, [4r+1] last end, [4r+2] mapped, [4r+3] unmapped; has[r]
__global__ void __launch_bounds__(256) k_bai_meta(const BaiRec *rec, bz_u64 P, bz_u64 n_rec, unsigned long long *meta, uint8_t *has)
{
	const bz_u64 stride = (bz_u64)gridDim.x * blockDim.x;
	for (bz_u64 i0 = blockIdx.x * (bz_u64)blockDim.x; i0 < P; i0 += stride) { // whole warps stay in the loop: the counts are aggregated per warp
		const bz_u64 i = i0 + threadIdx.x;
		const bool in = i < P;
		int k = -1, slot = 0;
		if (in) {
			const BaiRec &c = rec[i];
			k = c.ref;
			if (!i || rec[i - 1].ref != k) { has[k] = 1; meta[4 * k] = c.vbeg; }
			if (i + 1 == P) meta[4 * k + 1] = rec[n_rec - 1].vend; else if (rec[i + 1].ref != k) meta[4 * k + 1] = c.vend;
			slot = 4 * k + ((c.flag & 4) ? 3 : 2);
		}
		const unsigned peers = __match_any_sync(0xffffffffu, in ? slot : -1);
		if (in && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&meta[slot], (unsigned long long)__popc(peers));
	}
}

static int grid_of(bz_u64 n, int threads, int sms) { const bz_u64 b = (n + threads - 1) / threads; return b < 1 ? 1 : b < (bz_u64)sms * 8 ? (int)b : sms * 8; }

struct DevBai : BaiBackend {
	cudaStream_t st; int sms;
	const uint8_t *t; bz_u64 n, clen, nm;
	const GzMember *d_m;
	cudaEvent_t ev_index;
	void phase() override { cudaEventRecord(ev_index, st); }
	DBuf d_seg, d_which, d_base, d_rec, d_res, d_flag, d_first, d_nsel, d_key[2], d_val[2], d_ch, d_newc, d_newb, d_cidx, d_bidx, d_chunks, d_bins,
	     d_nint, d_lbase, d_lin, d_meta, d_has, d_tmp;
	int walk(std::vector<BaiSeg> &seg, const std::vector<int> &which, int n_ref) override
	{
		int rc;
		const size_t ns = seg.size(), nw = which.size();
		if ((rc = d_seg.need(ns * sizeof(BaiSeg))) || (rc = d_which.need(nw * 4))) return rc;
		CK(cudaMemcpyAsync(d_seg.p, seg.data(), ns * sizeof(BaiSeg), cudaMemcpyHostToDevice, st));
		CK(cudaMemcpyAsync(d_which.p, which.data(), nw * 4, cudaMemcpyHostToDevice, st));
		k_bai_walk<<<grid_of(nw, 128, sms), 128, 0, st>>>(t, n, n_ref, d_seg.as<BaiSeg>(), d_which.as<int>(), (int)nw);
		CK(cudaGetLastError());
		CK(cudaMemcpyAsync(seg.data(), d_seg.p, ns * sizeof(BaiSeg), cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		return 0;
	}
	int records(const std::vector<BaiSeg> &seg, const std::vector<bz_u64> &base, bz_u64 n_rec) override
	{
		int rc;
		const size_t ns = seg.size();
		if ((rc = d_seg.need(ns * sizeof(BaiSeg))) || (rc = d_base.need((ns + 1) * 8)) || (rc = d_rec.need((n_rec ? n_rec : 1) * sizeof(BaiRec)))) return rc;
		CK(cudaMemcpyAsync(d_seg.p, seg.data(), ns * sizeof(BaiSeg), cudaMemcpyHostToDevice, st));
		CK(cudaMemcpyAsync(d_base.p, base.data(), (ns + 1) * 8, cudaMemcpyHostToDevice, st));
		k_bai_records<<<grid_of(ns, 128, sms), 128, 0, st>>>(t, n, d_seg.as<BaiSeg>(), d_base.as<bz_u64>(), (int)ns, d_m, nm, clen, d_rec.as<BaiRec>());
		CK(cudaGetLastError());
		return 0;
	}
	int check(bz_u64 n_rec, int n_ref, bz_u64 *first_bad, bz_u64 *n_pos) override
	{
		int rc;
		if ((rc = d_res.need(16))) return rc;
		bz_u64 init[2] = {BAI_NONE, 0};
		CK(cudaMemcpyAsync(d_res.p, init, 16, cudaMemcpyHostToDevice, st));
		if (n_rec) k_bai_check<<<grid_of(n_rec, 256, sms), 256, 0, st>>>(d_rec.as<BaiRec>(), n_rec, n_ref, d_res.as<unsigned long long>());
		CK(cudaGetLastError());
		CK(cudaMemcpyAsync(init, d_res.p, 16, cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		*first_bad = init[0]; *n_pos = init[1];
		return 0;
	}
	int rec_at(bz_u64 i, BaiRec *r) override
	{
		CK(cudaMemcpyAsync(r, d_rec.as<BaiRec>() + i, sizeof(BaiRec), cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		return 0;
	}
	int index(bz_u64 n_rec, bz_u64 P, int n_ref, BaiOut &o) override
	{
		int rc;
		const bz_u64 np = P ? P : 1;
		if ((rc = d_flag.need(np)) || (rc = d_first.need(np * 4)) || (rc = d_nsel.need(4)) || (rc = d_key[0].need(np * 8)) || (rc = d_key[1].need(np * 8)) ||
		    (rc = d_val[0].need(np * 4)) || (rc = d_val[1].need(np * 4)) || (rc = d_ch.need(np * sizeof(BaiChunk))) || (rc = d_newc.need(np * 4)) ||
		    (rc = d_newb.need(np * 4)) || (rc = d_cidx.need(np * 4)) || (rc = d_bidx.need(np * 4)) || (rc = d_chunks.need(np * sizeof(BaiChunk))) ||
		    (rc = d_bins.need(np * sizeof(BaiBin))) || (rc = d_nint.need(((size_t)n_ref + 1) * 4)) || (rc = d_lbase.need(((size_t)n_ref + 1) * 8)) ||
		    (rc = d_meta.need(((size_t)n_ref + 1) * 32)) || (rc = d_has.need((size_t)n_ref + 1)))
			return rc;
		int nrun = 0;
		const int gP = grid_of(np, 256, sms);
		if (P) {
			// runs
			k_bai_run_flags<<<gP, 256, 0, st>>>(d_rec.as<BaiRec>(), P, d_flag.as<uint8_t>());
			cub::CountingInputIterator<u32> iota(0);
			size_t tb = 0;
			CK(cub::DeviceSelect::Flagged(0, tb, iota, d_flag.as<uint8_t>(), d_first.as<u32>(), d_nsel.as<int>(), (int)P, st));
			if ((rc = d_tmp.need(tb))) return rc;
			CK(cub::DeviceSelect::Flagged(d_tmp.p, tb, iota, d_flag.as<uint8_t>(), d_first.as<u32>(), d_nsel.as<int>(), (int)P, st));
			k_bai_runs<<<gP, 256, 0, st>>>(d_rec.as<BaiRec>(), P, d_first.as<u32>(), d_nsel.as<int>(), d_key[0].as<bz_u64>(), d_val[0].as<u32>(), d_ch.as<BaiChunk>());
			CK(cudaMemcpyAsync(&nrun, d_nsel.p, 4, cudaMemcpyDeviceToHost, st));
			CK(cudaStreamSynchronize(st));
			// by (reference, bin), file order kept
			cub::DoubleBuffer<bz_u64> kb(d_key[0].as<bz_u64>(), d_key[1].as<bz_u64>());
			cub::DoubleBuffer<u32> vb(d_val[0].as<u32>(), d_val[1].as<u32>());
			int endbit = 16;
			while (endbit < 48 && ((bz_u64)n_ref >> (endbit - 16))) ++endbit;
			tb = 0;
			CK(cub::DeviceRadixSort::SortPairs(0, tb, kb, vb, nrun, 0, endbit, st));
			if ((rc = d_tmp.need(tb))) return rc;
			CK(cub::DeviceRadixSort::SortPairs(d_tmp.p, tb, kb, vb, nrun, 0, endbit, st));
			k_bai_opens<<<gP, 256, 0, st>>>(kb.Current(), vb.Current(), d_ch.as<BaiChunk>(), d_nsel.as<int>(), d_newc.as<u32>(), d_newb.as<u32>());
			tb = 0;
			CK(cub::DeviceScan::InclusiveSum(0, tb, d_newc.as<u32>(), d_cidx.as<u32>(), nrun, st));
			if ((rc = d_tmp.need(tb))) return rc;
			CK(cub::DeviceScan::InclusiveSum(d_tmp.p, tb, d_newc.as<u32>(), d_cidx.as<u32>(), nrun, st));
			CK(cub::DeviceScan::InclusiveSum(d_tmp.p, tb, d_newb.as<u32>(), d_bidx.as<u32>(), nrun, st));
			k_bai_chunks<<<gP, 256, 0, st>>>(kb.Current(), vb.Current(), d_ch.as<BaiChunk>(), d_nsel.as<int>(), d_newc.as<u32>(), d_newb.as<u32>(),
			                                 d_cidx.as<u32>(), d_bidx.as<u32>(), d_chunks.as<BaiChunk>(), d_bins.as<BaiBin>());
			CK(cudaGetLastError());
		}
		// linear index
		CK(cudaMemsetAsync(d_nint.p, 0, ((size_t)n_ref + 1) * 4, st));
		if (P) k_bai_nint<<<gP, 256, 0, st>>>(d_rec.as<BaiRec>(), P, d_nint.as<u32>());
		std::vector<u32> nint(n_ref + 1);
		CK(cudaMemcpyAsync(nint.data(), d_nint.p, ((size_t)n_ref + 1) * 4, cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		o.lin_base.assign(n_ref + 1, 0);
		for (int r = 0; r < n_ref; ++r) o.lin_base[r + 1] = o.lin_base[r] + nint[r];
		const bz_u64 nl = o.lin_base[n_ref];
		if ((rc = d_lin.need((nl ? nl : 1) * 8))) return rc;
		CK(cudaMemcpyAsync(d_lbase.p, o.lin_base.data(), ((size_t)n_ref + 1) * 8, cudaMemcpyHostToDevice, st));
		CK(cudaMemsetAsync(d_lin.p, 0xff, (nl ? nl : 1) * 8, st));
		CK(cudaMemsetAsync(d_meta.p, 0, ((size_t)n_ref + 1) * 32, st));
		CK(cudaMemsetAsync(d_has.p, 0, (size_t)n_ref + 1, st));
		if (P) {
			k_bai_lin<<<gP, 256, 0, st>>>(d_rec.as<BaiRec>(), P, d_lbase.as<bz_u64>(), d_lin.as<unsigned long long>());
			k_bai_lin_fill<<<grid_of(n_ref, 32, sms), 32, 0, st>>>(d_lbase.as<bz_u64>(), n_ref, d_lin.as<bz_u64>());
			k_bai_meta<<<gP, 256, 0, st>>>(d_rec.as<BaiRec>(), P, n_rec, d_meta.as<unsigned long long>(), d_has.as<uint8_t>());
			CK(cudaGetLastError());
		}
		// to the host
		int nc = 0, nb = 0;
		if (nrun) {
			CK(cudaMemcpyAsync(&nc, d_cidx.as<u32>() + nrun - 1, 4, cudaMemcpyDeviceToHost, st));
			CK(cudaMemcpyAsync(&nb, d_bidx.as<u32>() + nrun - 1, 4, cudaMemcpyDeviceToHost, st));
			CK(cudaStreamSynchronize(st));
		}
		o.chunks.resize(nc); o.bins.resize(nb); o.lin.resize(nl); o.meta.resize(4 * (size_t)n_ref); o.has.resize(n_ref);
		if (nc) CK(cudaMemcpyAsync(o.chunks.data(), d_chunks.p, (size_t)nc * sizeof(BaiChunk), cudaMemcpyDeviceToHost, st));
		if (nb) CK(cudaMemcpyAsync(o.bins.data(), d_bins.p, (size_t)nb * sizeof(BaiBin), cudaMemcpyDeviceToHost, st));
		if (nl) CK(cudaMemcpyAsync(o.lin.data(), d_lin.p, nl * 8, cudaMemcpyDeviceToHost, st));
		if (n_ref) {
			CK(cudaMemcpyAsync(o.meta.data(), d_meta.p, (size_t)n_ref * 32, cudaMemcpyDeviceToHost, st));
			CK(cudaMemcpyAsync(o.has.data(), d_has.p, (size_t)n_ref, cudaMemcpyDeviceToHost, st));
		}
		CK(cudaStreamSynchronize(st));
		return 0;
	}
};

struct ssq_bai {
	int device;
	size_t seg;
	ssq_gunzip_t *g;
	DevBai be;
	DBuf d_in, d_text, d_m;
	uint8_t *h_in; size_t h_cap;
	std::vector<uint64_t> mt;
	cudaEvent_t ev[4];
	float ms[3];
};

extern "C" int ssq_bai_create(int device, size_t seg_bytes, ssq_bai_t **out)
{
	if (!out || (seg_bytes && seg_bytes < 64)) { ssq_set_error("ssq_bai_create: invalid arguments"); return SSQ_EINVAL; }
	*out = 0;
	int rc = ssq_use_device(device);
	if (rc) return rc;
	ssq_bai *b = new ssq_bai();
	b->device = device; b->seg = seg_bytes ? seg_bytes : BAI_SEG_DEFAULT; b->g = 0; b->h_in = 0; b->h_cap = 0;
	memset(b->ms, 0, sizeof b->ms);
	for (int i = 0; i < 4; ++i) b->ev[i] = 0;
	if ((rc = ssq_gunzip_create(device, 0, &b->g))) { delete b; return rc; }
	b->be.st = (cudaStream_t)ssq_gunzip_stream(b->g);
	for (int i = 0; i < 4; ++i) if (cudaEventCreate(&b->ev[i]) != cudaSuccess) { ssq_set_error("ssq_bai_create: cudaEventCreate failed"); ssq_bai_free(b); return SSQ_ECUDA; }
	if (cudaDeviceGetAttribute(&b->be.sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess) { ssq_set_error("ssq_bai_create: no SM count"); ssq_bai_free(b); return SSQ_ECUDA; }
	*out = b;
	return SSQ_OK;
}

extern "C" void ssq_bai_free(ssq_bai_t *b)
{
	if (!b) return;
	cudaSetDevice(b->device);
	if (b->be.st) cudaStreamSynchronize(b->be.st);
	for (int i = 0; i < 4; ++i) if (b->ev[i]) cudaEventDestroy(b->ev[i]);
	if (b->h_in) cudaFreeHost(b->h_in);
	ssq_gunzip_free(b->g);
	delete b;
}

extern "C" void *ssq_bai_stream(ssq_bai_t *b) { return b ? (void*)b->be.st : 0; }

extern "C" int ssq_bai_times(const ssq_bai_t *b, float ms[3])
{
	if (!b || !ms) return SSQ_EINVAL;
	memcpy(ms, b->ms, sizeof b->ms);
	return SSQ_OK;
}

extern "C" int ssq_bai_build(ssq_bai_t *b, const void *bam, size_t len, void **bai_out, size_t *bai_len)
{
	if (!b || (!bam && len) || !bai_out || !bai_len) { ssq_set_error("ssq_bai_build: invalid arguments"); return SSQ_EINVAL; }
	*bai_out = 0; *bai_len = 0;
	int rc = ssq_use_device(b->device);
	if (rc) return rc;
	cudaStream_t st = b->be.st;
	if (!len) { ssq_set_error("ssq_bai_build: not a BAM file: empty input"); return SSQ_EFORMAT; }
	// stage through pinned memory
	if (b->h_cap < len) {
		if (b->h_in) cudaFreeHost(b->h_in);
		b->h_in = 0; b->h_cap = 0;
		if (cudaMallocHost((void**)&b->h_in, len) != cudaSuccess) { b->h_in = 0; ssq_set_error("ssq_bai_build: cudaMallocHost(%zu) failed", len); return SSQ_ENOMEM; }
		b->h_cap = len;
	}
	if ((rc = b->d_in.need(len))) return rc;
	CK(cudaEventRecord(b->ev[0], st));
	const size_t piece = 64u << 20; // each piece has its own place in h_in: it is copied in while the next one is staged
	for (size_t at = 0; at < len; at += piece) {
		const size_t k = len - at < piece ? len - at : piece;
		memcpy(b->h_in + at, (const uint8_t*)bam + at, k);
		CK(cudaMemcpyAsync(b->d_in.as<uint8_t>() + at, b->h_in + at, k, cudaMemcpyHostToDevice, st));
	}
	// inflate (grow the buffers once when the text or the member table does not fit)
	size_t tl = 0, nm = 0;
	for (int pass = 0;; ++pass) {
		if (b->mt.size() < 2) b->mt.resize(2);
		rc = ssq_gunzip_inflate_bgzf_dev(b->g, b->d_in.p, len, b->d_text.p, b->d_text.cap, &tl, b->mt.data(), b->mt.size() / 2, &nm);
		if (rc != SSQ_ECAP || pass) break;
		if ((rc = b->d_text.need(tl ? tl : 1))) return rc;
		if (b->mt.size() < 2 * nm) b->mt.resize(2 * nm);
	}
	if (rc) { const std::string e = ssq_last_error(); ssq_set_error("ssq_bai_build: %s", e.c_str()); return rc; }
	CK(cudaEventRecord(b->ev[1], st));
	std::vector<GzMember> m(nm);
	for (size_t k = 0; k < nm; ++k) {
		m[k].coff = b->mt[2 * k]; m[k].toff = b->mt[2 * k + 1];
		m[k].csize = (u32)((k + 1 < nm ? b->mt[2 * k + 2] : len) - m[k].coff);
		m[k].isize = (u32)((k + 1 < nm ? b->mt[2 * k + 3] : tl) - m[k].toff);
	}
	if (!nm) { ssq_set_error("ssq_bai_build: not a BAM file: no BGZF member"); return SSQ_EFORMAT; }
	if ((rc = b->d_m.need(nm * sizeof(GzMember)))) return rc;
	CK(cudaMemcpyAsync(b->d_m.p, m.data(), nm * sizeof(GzMember), cudaMemcpyHostToDevice, st));
	DevBai &be = b->be;
	be.t = b->d_text.as<uint8_t>(); be.n = tl; be.clen = len; be.nm = nm; be.d_m = b->d_m.as<GzMember>();
	auto fetch = [&](bz_u64 k, uint8_t *buf) { CK(cudaMemcpyAsync(buf, b->d_text.p, k, cudaMemcpyDeviceToHost, st)); CK(cudaStreamSynchronize(st)); return 0; };
	std::string bai;
	be.ev_index = b->ev[2];
	rc = bai_from_text(be, fetch, tl, m, b->seg, bai);
	if (rc) { if (rc == SSQ_EFORMAT) { const std::string e = ssq_last_error(); ssq_set_error("ssq_bai_build: %s", e.c_str()); } return rc; }
	CK(cudaEventRecord(b->ev[3], st));
	CK(cudaEventSynchronize(b->ev[3]));
	CK(cudaEventElapsedTime(&b->ms[0], b->ev[0], b->ev[1]));
	CK(cudaEventElapsedTime(&b->ms[1], b->ev[1], b->ev[2]));
	CK(cudaEventElapsedTime(&b->ms[2], b->ev[2], b->ev[3]));
	if (!(*bai_out = malloc(bai.size()))) { ssq_set_error("ssq_bai_build: out of memory"); return SSQ_ENOMEM; }
	memcpy(*bai_out, bai.data(), bai.size());
	*bai_len = bai.size();
	return SSQ_OK;
}
