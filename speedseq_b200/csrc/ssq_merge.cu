// ssq_merge.cu — the merge of coordinate-sorted BAM files on the device: the phases of ssq_merge.cuh as kernels, driven by mg_run.
//   window   the compressed window to the device, ssq_gunzip_inflate_bgzf_dev behind the carried bytes (copied from the input's
//            other text buffer: each input has two and alternates).
//   records  k_merge_walk: a thread per segment (the BAI walker); k_merge_records: a thread per segment writes its record
//            offsets; k_merge_keys: a thread per record writes its key and checks the order, the first failure by atomicMin.
//   gather   k_merge_sizes: a thread per output position; cub::DeviceScan gives the output offsets; k_merge_gather: a warp per
//            record copies it.  The buffer goes through ssq_bgzf_deflate_dev (z given) or back to the host.
// Host work: the windows' member tables, the link checks of the walk, sambamba's heap over the keys, the merged header.
// C-ABI: ssq_merge_create / ssq_merge_run / ssq_merge_header / ssq_merge_times / ssq_merge_stream / ssq_merge_free (include/ssq.h).
#include <stdlib.h>
#include <string.h>
#include <vector>
#include <cub/cub.cuh>
#include "ssq_host.h"
#include "ssq_merge.cuh"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { ssq_set_error("%s:%d: %s", __FILE__, __LINE__, cudaGetErrorString(e_)); return SSQ_ECUDA; } } while (0)

__global__ void __launch_bounds__(128) k_merge_walk(const uint8_t *t, bz_u64 n, int n_ref, BaiSeg *seg, const int *which, int nw)
{
	for (int w = blockIdx.x * blockDim.x + threadIdx.x; w < nw; w += gridDim.x * blockDim.x) bai_guess_walk(t, n, n_ref, seg[which[w]]);
}
__global__ void __launch_bounds__(128) k_merge_records(const uint8_t *t, bz_u64 n, const BaiSeg *seg, const bz_u64 *base, int ns, bz_u64 *roff)
{
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < ns; i += gridDim.x * blockDim.x) mg_walk_write(t, n, seg[i], roff + base[i]);
}
__global__ void __launch_bounds__(256) k_merge_keys(const uint8_t *t, const bz_u64 *roff, bz_u64 n, int n_ref, bz_u64 *key, unsigned long long *bad)
{
	for (bz_u64 i = blockIdx.x * (bz_u64)blockDim.x + threadIdx.x; i < n; i += (bz_u64)gridDim.x * blockDim.x) {
		const int e = mg_check(t, roff, i, n_ref, &key[i]);
		if (e) atomicMin(bad, (unsigned long long)(i << 3 | (bz_u64)e));
	}
}
// output position j: (input, record) -> the record's length
__global__ void __launch_bounds__(256) k_merge_sizes(const bz_u64 *order, bz_u64 n, const uint8_t *const *text, const bz_u64 *const *roff, bz_u64 *size)
{
	for (bz_u64 j = blockIdx.x * (bz_u64)blockDim.x + threadIdx.x; j < n; j += (bz_u64)gridDim.x * blockDim.x) {
		const bz_u64 o = order[j];
		size[j] = 4 + (bz_u64)bai_u32(text[o >> MG_IDX_BITS], roff[o >> MG_IDX_BITS][o & MG_IDX_MASK]);
	}
}
__global__ void __launch_bounds__(256) k_merge_gather(const bz_u64 *order, bz_u64 n, const uint8_t *const *text, const bz_u64 *const *roff, const bz_u64 *size,
                                                    const bz_u64 *at, uint8_t *out)
{
	const int lane = threadIdx.x & 31;
	for (bz_u64 j = (blockIdx.x * (bz_u64)blockDim.x + threadIdx.x) >> 5; j < n; j += ((bz_u64)gridDim.x * blockDim.x) >> 5) {
		const bz_u64 o = order[j];
		const uint8_t *src = text[o >> MG_IDX_BITS] + roff[o >> MG_IDX_BITS][o & MG_IDX_MASK];
		uint8_t *dst = out + at[j];
		for (bz_u64 b = lane; b < size[j]; b += 32) dst[b] = src[b];
	}
}

static int grid_of(bz_u64 n, int threads, int sms) { const bz_u64 b = (n + threads - 1) / threads; return b < 1 ? 1 : b < (bz_u64)sms * 8 ? (int)b : sms * 8; }

struct DevMerge : MergeBackend {
	cudaStream_t st; int sms;
	ssq_gunzip_t *g;
	ssq_bgzf_t *z; int level;
	ssq_merge_sink_t sink; void *ctx;
	struct In { DBuf text[2], roff; int cur = 0; };
	std::vector<In> in;
	DBuf d_c, d_seg, d_which, d_base, d_key, d_bad, d_order, d_ptr, d_size, d_at, d_out, d_z, d_tmp;
	uint8_t *h_c = 0, *h_out = 0; size_t h_c_cap = 0, h_out_cap = 0;
	std::vector<uint64_t> mt;
	~DevMerge() { if (h_c) cudaFreeHost(h_c); if (h_out) cudaFreeHost(h_out); }
	static int pinned(uint8_t *&p, size_t &cap, size_t n)
	{
		if (cap >= n) return 0;
		if (p) cudaFreeHost(p);
		p = 0; cap = 0;
		if (cudaMallocHost((void**)&p, n) != cudaSuccess) { p = 0; ssq_set_error("cudaMallocHost(%zu) failed", n); return SSQ_ENOMEM; }
		cap = n;
		return 0;
	}
	uint8_t *text(int k) { return in[k].text[in[k].cur].as<uint8_t>(); }
	int fill(int k, bz_u64 from, bz_u64 keep, const uint8_t *c, bz_u64 clen, const std::vector<GzMember> &m, bz_u64 *err_at) override
	{
		int rc;
		In &I = in[k];
		DBuf &dst = I.text[1 - I.cur];
		const bz_u64 tl = keep + m.back().toff + m.back().isize;
		if ((rc = dst.need(tl + 1)) || (rc = d_c.need(clen)) || (rc = pinned(h_c, h_c_cap, clen))) return rc;
		if (keep) CK(cudaMemcpyAsync(dst.p, I.text[I.cur].as<uint8_t>() + from, keep, cudaMemcpyDeviceToDevice, st));
		memcpy(h_c, c, clen);
		CK(cudaMemcpyAsync(d_c.p, h_c, clen, cudaMemcpyHostToDevice, st));
		if (mt.size() < 2 * m.size()) mt.resize(2 * m.size());
		size_t out_len = 0, nm = 0;
		rc = ssq_gunzip_inflate_bgzf_dev(g, d_c.p, clen, dst.as<uint8_t>() + keep, dst.cap - keep, &out_len, mt.data(), m.size(), &nm);
		if (rc == SSQ_EDATA) { // the member that failed: the first whose offset the device did not confirm
			size_t j = 0;
			while (j < nm && j < m.size() && mt[2 * j] == m[j].coff) ++j;
			*err_at = j < m.size() ? m[j].coff : 0;
		}
		if (rc) return rc;
		if (out_len + keep != tl || nm != m.size()) { *err_at = 0; return SSQ_EDATA; }
		I.cur = 1 - I.cur;
		return 0;
	}
	int peek(int k, bz_u64 at, void *buf, u32 len) override
	{
		CK(cudaMemcpyAsync(buf, text(k) + at, len, cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		return 0;
	}
	int walk(int k, std::vector<BaiSeg> &seg, const std::vector<int> &which, int n_ref) override
	{
		int rc;
		const size_t ns = seg.size(), nw = which.size();
		if ((rc = d_seg.need(ns * sizeof(BaiSeg))) || (rc = d_which.need(nw * 4))) return rc;
		CK(cudaMemcpyAsync(d_seg.p, seg.data(), ns * sizeof(BaiSeg), cudaMemcpyHostToDevice, st));
		CK(cudaMemcpyAsync(d_which.p, which.data(), nw * 4, cudaMemcpyHostToDevice, st));
		k_merge_walk<<<grid_of(nw, 128, sms), 128, 0, st>>>(text(k), seg.back().lim, n_ref, d_seg.as<BaiSeg>(), d_which.as<int>(), (int)nw);
		CK(cudaGetLastError());
		CK(cudaMemcpyAsync(seg.data(), d_seg.p, ns * sizeof(BaiSeg), cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		return 0;
	}
	int records(int k, const std::vector<BaiSeg> &seg, const std::vector<bz_u64> &base, bz_u64 n_rec, int n_ref, std::vector<bz_u64> &keys, bz_u64 *bad) override
	{
		int rc;
		const size_t ns = seg.size();
		const bz_u64 n = seg.back().lim;
		if ((rc = d_seg.need(ns * sizeof(BaiSeg))) || (rc = d_base.need((ns + 1) * 8)) || (rc = in[k].roff.need(n_rec * 8)) || (rc = d_key.need(n_rec * 8)) || (rc = d_bad.need(8))) return rc;
		CK(cudaMemcpyAsync(d_seg.p, seg.data(), ns * sizeof(BaiSeg), cudaMemcpyHostToDevice, st));
		CK(cudaMemcpyAsync(d_base.p, base.data(), (ns + 1) * 8, cudaMemcpyHostToDevice, st));
		CK(cudaMemsetAsync(d_bad.p, 0xff, 8, st));
		k_merge_records<<<grid_of(ns, 128, sms), 128, 0, st>>>(text(k), n, d_seg.as<BaiSeg>(), d_base.as<bz_u64>(), (int)ns, in[k].roff.as<bz_u64>());
		k_merge_keys<<<grid_of(n_rec, 256, sms), 256, 0, st>>>(text(k), in[k].roff.as<bz_u64>(), n_rec, n_ref, d_key.as<bz_u64>(), d_bad.as<unsigned long long>());
		CK(cudaGetLastError());
		keys.resize(n_rec);
		CK(cudaMemcpyAsync(keys.data(), d_key.p, n_rec * 8, cudaMemcpyDeviceToHost, st));
		CK(cudaMemcpyAsync(bad, d_bad.p, 8, cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		return 0;
	}
	int gather(const std::vector<bz_u64> &order, bz_u64 bytes_max) override
	{
		int rc;
		const bz_u64 n = order.size();
		const size_t ni = in.size();
		std::vector<const void*> ptr(2 * ni);
		for (size_t k = 0; k < ni; ++k) { ptr[k] = text((int)k); ptr[ni + k] = in[k].roff.p; }
		if ((rc = d_order.need(n * 8)) || (rc = d_ptr.need(2 * ni * sizeof(void*))) || (rc = d_size.need(n * 8)) || (rc = d_at.need(n * 8)) || (rc = d_out.need(bytes_max + 1))) return rc;
		CK(cudaMemcpyAsync(d_order.p, order.data(), n * 8, cudaMemcpyHostToDevice, st));
		CK(cudaMemcpyAsync(d_ptr.p, ptr.data(), 2 * ni * sizeof(void*), cudaMemcpyHostToDevice, st));
		const uint8_t *const *tp = d_ptr.as<const uint8_t*>();
		const bz_u64 *const *rp = d_ptr.as<const bz_u64*>() + ni;
		k_merge_sizes<<<grid_of(n, 256, sms), 256, 0, st>>>(d_order.as<bz_u64>(), n, tp, rp, d_size.as<bz_u64>());
		size_t tb = 0;
		CK(cub::DeviceScan::ExclusiveSum(0, tb, d_size.as<bz_u64>(), d_at.as<bz_u64>(), (int)n, st));
		if ((rc = d_tmp.need(tb))) return rc;
		CK(cub::DeviceScan::ExclusiveSum(d_tmp.p, tb, d_size.as<bz_u64>(), d_at.as<bz_u64>(), (int)n, st));
		k_merge_gather<<<grid_of(n * 32, 256, sms), 256, 0, st>>>(d_order.as<bz_u64>(), n, tp, rp, d_size.as<bz_u64>(), d_at.as<bz_u64>(), d_out.as<uint8_t>());
		CK(cudaGetLastError());
		bz_u64 last[2];
		CK(cudaMemcpyAsync(&last[0], d_at.as<bz_u64>() + n - 1, 8, cudaMemcpyDeviceToHost, st));
		CK(cudaMemcpyAsync(&last[1], d_size.as<bz_u64>() + n - 1, 8, cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		bz_u64 len = last[0] + last[1];
		const uint8_t *src = d_out.as<uint8_t>();
		if (z) { // BGZF members of the records on the device (no end-of-file block: the caller writes it)
			size_t cap = len + (len / 0xff00 + 1) * 64 + 64, clen = 0, need = 0;
			if ((rc = d_z.need(cap))) return rc;
			rc = ssq_bgzf_deflate_dev(z, d_out.p, len, level, 0, d_z.p, d_z.cap, &clen, &need);
			if (rc == SSQ_ECAP) { if ((rc = d_z.need(need))) return rc; rc = ssq_bgzf_deflate_dev(z, d_out.p, len, level, 0, d_z.p, d_z.cap, &clen, &need); }
			if (rc) return rc;
			src = d_z.as<uint8_t>(); len = clen;
		}
		if ((rc = pinned(h_out, h_out_cap, len))) return rc;
		CK(cudaMemcpyAsync(h_out, src, len, cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		if (sink(ctx, h_out, len)) { ssq_set_error("the output could not be written"); return SSQ_EIO; }
		return 0;
	}
};

struct ssq_merge {
	int device;
	size_t window;
	ssq_gunzip_t *g;
	float ms[3];
};

extern "C" int ssq_merge_create(int device, size_t window_bytes, ssq_merge_t **out)
{
	if (!out) { ssq_set_error("ssq_merge_create: invalid arguments"); return SSQ_EINVAL; }
	*out = 0;
	int rc = ssq_use_device(device);
	if (rc) return rc;
	ssq_merge *m = new ssq_merge();
	m->device = device; m->window = window_bytes ? window_bytes : MG_WINDOW_DEFAULT;
	memset(m->ms, 0, sizeof m->ms);
	if ((rc = ssq_gunzip_create(device, 0, &m->g))) { delete m; return rc; }
	*out = m;
	return SSQ_OK;
}

extern "C" void ssq_merge_free(ssq_merge_t *m)
{
	if (!m) return;
	cudaSetDevice(m->device);
	ssq_gunzip_free(m->g);
	delete m;
}

extern "C" void *ssq_merge_stream(ssq_merge_t *m) { return m ? ssq_gunzip_stream(m->g) : 0; }

extern "C" int ssq_merge_times(const ssq_merge_t *m, float ms[3])
{
	if (!m || !ms) return SSQ_EINVAL;
	memcpy(ms, m->ms, sizeof m->ms);
	return SSQ_OK;
}

extern "C" int ssq_merge_header(const char *const *paths, int n_in, char **text)
{
	if (!paths || !text) { ssq_set_error("ssq_merge_header: invalid arguments"); return SSQ_EINVAL; }
	*text = 0;
	std::vector<MgInput> in;
	std::string t;
	const int rc = mg_open(paths, n_in, in, t);
	if (rc) return rc;
	if (!(*text = (char*)malloc(t.size() + 1))) return SSQ_ENOMEM;
	memcpy(*text, t.c_str(), t.size() + 1);
	return SSQ_OK;
}

extern "C" int ssq_merge_run(ssq_merge_t *m, const char *const *paths, int n_in, ssq_bgzf_t *z, int level, ssq_merge_sink_t sink, void *ctx, uint64_t *n_records)
{
	if (!m || !paths || !sink) { ssq_set_error("ssq_merge_run: invalid arguments"); return SSQ_EINVAL; }
	int rc = ssq_use_device(m->device);
	if (rc) return rc;
	std::vector<MgInput> in;
	std::string text;
	if ((rc = mg_open(paths, n_in, in, text))) return rc;
	const std::string hdr = mg_bam_header(text, in[0]);
	if (z) { // the header in blocks of its own
		void *out = 0; size_t len = 0;
		if ((rc = ssq_bgzf_deflate(z, hdr.data(), hdr.size(), level, 0, &out, &len))) return rc;
		rc = sink(ctx, out, len);
		free(out);
	} else rc = sink(ctx, hdr.data(), hdr.size());
	if (rc) { ssq_set_error("the output could not be written"); return SSQ_EIO; }
	DevMerge be;
	be.g = m->g; be.st = (cudaStream_t)ssq_gunzip_stream(m->g); be.z = z; be.level = level; be.sink = sink; be.ctx = ctx;
	be.in.resize(n_in);
	if (cudaDeviceGetAttribute(&be.sms, cudaDevAttrMultiProcessorCount, m->device) != cudaSuccess) { ssq_set_error("ssq_merge_run: no SM count"); return SSQ_ECUDA; }
	double ms[3] = {0, 0, 0};
	bz_u64 n = 0;
	rc = mg_run(be, in, m->window, BAI_SEG_DEFAULT, &n, ms);
	for (int i = 0; i < 3; ++i) m->ms[i] = (float)ms[i];
	if (n_records) *n_records = n;
	return rc;
}
