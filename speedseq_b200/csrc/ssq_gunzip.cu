// ssq_gunzip.cu — gzip decoding on the device: the phases of ssq_gunzip.cuh as kernels (sync search: one warp per chunk, a lane
// per candidate bit offset; decode: one warp per chunk, its first lane decoding, the Huffman tables in shared memory; resolve: one
// CTA over the chunk tails in order, then a block per chunk; CRC: a thread per piece), driven window by window by gz_window.
// Grids are sized from the SM count.  Device memory per object is fixed at create: GZ_MAXCH slots of GZ_SLOT 16-bit symbols (1 GB),
// the window's text behind 32 KB of context (512 MB) and the window's compressed input (GZ_MAXCH chunks + 1 MB).
// C-ABI: ssq_gunzip_create / ssq_gunzip_inflate / ssq_gunzip_inflate_dev / ssq_gunzip_stats (include/ssq.h).
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "ssq_host.h"
#include "ssq_gunzip.cuh"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { ssq_set_error("%s:%d: %s", __FILE__, __LINE__, cudaGetErrorString(e_)); return SSQ_ECUDA; } } while (0)

__global__ void __launch_bounds__(32) k_gz_sync(GzIn I, int n, bz_u64 lo, bz_u64 cbits, bz_u64 wend, bz_u64 *s)
{
	extern __shared__ __align__(16) unsigned char gz_sm[];
	GzTab &T = reinterpret_cast<GzTab*>(gz_sm)[threadIdx.x];
	const int lane = threadIdx.x;
	for (int i = 1 + blockIdx.x; i < n; i += gridDim.x) {
		const bz_u64 a = lo + (bz_u64)i * cbits, b = a + cbits < wend ? a + cbits : wend;
		bz_u64 found = GZ_NONE;
		for (u32 r = 0; a + (bz_u64)r * 32 < b; ++r) {
			bz_u64 c;
			const unsigned m = __ballot_sync(0xffffffffu, gz_sync_lane(I, T, a, b, r, lane, &c));
			if (m) { found = a + (bz_u64)r * 32 + (bz_u64)(__ffs(m) - 1); break; }
		}
		if (lane == 0) s[i] = found;
	}
}

__global__ void __launch_bounds__(32) k_gz_decode(GzIn I, const int *which, int nw, GzChunk *ch, GzEvent *ev, uint16_t *slots)
{
	__shared__ GzTab T;
	if (threadIdx.x) return;
	for (int w = blockIdx.x; w < nw; w += gridDim.x) {
		const int k = which[w];
		gz_decode(I, T, ch[k], slots + (bz_u64)k * GZ_SLOT, ev + (bz_u64)k * GZ_EVCAP);
	}
}

// the last 32 KB of every chunk, in chunk order: each is context of the chunk after it
__global__ void __launch_bounds__(1024) k_gz_resolve_tails(const uint16_t *slots, int n, const u32 *len, const bz_u64 *off, uint8_t *wout)
{
	for (int k = 0; k < n; ++k) {
		gz_resolve_range(slots + (bz_u64)k * GZ_SLOT, off[k], len[k] > GZ_CTX ? len[k] - GZ_CTX : 0, len[k], wout, threadIdx.x, blockDim.x);
		__syncthreads();
	}
}
__global__ void __launch_bounds__(256) k_gz_resolve_rest(const uint16_t *slots, int n, const u32 *len, const bz_u64 *off, uint8_t *wout)
{
	for (int k = blockIdx.x; k < n; k += gridDim.x)
		gz_resolve_range(slots + (bz_u64)k * GZ_SLOT, off[k], 0, len[k] > GZ_CTX ? len[k] - GZ_CTX : 0, wout, threadIdx.x, blockDim.x);
}
__global__ void __launch_bounds__(256) k_gz_crc(const uint8_t *wout, const bz_u64 *off, const u32 *len, int n, u32 *out)
{
	__shared__ u32 tab[256];
	tab[threadIdx.x] = bz_crc_entry(threadIdx.x);
	__syncthreads();
	for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) out[i] = gz_crc_piece(tab, wout + GZ_CTX + off[i], len[i]);
}

struct DevBackend : GzBackend {
	int sms;
	cudaStream_t st;
	DBuf d_sync, d_ch, d_ev, d_which, d_len, d_off, d_poff, d_plen, d_pcrc, d_slots, d_wout, d_tmp;
	int sync(const GzIn &I, int n, bz_u64 lo, bz_u64 cbits, bz_u64 wend, bz_u64 *s) override
	{
		const int grid = n - 1 < sms * 3 ? n - 1 : sms * 3;
		k_gz_sync<<<grid, 32, 32 * sizeof(GzTab), st>>>(I, n, lo, cbits, wend, d_sync.as<bz_u64>());
		CK(cudaGetLastError());
		CK(cudaMemcpyAsync(s + 1, d_sync.as<bz_u64>() + 1, (size_t)(n - 1) * 8, cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		return 0;
	}
	int decode(const GzIn &I, const std::vector<int> &which, GzChunk *ch, GzEvent *ev) override
	{
		if (which.empty()) return 0;
		const int m = which.back() + 1, nw = (int)which.size();
		CK(cudaMemcpyAsync(d_ch.p, ch, (size_t)m * sizeof(GzChunk), cudaMemcpyHostToDevice, st));
		CK(cudaMemcpyAsync(d_which.p, which.data(), (size_t)nw * sizeof(int), cudaMemcpyHostToDevice, st));
		k_gz_decode<<<nw < sms * 16 ? nw : sms * 16, 32, 0, st>>>(I, d_which.as<int>(), nw, d_ch.as<GzChunk>(), d_ev.as<GzEvent>(), d_slots.as<uint16_t>());
		CK(cudaGetLastError());
		CK(cudaMemcpyAsync(ch, d_ch.p, (size_t)m * sizeof(GzChunk), cudaMemcpyDeviceToHost, st));
		CK(cudaMemcpyAsync(ev, d_ev.p, (size_t)m * GZ_EVCAP * sizeof(GzEvent), cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		return 0;
	}
	int resolve(int n, const u32 *len, const bz_u64 *off) override
	{
		CK(cudaMemcpyAsync(d_len.p, len, (size_t)n * 4, cudaMemcpyHostToDevice, st));
		CK(cudaMemcpyAsync(d_off.p, off, (size_t)n * 8, cudaMemcpyHostToDevice, st));
		k_gz_resolve_tails<<<1, 1024, 0, st>>>(d_slots.as<uint16_t>(), n, d_len.as<u32>(), d_off.as<bz_u64>(), d_wout.as<uint8_t>());
		k_gz_resolve_rest<<<n < sms * 8 ? n : sms * 8, 256, 0, st>>>(d_slots.as<uint16_t>(), n, d_len.as<u32>(), d_off.as<bz_u64>(), d_wout.as<uint8_t>());
		CK(cudaGetLastError());
		return 0;
	}
	int crc(const std::vector<bz_u64> &off, const std::vector<u32> &len, std::vector<u32> &out) override
	{
		const int n = (int)off.size();
		out.resize(n);
		if (!n) return 0;
		int rc;
		if ((rc = d_poff.need((size_t)n * 8)) || (rc = d_plen.need((size_t)n * 4)) || (rc = d_pcrc.need((size_t)n * 4))) return rc;
		CK(cudaMemcpyAsync(d_poff.p, off.data(), (size_t)n * 8, cudaMemcpyHostToDevice, st));
		CK(cudaMemcpyAsync(d_plen.p, len.data(), (size_t)n * 4, cudaMemcpyHostToDevice, st));
		const int blocks = (n + 255) / 256;
		k_gz_crc<<<blocks < sms * 8 ? blocks : sms * 8, 256, 0, st>>>(d_wout.as<uint8_t>(), d_poff.as<bz_u64>(), d_plen.as<u32>(), n, d_pcrc.as<u32>());
		CK(cudaGetLastError());
		CK(cudaMemcpyAsync(out.data(), d_pcrc.p, (size_t)n * 4, cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		return 0;
	}
	// after a window of `text` bytes: its last 32 KB (with the context before it) become the next window's context
	int shift(bz_u64 text)
	{
		CK(cudaMemcpyAsync(d_tmp.p, d_wout.as<uint8_t>() + text, GZ_CTX, cudaMemcpyDeviceToDevice, st));
		CK(cudaMemcpyAsync(d_wout.p, d_tmp.p, GZ_CTX, cudaMemcpyDeviceToDevice, st));
		return 0;
	}
};

struct ssq_gunzip {
	int device;
	size_t chunk, incap;
	DevBackend be;
	DBuf d_in;
	uint8_t *h_in, *h_pend;           // pinned: input staging, text not yet delivered
	size_t pend_cap, pend_len, pend_at;
	GzState S;                        // the stream of ssq_gunzip_inflate
	bz_u64 in_total;                     // compressed bytes of that stream already dropped
	std::vector<GzChunk> ch;
	std::vector<GzEvent> ev;
	int64_t stats[4];
};

extern "C" int ssq_gunzip_create(int device, size_t chunk_bytes, ssq_gunzip_t **out)
{
	if (!out || (chunk_bytes && (chunk_bytes < 256 || chunk_bytes > (4u << 20)))) { ssq_set_error("ssq_gunzip_create: invalid arguments"); return SSQ_EINVAL; }
	*out = 0;
	int rc = ssq_use_device(device);
	if (rc) return rc;
	ssq_gunzip *g = new ssq_gunzip();
	g->device = device; g->h_in = g->h_pend = 0; g->pend_cap = g->pend_len = g->pend_at = 0; g->in_total = 0;
	memset(g->stats, 0, sizeof g->stats);
	gz_state_init(g->S);
	g->chunk = chunk_bytes ? chunk_bytes : GZ_CHUNK_DEFAULT;
	g->incap = g->chunk * GZ_MAXCH + GZ_SLACK;
	g->be.st = 0;
	if (cudaStreamCreateWithFlags(&g->be.st, cudaStreamNonBlocking) != cudaSuccess || cudaDeviceGetAttribute(&g->be.sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess ||
	    cudaFuncSetAttribute(k_gz_sync, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(32 * sizeof(GzTab))) != cudaSuccess) {
		ssq_set_error("ssq_gunzip_create: cannot set up the decoder kernels"); ssq_gunzip_free(g); return SSQ_ECUDA;
	}
	DevBackend &b = g->be;
	if ((rc = b.d_sync.need(GZ_MAXCH * 8)) || (rc = b.d_ch.need(GZ_MAXCH * sizeof(GzChunk))) || (rc = b.d_ev.need((size_t)GZ_MAXCH * GZ_EVCAP * sizeof(GzEvent))) ||
	    (rc = b.d_which.need(GZ_MAXCH * 4)) || (rc = b.d_len.need(GZ_MAXCH * 4)) || (rc = b.d_off.need(GZ_MAXCH * 8)) || (rc = b.d_tmp.need(GZ_CTX)) ||
	    (rc = b.d_slots.need((size_t)GZ_MAXCH * GZ_SLOT * 2)) || (rc = b.d_wout.need(GZ_CTX + (size_t)GZ_MAXCH * GZ_SLOT)) || (rc = g->d_in.need(g->incap))) {
		ssq_gunzip_free(g); return rc;
	}
	if (cudaMemsetAsync(b.d_wout.p, 0, GZ_CTX, b.st) != cudaSuccess || cudaMallocHost((void**)&g->h_in, g->incap) != cudaSuccess) {
		ssq_set_error("ssq_gunzip_create: cudaMallocHost failed"); ssq_gunzip_free(g); return SSQ_ENOMEM;
	}
	*out = g;
	return SSQ_OK;
}

extern "C" void ssq_gunzip_free(ssq_gunzip_t *g)
{
	if (!g) return;
	cudaSetDevice(g->device);
	if (g->be.st) cudaStreamSynchronize(g->be.st);
	if (g->h_in) cudaFreeHost(g->h_in);
	if (g->h_pend) cudaFreeHost(g->h_pend);
	if (g->be.st) cudaStreamDestroy(g->be.st);
	delete g;
}

extern "C" void *ssq_gunzip_stream(ssq_gunzip_t *g) { return g ? (void*)g->be.st : 0; }

extern "C" int ssq_gunzip_stats(const ssq_gunzip_t *g, int64_t out[4])
{
	if (!g || !out) return SSQ_EINVAL;
	memcpy(out, g->stats, sizeof g->stats);
	return SSQ_OK;
}

static void add_stats(ssq_gunzip *g, const int64_t *before, const int64_t *after) { for (int i = 0; i < 4; ++i) g->stats[i] += after[i] - before[i]; }

extern "C" int ssq_gunzip_inflate_dev(ssq_gunzip_t *g, const void *d_in, size_t n, void *d_out, size_t out_cap, size_t *out_len)
{
	if (!g || (!d_in && n) || (!d_out && out_cap) || !out_len) { ssq_set_error("ssq_gunzip_inflate_dev: invalid arguments"); return SSQ_EINVAL; }
	int rc = ssq_use_device(g->device);
	if (rc) return rc;
	GzState S; gz_state_init(S);
	CK(cudaMemsetAsync(g->be.d_wout.p, 0, GZ_CTX, g->be.st));
	bool fits = true;
	auto emit = [&](bz_u64 text) {
		if (S.total > out_cap) fits = false;
		if (fits && text && cudaMemcpyAsync((uint8_t*)d_out + (S.total - text), g->be.d_wout.as<uint8_t>() + GZ_CTX, text, cudaMemcpyDeviceToDevice, g->be.st) != cudaSuccess) {
			ssq_set_error("ssq_gunzip_inflate_dev: copy failed"); return SSQ_ECUDA;
		}
		return g->be.shift(text);
	};
	bz_u64 at = 0;
	const int64_t zero[4] = {0, 0, 0, 0};
	rc = gz_run(g->be, S, (const uint8_t*)d_in, n, g->chunk, emit, &at);
	add_stats(g, zero, S.stats);
	if (rc == SSQ_EDATA) { ssq_set_error("ssq_gunzip_inflate_dev: corrupt or truncated gzip data at compressed byte %llu", (unsigned long long)at); return rc; }
	if (rc) return rc;
	CK(cudaStreamSynchronize(g->be.st));
	*out_len = S.total;
	if (!fits) { ssq_set_error("ssq_gunzip_inflate_dev: %llu bytes of output, room for %zu", (unsigned long long)S.total, out_cap); return SSQ_ECAP; }
	return SSQ_OK;
}

// the next streaming call starts a new stream (after the end of one, or an error)
static void restart(ssq_gunzip *g)
{
	gz_state_init(g->S);
	g->in_total = 0; g->pend_len = g->pend_at = 0;
	cudaMemsetAsync(g->be.d_wout.p, 0, GZ_CTX, g->be.st);
}

static void deliver(ssq_gunzip *g, void *out, size_t out_cap, size_t *out_len)
{
	const size_t k = g->pend_len - g->pend_at < out_cap ? g->pend_len - g->pend_at : out_cap;
	memcpy(out, g->h_pend + g->pend_at, k);
	g->pend_at += k; *out_len = k;
	if (g->pend_at == g->pend_len) g->pend_at = g->pend_len = 0;
}

extern "C" int ssq_gunzip_inflate(ssq_gunzip_t *g, const void *in, size_t n, int final, size_t *used, void *out, size_t out_cap, size_t *out_len, int *done)
{
	if (!g || (!in && n) || (!out && out_cap) || !used || !out_len || !done) { ssq_set_error("ssq_gunzip_inflate: invalid arguments"); return SSQ_EINVAL; }
	*used = 0; *out_len = 0; *done = 0;
	int rc = ssq_use_device(g->device);
	if (rc) return rc;
	if (g->pend_len) { deliver(g, out, out_cap, out_len); *done = g->S.eos && !g->pend_len; if (*done) restart(g); return SSQ_OK; }
	const size_t take = n < g->incap ? n : g->incap;
	const int fin = final && n <= g->incap;
	if (!fin && take < g->incap) return SSQ_OK; // decode full windows only: ask for more input
	memcpy(g->h_in, in, take);
	CK(cudaMemcpyAsync(g->d_in.p, g->h_in, take, cudaMemcpyHostToDevice, g->be.st));
	GzIn I; I.p = g->d_in.as<uint8_t>(); I.n = take; I.final = fin;
	int64_t before[4];
	memcpy(before, g->S.stats, sizeof before);
	const GzPos pos0 = g->S.pos;
	bz_u64 text = 0, at = 0;
	rc = gz_window(g->be, g->S, I, g->chunk, g->ch, g->ev, &text, &at);
	add_stats(g, before, g->S.stats);
	if (!rc && fin && !g->S.eos && !text && g->S.pos.bit == pos0.bit && g->S.pos.mode == pos0.mode) { rc = SSQ_EDATA; at = g->S.pos.bit >> 3; }
	if (rc == SSQ_EDATA) ssq_set_error("ssq_gunzip_inflate: corrupt or truncated gzip data at compressed byte %llu", (unsigned long long)(g->in_total + at));
	if (rc) { restart(g); return rc; }
	if (text <= out_cap) {
		if (text) CK(cudaMemcpyAsync(out, g->be.d_wout.as<uint8_t>() + GZ_CTX, text, cudaMemcpyDeviceToHost, g->be.st));
		*out_len = text;
	} else {
		if (g->pend_cap < text) {
			if (g->h_pend) cudaFreeHost(g->h_pend);
			g->pend_cap = 0;
			if (cudaMallocHost((void**)&g->h_pend, text) != cudaSuccess) { g->h_pend = 0; ssq_set_error("ssq_gunzip_inflate: cudaMallocHost(%llu) failed", (unsigned long long)text); return SSQ_ENOMEM; }
			g->pend_cap = text;
		}
		CK(cudaMemcpyAsync(g->h_pend, g->be.d_wout.as<uint8_t>() + GZ_CTX, text, cudaMemcpyDeviceToHost, g->be.st));
		g->pend_len = text; g->pend_at = 0;
	}
	if ((rc = g->be.shift(text))) return rc;
	CK(cudaStreamSynchronize(g->be.st));
	if (g->pend_len) deliver(g, out, out_cap, out_len);
	const bz_u64 c = gz_consumed(g->S.pos);
	gz_rebase(g->S.pos, c);
	*used = c; g->in_total += c;
	*done = g->S.eos && !g->pend_len;
	if (*done) restart(g);
	return SSQ_OK;
}
