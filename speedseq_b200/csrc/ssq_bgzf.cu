// ssq_bgzf.cu — BGZF compression on the device: the member encoder of ssq_bgzf.cuh as one kernel (one CTA of BZ_NT threads per
// member, payload and tables in shared memory, the grid sized from the SM count), then a gather that compacts the fixed-stride
// output slots into one BGZF stream.  C-ABI: ssq_bgzf_create / ssq_bgzf_deflate / ssq_bgzf_deflate_dev (include/ssq.h).
#include <stdlib.h>
#include <string.h>
#include <vector>
#include <cub/block/block_scan.cuh>
#include "ssq_host.h"
#include "ssq_bgzf.cuh"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { ssq_set_error("%s:%d: %s", __FILE__, __LINE__, cudaGetErrorString(e_)); return SSQ_ECUDA; } } while (0)

static const int BZ_CHUNK = 2048; // members per launch (133 MB of input)
static const unsigned char BZ_EOF[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0, 0x1b, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0};

__global__ void __launch_bounds__(BZ_NT) k_bgzf_members(const uint8_t *in, u64 n, int n_members, int level, u32 *tok, uint8_t *slots, u32 *sizes)
{
	extern __shared__ __align__(16) unsigned char bz_sm[];
	BzSmem &S = *reinterpret_cast<BzSmem*>(bz_sm);
	typedef cub::BlockScan<u32, BZ_NT> Scan;
	__shared__ typename Scan::TempStorage scan_tmp;
	const int t = threadIdx.x;
	for (int m = blockIdx.x; m < n_members; m += gridDim.x) {
		BzJob J;
		J.src = in + (u64)m * BZ_PAYLOAD;
		J.n = (u32)(n - (u64)m * BZ_PAYLOAD < BZ_PAYLOAD ? n - (u64)m * BZ_PAYLOAD : BZ_PAYLOAD);
		J.tok = tok + (u64)blockIdx.x * BZ_PAYLOAD; J.slot = slots + (u64)m * BZ_SLOT; J.size = sizes + m;
		bz_load(S, J, level, t);
		__syncthreads();
		bz_crc(S, t);
		for (u32 base = 0; base < S.n; base += BZ_NT) {
			bz_find(S, base, t);
			__syncthreads();
			bz_insert_parse(S, J, base, t);
			__syncthreads();
		}
		bz_hist(S, J, t);
		__syncthreads();
		bz_rank(S, t);
		__syncthreads();
		if (t == 0) bz_plan(S);
		__syncthreads();
		bz_zero(S, J, t);
		__syncthreads();
		if (t == 0) bz_header(S, J);
		bz_stored_copy(S, J, t);
		bz_u64 run = S.hdr_bits;
		if (S.btype) for (u32 c = 0; c < S.ntok; c += BZ_NT) {
			bz_u64 v;
			const u32 nb = bz_tok_bits(S, J, c + t, &v);
			u32 ex, tot;
			Scan(scan_tmp).ExclusiveSum(nb, ex, tot);
			if (nb) bz_put((bz_u64*)(J.slot + BZ_SLOT_BITS), run + ex, v, nb);
			run += tot;
			__syncthreads();
		}
		if (t == 0) bz_eob(S, J, run);
		__syncthreads();
		if (t == 0) bz_finish(S, J);
		__syncthreads();
	}
}

// member m: slot bytes [6, 6 + size) -> out + off[m]
__global__ void k_bgzf_gather(const uint8_t *slots, const u32 *sizes, const u64 *off, int n_members, uint8_t *out)
{
	for (int m = blockIdx.x; m < n_members; m += gridDim.x) {
		const uint8_t *s = slots + (u64)m * BZ_SLOT + BZ_SLOT_MEMBER;
		uint8_t *d = out + off[m];
		const u32 len = sizes[m];
		for (u32 i = threadIdx.x; i < len; i += blockDim.x) d[i] = s[i];
	}
}

struct ssq_bgzf {
	int device, grid;
	cudaStream_t st;
	DBuf d_in, d_tok, d_slots, d_sizes, d_off, d_out;
	uint8_t *h_in, *h_out; // pinned staging, BZ_CHUNK members each
	std::vector<u32> sizes;
	std::vector<u64> off;
};

extern "C" int ssq_bgzf_create(int device, ssq_bgzf_t **out)
{
	if (!out) return SSQ_EINVAL;
	*out = 0;
	int rc = ssq_use_device(device);
	if (rc) return rc;
	ssq_bgzf *z = new ssq_bgzf();
	z->device = device; z->h_in = z->h_out = 0; z->st = 0;
	int sms = 0, per_sm = 0;
	const size_t smem = sizeof(BzSmem);
	if (cudaStreamCreateWithFlags(&z->st, cudaStreamNonBlocking) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device) != cudaSuccess ||
	    cudaFuncSetAttribute(k_bgzf_members, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess ||
	    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_bgzf_members, BZ_NT, smem) != cudaSuccess || per_sm < 1) {
		ssq_set_error("ssq_bgzf_create: cannot set up the encoder kernel (%zu bytes of shared memory per block)", smem);
		ssq_bgzf_free(z); return SSQ_ECUDA;
	}
	z->grid = sms * per_sm;
	if ((rc = z->d_in.need((size_t)BZ_CHUNK * BZ_PAYLOAD)) || (rc = z->d_tok.need((size_t)z->grid * BZ_PAYLOAD * 4)) || (rc = z->d_slots.need((size_t)BZ_CHUNK * BZ_SLOT)) ||
	    (rc = z->d_sizes.need(BZ_CHUNK * 4)) || (rc = z->d_off.need(BZ_CHUNK * 8)) || (rc = z->d_out.need((size_t)BZ_CHUNK * BZ_SLOT))) { ssq_bgzf_free(z); return rc; }
	if (cudaMallocHost((void**)&z->h_in, (size_t)BZ_CHUNK * BZ_PAYLOAD) != cudaSuccess || cudaMallocHost((void**)&z->h_out, (size_t)BZ_CHUNK * BZ_SLOT) != cudaSuccess) {
		ssq_set_error("ssq_bgzf_create: cudaMallocHost failed"); ssq_bgzf_free(z); return SSQ_ENOMEM;
	}
	z->sizes.resize(BZ_CHUNK); z->off.resize(BZ_CHUNK);
	*out = z;
	return SSQ_OK;
}

extern "C" void ssq_bgzf_free(ssq_bgzf_t *z)
{
	if (!z) return;
	cudaSetDevice(z->device);
	if (z->st) cudaStreamSynchronize(z->st);
	if (z->h_in) cudaFreeHost(z->h_in);
	if (z->h_out) cudaFreeHost(z->h_out);
	if (z->st) cudaStreamDestroy(z->st);
	delete z;
}

extern "C" void *ssq_bgzf_stream(ssq_bgzf_t *z) { return z ? (void*)z->st : 0; }

// one launch: members of d_src[0, n) into the slots; their sizes and offsets (from `at`) on the host; returns the bytes they take
static int encode_chunk(ssq_bgzf *z, const uint8_t *d_src, size_t n, int level, int nm, u64 *bytes)
{
	const int grid = nm < z->grid ? nm : z->grid;
	k_bgzf_members<<<grid, BZ_NT, sizeof(BzSmem), z->st>>>(d_src, n, nm, level, z->d_tok.as<u32>(), z->d_slots.as<uint8_t>(), z->d_sizes.as<u32>());
	CK(cudaGetLastError());
	CK(cudaMemcpyAsync(z->sizes.data(), z->d_sizes.p, (size_t)nm * 4, cudaMemcpyDeviceToHost, z->st));
	CK(cudaStreamSynchronize(z->st));
	u64 s = 0;
	for (int m = 0; m < nm; ++m) { z->off[m] = s; s += z->sizes[m]; }
	*bytes = s;
	return SSQ_OK;
}
static int gather_chunk(ssq_bgzf *z, int nm, uint8_t *d_dst)
{
	CK(cudaMemcpyAsync(z->d_off.p, z->off.data(), (size_t)nm * 8, cudaMemcpyHostToDevice, z->st));
	k_bgzf_gather<<<nm < z->grid * 4 ? nm : z->grid * 4, 256, 0, z->st>>>(z->d_slots.as<uint8_t>(), z->d_sizes.as<u32>(), z->d_off.as<u64>(), nm, d_dst);
	CK(cudaGetLastError());
	return SSQ_OK;
}

extern "C" int ssq_bgzf_deflate_dev(ssq_bgzf_t *z, const void *d_in, size_t n, int level, int with_eof, void *d_out, size_t out_cap, size_t *out_len, size_t *needed)
{
	if (!z || (!d_in && n) || (!d_out && out_cap) || !out_len || level < -1 || level > 9) { ssq_set_error("ssq_bgzf_deflate_dev: invalid arguments"); return SSQ_EINVAL; }
	int rc = ssq_use_device(z->device);
	if (rc) return rc;
	const size_t n_blk = (n + BZ_PAYLOAD - 1) / BZ_PAYLOAD;
	u64 at = 0;
	for (size_t b = 0; b < n_blk; b += BZ_CHUNK) {
		const int nm = (int)(n_blk - b < (size_t)BZ_CHUNK ? n_blk - b : BZ_CHUNK);
		const size_t lo = b * BZ_PAYLOAD, len = n - lo < (size_t)nm * BZ_PAYLOAD ? n - lo : (size_t)nm * BZ_PAYLOAD;
		u64 bytes;
		if ((rc = encode_chunk(z, (const uint8_t*)d_in + lo, len, level, nm, &bytes))) return rc;
		if (at + bytes <= out_cap && (rc = gather_chunk(z, nm, (uint8_t*)d_out + at))) return rc;
		at += bytes;
	}
	const u64 total = at + (with_eof ? 28 : 0);
	if (needed) *needed = total;
	*out_len = total;
	if (total > out_cap) { ssq_set_error("ssq_bgzf_deflate_dev: %llu bytes of output, room for %zu", (unsigned long long)total, out_cap); return SSQ_ECAP; }
	if (with_eof) CK(cudaMemcpyAsync((uint8_t*)d_out + at, BZ_EOF, 28, cudaMemcpyHostToDevice, z->st));
	CK(cudaStreamSynchronize(z->st));
	return SSQ_OK;
}

extern "C" int ssq_bgzf_deflate(ssq_bgzf_t *z, const void *in, size_t n, int level, int with_eof, void **out, size_t *out_len)
{
	if (!z || (!in && n) || !out || !out_len || level < -1 || level > 9) { ssq_set_error("ssq_bgzf_deflate: invalid arguments"); return SSQ_EINVAL; }
	int rc = ssq_use_device(z->device);
	if (rc) return rc;
	const size_t n_blk = (n + BZ_PAYLOAD - 1) / BZ_PAYLOAD;
	uint8_t *o = (uint8_t*)malloc(n + 31 * n_blk + 28 + 1); // a member never exceeds its stored form: payload + 31 bytes
	if (!o) { ssq_set_error("ssq_bgzf_deflate: out of memory"); return SSQ_ENOMEM; }
	cudaPointerAttributes pa;
	const bool pinned = n && cudaPointerGetAttributes(&pa, in) == cudaSuccess && pa.type == cudaMemoryTypeHost;
	cudaGetLastError();
	u64 at = 0;
	for (size_t b = 0; b < n_blk; b += BZ_CHUNK) {
		const int nm = (int)(n_blk - b < (size_t)BZ_CHUNK ? n_blk - b : BZ_CHUNK);
		const size_t lo = b * BZ_PAYLOAD, len = n - lo < (size_t)nm * BZ_PAYLOAD ? n - lo : (size_t)nm * BZ_PAYLOAD;
		const uint8_t *src = (const uint8_t*)in + lo;
		if (!pinned) { memcpy(z->h_in, src, len); src = z->h_in; }
		u64 bytes;
		if (cudaMemcpyAsync(z->d_in.p, src, len, cudaMemcpyHostToDevice, z->st) != cudaSuccess) { free(o); ssq_set_error("ssq_bgzf_deflate: copy to the device failed"); return SSQ_ECUDA; }
		if ((rc = encode_chunk(z, z->d_in.as<uint8_t>(), len, level, nm, &bytes)) || (rc = gather_chunk(z, nm, z->d_out.as<uint8_t>()))) { free(o); return rc; }
		if (cudaMemcpyAsync(z->h_out, z->d_out.p, bytes, cudaMemcpyDeviceToHost, z->st) != cudaSuccess || cudaStreamSynchronize(z->st) != cudaSuccess) {
			free(o); ssq_set_error("ssq_bgzf_deflate: %s", cudaGetErrorString(cudaGetLastError())); return SSQ_ECUDA;
		}
		memcpy(o + at, z->h_out, bytes);
		at += bytes;
	}
	if (with_eof) { memcpy(o + at, BZ_EOF, 28); at += 28; }
	*out = o; *out_len = at;
	return SSQ_OK;
}
