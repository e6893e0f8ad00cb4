// ssq_index.cu — index loader (PREFIX.{bwt,sa,pac,ann,amb} -> HBM), options, error plumbing.
// Replaces upstream bwa_idx_load() / mem_opt_init() (start of `$BWA mem`, speedseq/bin/speedseq:438).
// On-disk format: the one of the reference's goldens speedseq/example/data/*.fasta.{amb,ann,pac,bwt,sa}
// (SURVEY.md §8c).  Host memory is only a staging area; nothing here computes on the CPU.
#include <cuda_runtime.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <math.h>
#include "ssq_host.h"

static __thread char g_err[512] = "";
void ssq_set_error(const char *fmt, ...)
{
	va_list ap;
	va_start(ap, fmt);
	vsnprintf(g_err, sizeof g_err, fmt, ap);
	va_end(ap);
}
extern "C" const char *ssq_last_error(void) { return g_err; }

extern "C" int ssq_device_count(void)
{
	int n = 0;
	if (cudaGetDeviceCount(&n) != cudaSuccess) return 0;
	return n;
}

int ssq_use_device(int device)
{
	int n = 0;
	if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) { ssq_set_error("no CUDA device is visible: libssq has no CPU path"); return SSQ_ENOGPU; }
	if (device < 0 || device >= n) { ssq_set_error("device %d out of range (%d visible)", device, n); return SSQ_ENOGPU; }
	if (cudaSetDevice(device) != cudaSuccess) { ssq_set_error("cudaSetDevice(%d) failed", device); return SSQ_ENOGPU; }
	int major = 0, minor = 0;
	cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, device);
	cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, device);
	if (major != 9 || minor != 0) { ssq_set_error("device %d has compute capability %d.%d; this library is built for sm_90a (H100) only", device, major, minor); return SSQ_ENOGPU; }
	return SSQ_OK;
}

extern "C" void ssq_opts_default(ssq_opts_t *o)
{
	memset(o, 0, sizeof *o);
	o->a = 1; o->b = 4; o->o_del = o->o_ins = 6; o->e_del = o->e_ins = 1;
	o->pen_unpaired = 17; o->pen_clip5 = o->pen_clip3 = 5; o->w = 100; o->zdrop = 100; o->T = 30;
	o->min_seed_len = 19; o->split_width = 10; o->max_occ = 500; o->max_chain_gap = 10000; o->max_mem_intv = 20;
	o->min_chain_weight = 0; o->max_chain_extend = 1 << 30; o->max_ins = 10000; o->max_matesw = 50; o->max_XA_hits = 5;
	o->split_factor = 1.5f; o->mask_level = 0.50f; o->drop_ratio = 0.50f; o->XA_drop_ratio = 0.80f; o->mask_level_redun = 0.95f;
	o->mapQ_coef_len = 50; o->mapQ_coef_fac = (int)log(50.0);
	o->n_threads = 1;
}

// re-block the on-disk rank structure (64 B per 128 symbols, u64 counts) into 32 B per 64 symbols with u32 counts
__global__ void k_reblock32(const u32 *__restrict__ bwt, u64 n_sym, u64 n_blk32, u32 *out)
{
	const u64 b = (u64)blockIdx.x * blockDim.x + threadIdx.x;
	if (b >= n_blk32) return;
	const u32 *src = bwt + ((b >> 1) << 4);
	const u64 *c64 = (const u64*)src;
	u32 add[4] = {0, 0, 0, 0};
	if (b & 1) {
#pragma unroll
		for (int w = 0; w < 4; ++w) {
			const u32 v = src[8 + w], lo = v & 0x55555555u, hi = (v >> 1) & 0x55555555u;
			add[0] += __popc(~hi & ~lo & 0x55555555u); add[1] += __popc(~hi & lo); add[2] += __popc(hi & ~lo); add[3] += __popc(hi & lo);
		}
	}
	uint4 cnt, sym;
	cnt.x = (u32)(c64[0] + add[0]); cnt.y = (u32)(c64[1] + add[1]); cnt.z = (u32)(c64[2] + add[2]); cnt.w = (u32)(c64[3] + add[3]);
	const u64 first = ((b >> 1) << 7) + (b & 1) * 64; // first symbol of this block
	sym.x = first < n_sym ? src[8 + (b & 1) * 4] : 0; sym.y = first + 16 < n_sym ? src[9 + (b & 1) * 4] : 0;
	sym.z = first + 32 < n_sym ? src[10 + (b & 1) * 4] : 0; sym.w = first + 48 < n_sym ? src[11 + (b & 1) * 4] : 0;
	((uint4*)out)[b * 2] = cnt; ((uint4*)out)[b * 2 + 1] = sym;
}

static void *read_file(const char *fn, size_t skip, size_t *len)
{
	FILE *fp = fopen(fn, "rb");
	if (!fp) return 0;
	fseek(fp, 0, SEEK_END);
	long sz = ftell(fp);
	if (sz < (long)skip) { fclose(fp); return 0; }
	fseek(fp, (long)skip, SEEK_SET);
	*len = (size_t)sz - skip;
	void *p = 0;
	if (cudaMallocHost(&p, *len + 64) != cudaSuccess) { fclose(fp); return 0; } // pinned staging for the upload
	if (fread(p, 1, *len, fp) != *len) { cudaFreeHost(p); p = 0; }
	fclose(fp);
	return p;
}

#define CKI(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { ssq_set_error("%s:%d: %s", __FILE__, __LINE__, cudaGetErrorString(e_)); ssq_index_free(idx); return SSQ_ECUDA; } } while (0)

// Denser SA sample: row j*d gets the position the LF walk from it reaches on the on-disk sample (row 0 = -1, like sa[0]).
template <class T>
__global__ void k_sa_densify(DevIndex ix, int d, u64 n_dense, T *out)
{
	const u64 j = (u64)blockIdx.x * blockDim.x + threadIdx.x;
	if (j >= n_dense) return;
	ScalarFm fm(ix);
	unsigned long long n_sa = 0;
	const u64 v = sa_lookup(fm, j * (u64)d, n_sa, false);
	out[j] = (T)v; // -1 truncates to the all-ones sentinel
}

// k-mer jump-start table (opt-in): entry e = (L, code) with kmer_off(L) <= e < kmer_off(L + 1)
__global__ void k_kmer_build(DevIndex ix, int K, u32 n_entries, KmerEnt *out)
{
	const u32 e = blockIdx.x * blockDim.x + threadIdx.x;
	if (e >= n_entries) return;
	int L = 1;
	while (L < K && kmer_off(L + 1) <= e) ++L;
	ScalarFm fm(ix);
	out[e] = kmer_compute(fm, ix, L, e - kmer_off(L));
}

extern "C" int ssq_index_load(const char *prefix, int device, ssq_index_t **out)
{
	if (!prefix || !out) return SSQ_EINVAL;
	int rc = ssq_use_device(device);
	if (rc) return rc;
	ssq_index *idx = (ssq_index*)calloc(1, sizeof(ssq_index));
	idx->device = device;
	char fn[4096];
	size_t len;
	// .bwt : u64 primary, u64 L2[1..4], then occ-interleaved words
	snprintf(fn, sizeof fn, "%s.bwt", prefix);
	uint8_t *h = (uint8_t*)read_file(fn, 0, &len);
	if (!h || len < 40 + 64) { ssq_set_error("cannot read %s", fn); if (h) cudaFreeHost(h); ssq_index_free(idx); return SSQ_EIO; }
	u64 hdr[5];
	memcpy(hdr, h, 40);
	idx->dev.primary = hdr[0];
	idx->dev.L2[0] = 0; memcpy(&idx->dev.L2[1], hdr + 1, 32);
	idx->dev.seq_len = idx->dev.L2[4];
	{
		const size_t bytes = len - 40;
		const u64 n_blocks = (idx->dev.seq_len + 127) / 128 + 1; // last block: counts only
		if (bytes < (idx->dev.seq_len + 15) / 16 * 4 + n_blocks * 32) { ssq_set_error("%s is truncated", fn); cudaFreeHost(h); ssq_index_free(idx); return SSQ_EIO; }
		void *d = 0;
		const size_t padded = ((bytes + 63) / 64 + 1) * 64; // every block readable as a full 64-B line
		CKI(cudaMalloc(&d, padded));
		CKI(cudaMemset(d, 0, padded));
		CKI(cudaMemcpy(d, h + 40, bytes, cudaMemcpyHostToDevice));
		idx->dev.bwt = (const u32*)d; idx->dev_bytes += padded;
		if (idx->dev.seq_len < 0xffffffffull && !getenv("SSQ_NO_BWT32")) {
			const u64 nb = (idx->dev.seq_len + 63) / 64 + 1;
			void *d32 = 0;
			CKI(cudaMalloc(&d32, nb * 32 + 64));
			CKI(cudaMemset(d32, 0, nb * 32 + 64));
			k_reblock32<<<(unsigned)((nb + 255) / 256), 256>>>((const u32*)d, idx->dev.seq_len, nb, (u32*)d32);
			CKI(cudaGetLastError());
			CKI(cudaDeviceSynchronize());
			idx->dev.bwt32 = (const u32*)d32; idx->dev_bytes += nb * 32 + 64;
		}
	}
	cudaFreeHost(h);
	// .sa : u64 primary, L2[1..4], sa_intv, seq_len, then SA[32k] k>=1
	snprintf(fn, sizeof fn, "%s.sa", prefix);
	h = (uint8_t*)read_file(fn, 0, &len);
	if (!h || len < 56) { ssq_set_error("cannot read %s", fn); if (h) cudaFreeHost(h); ssq_index_free(idx); return SSQ_EIO; }
	{
		u64 sh[7];
		memcpy(sh, h, 56);
		if (sh[0] != idx->dev.primary || sh[6] != idx->dev.seq_len || (sh[5] & (sh[5] - 1)) != 0) { ssq_set_error("%s does not match the .bwt", fn); cudaFreeHost(h); ssq_index_free(idx); return SSQ_EIO; }
		idx->dev.sa_intv = (i32)sh[5];
		idx->dev.n_sa = (idx->dev.seq_len + sh[5]) / sh[5];
		if (len - 56 < (idx->dev.n_sa - 1) * 8) { ssq_set_error("%s is truncated", fn); cudaFreeHost(h); ssq_index_free(idx); return SSQ_EIO; }
		void *d = 0;
		const u64 minus1 = (u64)-1;
		CKI(cudaMalloc(&d, idx->dev.n_sa * 8));
		CKI(cudaMemcpy(d, &minus1, 8, cudaMemcpyHostToDevice));
		CKI(cudaMemcpy((u64*)d + 1, h + 56, (idx->dev.n_sa - 1) * 8, cudaMemcpyHostToDevice));
		idx->dev.sa = (const u64*)d; idx->dev_bytes += idx->dev.n_sa * 8;
	}
	cudaFreeHost(h);
	{ // denser sample: a 4x shorter LF walk per seed occurrence for little HBM (GRCh37: 6.2 G rows / 8 x 8 B = 6.2 GB of the H100's 80 GB)
		const int d = getenv("SSQ_SA_DENSE") ? atoi(getenv("SSQ_SA_DENSE")) : 8;
		if (d > 0 && d < idx->dev.sa_intv && (d & (d - 1)) == 0) {
			const u64 nd = idx->dev.seq_len / d + 1;
			const bool small = idx->dev.seq_len < 0xffffffffull && !getenv("SSQ_SA_U64"); // SSQ_SA_U64: tests force the u64 sample of >= 2^32-row indexes
			void *dd = 0;
			CKI(cudaMalloc(&dd, nd * (small ? 4 : 8)));
			if (small) k_sa_densify<u32><<<(unsigned)((nd + 255) / 256), 256>>>(idx->dev, d, nd, (u32*)dd);
			else k_sa_densify<u64><<<(unsigned)((nd + 255) / 256), 256>>>(idx->dev, d, nd, (u64*)dd);
			CKI(cudaGetLastError());
			CKI(cudaDeviceSynchronize());
			if (small) idx->dev.sad32 = (const u32*)dd; else idx->dev.sad64 = (const u64*)dd;
			idx->dev.sad_intv = d; idx->dev_bytes += nd * (small ? 4 : 8);
		}
	}
	{ // k-mer jump-start table for the seeding kernels: K = SSQ_KMER_K (1..12; 0 = no table), else SSQ_KMER_K_DEFAULT (see ssq_dev.cuh)
		const int K = getenv("SSQ_KMER_K") ? atoi(getenv("SSQ_KMER_K")) : SSQ_KMER_K_DEFAULT;
		if (K >= 1 && K <= 12 && idx->dev.bwt32) {
			const u32 ne = kmer_entries(K);
			void *dk = 0;
			CKI(cudaMalloc(&dk, (size_t)ne * sizeof(KmerEnt)));
			k_kmer_build<<<(ne + 255) / 256, 256>>>(idx->dev, K, ne, (KmerEnt*)dk);
			CKI(cudaGetLastError());
			CKI(cudaDeviceSynchronize());
			idx->dev.kmer = (const KmerEnt*)dk; idx->dev.kmer_k = K; idx->dev_bytes += (size_t)ne * sizeof(KmerEnt);
		}
	}
	// .ann
	snprintf(fn, sizeof fn, "%s.ann", prefix);
	{
		FILE *fp = fopen(fn, "r");
		long long ll; int ns; unsigned seed;
		char str[8192];
		if (!fp || fscanf(fp, "%lld%d%u", &ll, &ns, &seed) != 3 || ns <= 0) { ssq_set_error("cannot read %s", fn); if (fp) fclose(fp); ssq_index_free(idx); return SSQ_EIO; }
		idx->dev.l_pac = ll; idx->dev.n_seqs = ns; idx->n_seqs = ns;
		idx->names = (char**)calloc(ns, sizeof(char*));
		idx->ann_off = (i64*)calloc(ns, sizeof(i64));
		idx->ann_len = (i32*)calloc(ns, sizeof(i32));
		for (int i = 0; i < ns; ++i) {
			unsigned gi; int c, nambs;
			if (fscanf(fp, "%u%8191s", &gi, str) != 2) { ssq_set_error("malformed %s", fn); fclose(fp); ssq_index_free(idx); return SSQ_EIO; }
			idx->names[i] = strdup(str);
			while ((c = fgetc(fp)) != '\n' && c != EOF);
			if (fscanf(fp, "%lld%d%d", &ll, &idx->ann_len[i], &nambs) != 3) { ssq_set_error("malformed %s", fn); fclose(fp); ssq_index_free(idx); return SSQ_EIO; }
			idx->ann_off[i] = ll;
		}
		fclose(fp);
		if ((u64)idx->dev.l_pac * 2 != idx->dev.seq_len) { ssq_set_error("%s: l_pac does not match the BWT length", fn); ssq_index_free(idx); return SSQ_EIO; }
		void *d1 = 0, *d2 = 0;
		CKI(cudaMalloc(&d1, ns * sizeof(i64))); CKI(cudaMalloc(&d2, ns * sizeof(i32)));
		CKI(cudaMemcpy(d1, idx->ann_off, ns * sizeof(i64), cudaMemcpyHostToDevice));
		CKI(cudaMemcpy(d2, idx->ann_len, ns * sizeof(i32), cudaMemcpyHostToDevice));
		idx->dev.ann_off = (const i64*)d1; idx->dev.ann_len = (const i32*)d2;
	}
	// .pac
	snprintf(fn, sizeof fn, "%s.pac", prefix);
	h = (uint8_t*)read_file(fn, 0, &len);
	if (!h || (i64)len < idx->dev.l_pac / 4 + 1) { ssq_set_error("cannot read %s", fn); if (h) cudaFreeHost(h); ssq_index_free(idx); return SSQ_EIO; }
	{
		void *d = 0;
		CKI(cudaMalloc(&d, len + 64));
		CKI(cudaMemset(d, 0, len + 64));
		CKI(cudaMemcpy(d, h, len, cudaMemcpyHostToDevice));
		idx->dev.pac = (const uint8_t*)d; idx->dev_bytes += len + 64;
	}
	cudaFreeHost(h);
	*out = idx;
	return SSQ_OK;
}

extern "C" void ssq_index_free(ssq_index_t *idx)
{
	if (!idx) return;
	cudaFree((void*)idx->dev.bwt); cudaFree((void*)idx->dev.bwt32); cudaFree((void*)idx->dev.sa); cudaFree((void*)idx->dev.pac); cudaFree((void*)idx->dev.sad32); cudaFree((void*)idx->dev.sad64); cudaFree((void*)idx->dev.kmer);
	cudaFree((void*)idx->dev.ann_off); cudaFree((void*)idx->dev.ann_len);
	for (int i = 0; i < idx->n_seqs && idx->names; ++i) free(idx->names[i]);
	free(idx->names); free(idx->ann_off); free(idx->ann_len);
	free(idx);
}

extern "C" uint64_t ssq_index_info(const ssq_index_t *idx, int what)
{
	switch (what) {
	case 0: return (uint64_t)idx->dev.l_pac;
	case 1: return idx->dev.seq_len;
	case 2: return idx->dev.primary;
	case 3: return (uint64_t)idx->dev.n_seqs;
	case 4: return ((idx->dev.seq_len + 15) / 16) + ((idx->dev.seq_len + 127) / 128 + 1) * 8;
	case 5: return idx->dev.n_sa;
	case 6: return (uint64_t)idx->dev_bytes;
	case 7: return idx->dev.bwt32 ? 32 : 64; // bytes fetched per rank query (one re-blocked sector, or one on-disk block)
	case 8: return idx->dev.sad32 ? 4 : 8;   // bytes per suffix-array sample read
	case 9: return (uint64_t)(idx->dev.sad_intv ? idx->dev.sad_intv : idx->dev.sa_intv); // rows between the samples the LF walk ends on
	}
	return 0;
}

extern "C" const char *ssq_index_contig(const ssq_index_t *idx, int i, int64_t *len)
{
	if (!idx || i < 0 || i >= idx->n_seqs) return 0;
	if (len) *len = idx->ann_len[i];
	return idx->names[i];
}
