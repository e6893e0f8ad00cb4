// ssq_sbtext.cu — samblaster over name-grouped SAM text on the device: the routines of ssq_sbtext.cuh as kernels.  Per call:
//   lines   a select of the '\n' positions (a flag per byte); a last line without '\n' counts when final
//   fields  a thread per line: tab offsets, FLAG, POS, CIGAR ops, RNAME looked up in the @SQ hash table, MC:Z / MQ:i present;
//           a thread per line marks the lines whose QNAME differs from the line before, a select gives the block starts
//   blocks  a thread per block: primary lines, signature, discordant / splitter marks, MC / MQ mate line; the lines and blocks the
//           device does not take come back as the smallest (line << 8 | reason) before anything is marked
//   dups    ssq_dupset_mark_dev against the object's set, in block order
//   text    a thread per line sizes its bytes in the three streams, three exclusive scans, a thread per line writes them, and the
//           three texts are copied into pinned buffers of the object
// C-ABI: ssq_sbtext_create / ssq_sbtext_run / ssq_sbtext_dupset / ssq_sbtext_stream / ssq_sbtext_free (include/ssq.h).
#include <stdlib.h>
#include <string.h>
#include <cub/cub.cuh>
#include "ssq_host.h"
#include "ssq_sbtext.cuh"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { ssq_set_error("%s:%d: %s", __FILE__, __LINE__, cudaGetErrorString(e_)); return SSQ_ECUDA; } } while (0)
#define SBT_NT 256

struct SbtIsNl { const char *t; __host__ __device__ __forceinline__ bool operator()(const u32 &i) const { return t[i] == '\n'; } };

__global__ void __launch_bounds__(SBT_NT) k_sbt_fields(const char *t, const u32 *nl, u32 n_nl, u32 n_lines, u32 len, const SbtCtg C, u32 *ops, SbtLine *L)
{
	const u32 i = blockIdx.x * SBT_NT + threadIdx.x;
	if (i >= n_lines) return;
	sbt_parse_line(t, i ? nl[i - 1] + 1 : 0, i < n_nl ? nl[i] : len, C, ops, L[i]);
}
__global__ void __launch_bounds__(SBT_NT) k_sbt_starts(const char *t, const SbtLine *L, u32 n_lines, uint8_t *flag)
{
	const u32 i = blockIdx.x * SBT_NT + threadIdx.x;
	if (i < n_lines) flag[i] = sbt_block_start(t, L, i) ? 1 : 0;
}
__global__ void __launch_bounds__(SBT_NT) k_sbt_blocks(const SbOpts o, const i64 *sb_off, const u32 *ops, SbtLine *L, const u32 *bstart, u32 n_blocks, u32 n_lines, u32 take,
                                                       u64 *k1, u64 *k2, uint8_t *valid, unsigned long long *first_err)
{
	const u32 b = blockIdx.x * SBT_NT + threadIdx.x;
	if (b >= take) return;
	const u32 b0 = bstart[b], b1 = b + 1 < n_blocks ? bstart[b + 1] : n_lines;
	const int e = sbt_block(o, sb_off, ops, L, b0, b1, b, k1 + b, k2 + b, valid + b);
	if (e) atomicMin(first_err, (unsigned long long)b0 << 8 | (unsigned)e);
}
__global__ void __launch_bounds__(SBT_NT) k_sbt_err(const SbtLine *L, u32 lines, unsigned long long *first_err)
{
	const u32 i = blockIdx.x * SBT_NT + threadIdx.x;
	if (i < lines && L[i].err) atomicMin(first_err, (unsigned long long)i << 8 | L[i].err);
}
// W = false: byte counts of line i in the three streams, and the counters; W = true: its bytes at the scanned offsets
template <bool W>
__global__ void __launch_bounds__(SBT_NT) k_sbt_text(const SbOpts o, const char *t, const SbtLine *L, const u32 *bstart, u32 lines, const uint8_t *dup, u64 *len0, u64 *len1, u64 *len2,
                                                     char *o0, char *o1, char *o2, unsigned long long *cnt)
{
	const u32 i = blockIdx.x * SBT_NT + threadIdx.x;
	if (i >= lines) return;
	u64 *len[3] = {len0, len1, len2};
	char *out[3] = {o0, o1, o2};
	const u32 blk = L[i].blk;
	const bool d = dup[blk] != 0;
	Sink<W> s[3];
	for (int k = 0; k < 3; ++k) { s[k].p = W ? out[k] + len[k][i] : 0; s[k].n = 0; }
	sbt_line_text(o, t, L, i, d, s);
	if (!W) {
		for (int k = 0; k < 3; ++k) len[k][i] = s[k].n;
		if (d && bstart[blk] == i) atomicAdd(cnt, 1ull);
		if (s[1].n) atomicAdd(cnt + 1, 1ull);
		if (s[2].n) atomicAdd(cnt + 2, 1ull);
	}
}

struct ssq_sbtext {
	int device;
	cudaStream_t st;
	SbOpts o;
	SbtHeader H;
	SbtCtg C;
	ssq_dupset_t *set;
	DBuf d_names, d_name_off, d_slot, d_off;
	DBuf text, nl, ops, lines, flag, bstart, nsel, k1, k2, valid, dup, err, cnt, len[3], out[3], tmp;
	char *h_out[3]; size_t h_cap[3];
};

static unsigned grid_of(u64 n) { return (unsigned)((n + SBT_NT - 1) / SBT_NT); }

extern "C" int ssq_sbtext_create(int device, const ssq_sb_opts_t *sb, const char *header, size_t header_len, ssq_sbtext_t **out)
{
	if (!sb || !out || (!header && header_len)) return SSQ_EINVAL;
	int rc = ssq_use_device(device);
	if (rc) return rc;
	ssq_sbtext *s = new ssq_sbtext();
	s->device = device; s->o = sbt_opts(*sb); s->set = 0;
	for (int k = 0; k < 3; ++k) { s->h_out[k] = 0; s->h_cap[k] = 0; }
	sbt_parse_header(header ? header : "", header_len, s->H);
	const SbtHeader &H = s->H;
	if (cudaStreamCreateWithFlags(&s->st, cudaStreamNonBlocking) != cudaSuccess) { delete s; ssq_set_error("cudaStreamCreate failed"); return SSQ_ECUDA; }
	if (s->d_names.need(H.names.size()) || s->d_name_off.need(H.name_off.size() * 4) || s->d_slot.need(H.slot.size() * 4) || s->d_off.need(H.off.size() * 8) ||
	    (rc = ssq_dupset_create(device, &s->set))) { rc = rc ? rc : SSQ_ENOMEM; ssq_sbtext_free(s); return rc; }
	if (cudaMemcpy(s->d_names.p, H.names.data(), H.names.size(), cudaMemcpyHostToDevice) != cudaSuccess ||
	    cudaMemcpy(s->d_name_off.p, H.name_off.data(), H.name_off.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess ||
	    cudaMemcpy(s->d_slot.p, H.slot.data(), H.slot.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess ||
	    cudaMemcpy(s->d_off.p, H.off.data(), H.off.size() * 8, cudaMemcpyHostToDevice) != cudaSuccess) { ssq_set_error("ssq_sbtext_create: copy of the @SQ table failed"); ssq_sbtext_free(s); return SSQ_ECUDA; }
	s->C.names = s->d_names.as<char>(); s->C.name_off = s->d_name_off.as<u32>(); s->C.slot = s->d_slot.as<i32>(); s->C.mask = H.mask;
	*out = s;
	return SSQ_OK;
}

extern "C" ssq_dupset_t *ssq_sbtext_dupset(ssq_sbtext_t *s) { return s ? s->set : 0; }
extern "C" void *ssq_sbtext_stream(ssq_sbtext_t *s) { return s ? (void*)s->st : 0; }
extern "C" void ssq_sbtext_free(ssq_sbtext_t *s)
{
	if (!s) return;
	if (s->st) cudaStreamSynchronize(s->st);
	for (int k = 0; k < 3; ++k) if (s->h_out[k]) cudaFreeHost(s->h_out[k]);
	if (s->set) ssq_dupset_free(s->set);
	if (s->st) cudaStreamDestroy(s->st);
	delete s;
}

extern "C" int ssq_sbtext_run(ssq_sbtext_t *s, const char *text, size_t len, int final, uint64_t max_blocks, size_t *used, ssq_sbtext_out_t *out)
{
	if (!s || !used || !out || (!text && len)) return SSQ_EINVAL;
	*used = 0;
	memset(out, 0, sizeof *out);
	if (len >= 0x7fffffffull) { ssq_set_error("ssq_sbtext_run: %zu bytes in one call (at most 2^31 - 2)", len); return SSQ_EINVAL; }
	int rc = ssq_use_device(s->device);
	if (rc) return rc;
	if (!len) return SSQ_OK;
	cudaStream_t st = s->st;
	// lines
	if (s->text.need(len) || s->nl.need(len * 4) || s->nsel.need(8)) return SSQ_ENOMEM;
	CK(cudaMemcpyAsync(s->text.p, text, len, cudaMemcpyHostToDevice, st));
	const char *t = s->text.as<char>();
	size_t tb = 0;
	cub::CountingInputIterator<u32> iota(0);
	const SbtIsNl is_nl = {t};
	CK(cub::DeviceSelect::If(0, tb, iota, s->nl.as<u32>(), s->nsel.as<int>(), (int)len, is_nl, st));
	if (s->tmp.need(tb)) return SSQ_ENOMEM;
	CK(cub::DeviceSelect::If(s->tmp.p, tb, iota, s->nl.as<u32>(), s->nsel.as<int>(), (int)len, is_nl, st));
	int n_nl = 0;
	u32 last_nl = 0;
	CK(cudaMemcpyAsync(&n_nl, s->nsel.p, sizeof n_nl, cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	if (n_nl) { CK(cudaMemcpyAsync(&last_nl, s->nl.as<u32>() + n_nl - 1, 4, cudaMemcpyDeviceToHost, st)); CK(cudaStreamSynchronize(st)); }
	const u32 n_lines = (u32)n_nl + (final && (n_nl ? last_nl + 1 < len : true) ? 1 : 0);
	if (!n_lines) return SSQ_OK;
	// fields, block starts
	if (s->ops.need((len / 2 + 1) * 4) || s->lines.need((size_t)n_lines * sizeof(SbtLine)) || s->flag.need(n_lines) || s->bstart.need((size_t)n_lines * 4)) return SSQ_ENOMEM;
	SbtLine *L = s->lines.as<SbtLine>();
	k_sbt_fields<<<grid_of(n_lines), SBT_NT, 0, st>>>(t, s->nl.as<u32>(), (u32)n_nl, n_lines, (u32)len, s->C, s->ops.as<u32>(), L);
	k_sbt_starts<<<grid_of(n_lines), SBT_NT, 0, st>>>(t, L, n_lines, s->flag.as<uint8_t>());
	CK(cudaGetLastError());
	CK(cub::DeviceSelect::Flagged(0, tb, iota, s->flag.as<uint8_t>(), s->bstart.as<u32>(), s->nsel.as<int>(), (int)n_lines, st));
	if (s->tmp.need(tb)) return SSQ_ENOMEM;
	CK(cub::DeviceSelect::Flagged(s->tmp.p, tb, iota, s->flag.as<uint8_t>(), s->bstart.as<u32>(), s->nsel.as<int>(), (int)n_lines, st));
	int n_blocks = 0;
	CK(cudaMemcpyAsync(&n_blocks, s->nsel.p, sizeof n_blocks, cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	const u64 take = sbt_take((u64)n_blocks, final, max_blocks);
	u32 lines = n_lines, next_beg = 0;
	if (take < (u64)n_blocks) {
		CK(cudaMemcpyAsync(&lines, s->bstart.as<u32>() + take, 4, cudaMemcpyDeviceToHost, st));
		CK(cudaStreamSynchronize(st));
		if (lines) { CK(cudaMemcpyAsync(&next_beg, s->nl.as<u32>() + lines - 1, 4, cudaMemcpyDeviceToHost, st)); CK(cudaStreamSynchronize(st)); ++next_beg; }
	}
	const size_t consumed = take < (u64)n_blocks ? next_beg : (final ? len : 0);
	if (!take) { *used = consumed; return SSQ_OK; }
	// blocks; the first line the device does not take
	if (s->k1.need(take * 8) || s->k2.need(take * 8) || s->valid.need(take) || s->dup.need(take) || s->err.need(8) || s->cnt.need(3 * 8)) return SSQ_ENOMEM;
	CK(cudaMemsetAsync(s->err.p, 0xff, 8, st));
	k_sbt_blocks<<<grid_of(take), SBT_NT, 0, st>>>(s->o, s->d_off.as<i64>(), s->ops.as<u32>(), L, s->bstart.as<u32>(), (u32)n_blocks, n_lines, (u32)take,
	                                                s->k1.as<u64>(), s->k2.as<u64>(), s->valid.as<uint8_t>(), s->err.as<unsigned long long>());
	k_sbt_err<<<grid_of(lines), SBT_NT, 0, st>>>(L, lines, s->err.as<unsigned long long>());
	CK(cudaGetLastError());
	unsigned long long first_err = 0;
	CK(cudaMemcpyAsync(&first_err, s->err.p, 8, cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	if (first_err != ~0ull) {
		const u32 line = (u32)(first_err >> 8);
		u32 beg = 0;
		if (line) { CK(cudaMemcpy(&beg, s->nl.as<u32>() + line - 1, 4, cudaMemcpyDeviceToHost)); ++beg; }
		char msg[512];
		sbt_refusal(msg, sizeof msg, line, beg, (int)(first_err & 0xff), text, len);
		ssq_set_error("%s", msg);
		return SSQ_EFORMAT;
	}
	// duplicates
	if ((rc = ssq_dupset_mark_dev(s->set, take, s->k1.as<u64>(), s->k2.as<u64>(), s->valid.as<uint8_t>(), s->dup.as<uint8_t>(), st))) return rc;
	// text: sizes, scans, bytes
	for (int k = 0; k < 3; ++k) if (s->len[k].need(((size_t)lines + 1) * 8)) return SSQ_ENOMEM;
	CK(cudaMemsetAsync(s->cnt.p, 0, 3 * 8, st));
	for (int k = 0; k < 3; ++k) CK(cudaMemsetAsync(s->len[k].as<u64>() + lines, 0, 8, st));
	k_sbt_text<false><<<grid_of(lines), SBT_NT, 0, st>>>(s->o, t, L, s->bstart.as<u32>(), lines, s->dup.as<uint8_t>(), s->len[0].as<u64>(), s->len[1].as<u64>(), s->len[2].as<u64>(), 0, 0, 0,
	                                                     s->cnt.as<unsigned long long>());
	CK(cudaGetLastError());
	CK(cub::DeviceScan::ExclusiveSum(0, tb, s->len[0].as<u64>(), s->len[0].as<u64>(), (int)lines + 1, st));
	if (s->tmp.need(tb)) return SSQ_ENOMEM;
	for (int k = 0; k < 3; ++k) CK(cub::DeviceScan::ExclusiveSum(s->tmp.p, tb, s->len[k].as<u64>(), s->len[k].as<u64>(), (int)lines + 1, st));
	u64 tot[3];
	unsigned long long cnt[3];
	for (int k = 0; k < 3; ++k) CK(cudaMemcpyAsync(&tot[k], s->len[k].as<u64>() + lines, 8, cudaMemcpyDeviceToHost, st));
	CK(cudaMemcpyAsync(cnt, s->cnt.p, sizeof cnt, cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	for (int k = 0; k < 3; ++k) {
		if (s->out[k].need(tot[k] + 1)) return SSQ_ENOMEM;
		if (tot[k] > s->h_cap[k]) {
			if (s->h_out[k]) cudaFreeHost(s->h_out[k]);
			s->h_cap[k] = tot[k] + tot[k] / 4 + 4096;
			if (cudaHostAlloc((void**)&s->h_out[k], s->h_cap[k], cudaHostAllocDefault) != cudaSuccess) { s->h_out[k] = 0; s->h_cap[k] = 0; ssq_set_error("cudaHostAlloc failed"); return SSQ_ENOMEM; }
		}
	}
	k_sbt_text<true><<<grid_of(lines), SBT_NT, 0, st>>>(s->o, t, L, s->bstart.as<u32>(), lines, s->dup.as<uint8_t>(), s->len[0].as<u64>(), s->len[1].as<u64>(), s->len[2].as<u64>(),
	                                                    s->out[0].as<char>(), s->out[1].as<char>(), s->out[2].as<char>(), 0);
	CK(cudaGetLastError());
	for (int k = 0; k < 3; ++k) if (tot[k]) CK(cudaMemcpyAsync(s->h_out[k], s->out[k].p, tot[k], cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	for (int k = 0; k < 3; ++k) { out->text[k] = s->h_out[k] ? s->h_out[k] : ""; out->len[k] = tot[k]; }
	out->n_ids = take; out->n_dup = cnt[0]; out->n_split_lines = cnt[1]; out->n_disc_lines = cnt[2];
	*used = consumed;
	return SSQ_OK;
}
