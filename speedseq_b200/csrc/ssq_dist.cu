// ssq_dist.cu — the one real exchange of the `speedseq align` path across GPUs, in C over NCCL (SURVEY.md §8e).
//
// Alignment shards by whole `bwa mem` batches (the only couplings inside alignment are per-batch: insert-size statistics and
// read ordinals), the index is replicated: no collective there.  samblaster's rule "the first pair seen with a signature is kept"
// (`$SAMBLASTER`, speedseq/bin/speedseq:439) is global over the whole input, though.  With N ranks, batches are dealt
// round-robin (round k: rank r works on batch k*N + r); in the duplicate stage of a round every rank
//   1. routes each pair signature (two 64-bit keys) to its OWNER rank = hash(signature) mod N      k_route + stable radix sort by owner
//   2. all-gathers the N x N count matrix, then exchanges the keys with grouped ncclSend/ncclRecv    16 B per pair out
//   3. as owner, marks what it received — laid out by source rank, which within a round IS global input order — against its
//      device-resident set of every signature it has owned so far (ssq_dupset_mark_dev: sort + adjacent-equal + binary search)
//   4. returns one byte per pair to the source with a second grouped send/recv, and the source scatters the bits back
// Equal signatures always meet at the same owner, rounds are processed in order, so the result is exactly the single-GPU result.
// Several stream lanes of one rank share the communicator: the dup stage of batch b waits for the stage of batch b-1
// (ssq_dupset_wait_turn on the owner set), so every rank issues its collectives in the same order.
#include <cuda_runtime.h>
#include <cub/cub.cuh>
#include <nccl.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>
#include "ssq_host.h"

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { ssq_set_error("%s:%d: %s", __FILE__, __LINE__, cudaGetErrorString(e_)); return SSQ_ECUDA; } } while (0)
#define NK(x) do { ncclResult_t r_ = (x); if (r_ != ncclSuccess) { ssq_set_error("%s:%d: NCCL: %s", __FILE__, __LINE__, ncclGetErrorString(r_)); return SSQ_ECUDA; } } while (0)

extern "C" int ssq_dupset_mark_dev(ssq_dupset_t *set, uint64_t n, const uint64_t *d_k1, const uint64_t *d_k2, const uint8_t *d_valid, uint8_t *d_is_dup, void *stream);

struct ssq_comm {
	int device, rank, world;
	ncclComm_t comm;
	ssq_dupset_t *owned; // signatures this rank owns
	DBuf dest, dest_s, idx, idx_s, cnt, allcnt, tmp, sk1, sk2, rk1, rk2, rvalid, rdup, sdup;
	unsigned long long bytes_out, bytes_back, rounds; // traffic of this rank since creation
};

__device__ __forceinline__ u64 mix64(u64 x) { x ^= x >> 33; x *= 0xff51afd7ed558ccdULL; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ULL; x ^= x >> 33; return x; }
// owner of every unit; invalid units (never duplicates) stay with their source and are not sent: owner = world (a bucket of its own)
__global__ void k_route(u64 n, int world, const u64 *__restrict__ k1, const u64 *__restrict__ k2, const uint8_t *__restrict__ valid, u32 *dest, u32 *idx, unsigned long long *cnt)
{
	const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const u32 d = valid[i] ? (u32)(mix64(k1[i] * 0x9e3779b97f4a7c15ULL ^ mix64(k2[i])) % (u64)world) : (u32)world;
	dest[i] = d; idx[i] = (u32)i;
	atomicAdd(&cnt[d], 1ull);
}
__global__ void k_gather_keys(u64 n, const u32 *__restrict__ idx_s, const u64 *__restrict__ k1, const u64 *__restrict__ k2, u64 *o1, u64 *o2)
{
	const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) { const u32 j = idx_s[i]; o1[i] = k1[j]; o2[i] = k2[j]; }
}
__global__ void k_fill_u8(u64 n, uint8_t *p, uint8_t v) { const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x; if (i < n) p[i] = v; }
__global__ void k_scatter_dup(u64 n_sent, u64 n_all, const u32 *__restrict__ idx_s, const uint8_t *__restrict__ back, uint8_t *dup)
{
	const u64 i = (u64)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n_all) return;
	dup[idx_s[i]] = i < n_sent ? back[i] : 0; // the unsent tail = the invalid units
}

extern "C" int ssq_comm_unique_id(void *id128)
{
	ncclUniqueId id;
	if (!id128) return SSQ_EINVAL;
	if (sizeof id != 128) { ssq_set_error("unexpected ncclUniqueId size"); return SSQ_EINVAL; }
	NK(ncclGetUniqueId(&id));
	memcpy(id128, &id, 128);
	return SSQ_OK;
}

extern "C" void ssq_comm_free(ssq_comm_t *c)
{
	if (!c) return;
	cudaSetDevice(c->device);
	if (c->comm) ncclCommDestroy(c->comm);
	if (c->owned) ssq_dupset_free(c->owned);
	delete c;
}

extern "C" int ssq_comm_create(const void *id128, int rank, int world, int device, ssq_comm_t **out)
{
	if (!id128 || !out || world < 1 || rank < 0 || rank >= world) return SSQ_EINVAL;
	int rc = ssq_use_device(device);
	if (rc) return rc;
	ssq_comm *c = new ssq_comm();
	c->device = device; c->rank = rank; c->world = world; c->comm = 0; c->owned = 0; c->bytes_out = c->bytes_back = c->rounds = 0;
	ncclUniqueId id;
	memcpy(&id, id128, 128);
	if (ncclCommInitRank(&c->comm, world, id, rank) != ncclSuccess) { ssq_set_error("ncclCommInitRank failed (rank %d of %d)", rank, world); delete c; return SSQ_ECUDA; }
	if ((rc = ssq_dupset_create(device, &c->owned))) { ssq_comm_free(c); return rc; }
	*out = c;
	return SSQ_OK;
}
extern "C" ssq_dupset_t *ssq_comm_dupset(ssq_comm_t *c) { return c ? c->owned : 0; }
extern "C" uint64_t ssq_comm_counter(const ssq_comm_t *c, int what) { return !c ? 0 : what == 0 ? c->bytes_out : what == 1 ? c->bytes_back : what == 2 ? c->rounds : 0; }

// one round of the exchange; collective: every rank of the communicator calls it, in the same order of rounds
extern "C" int ssq_comm_mark_round(ssq_comm_t *c, uint64_t n, const uint64_t *d_k1, const uint64_t *d_k2, const uint8_t *d_valid, uint8_t *d_is_dup, void *stream_)
{
	if (!c) return SSQ_EINVAL;
	int rc = ssq_use_device(c->device);
	if (rc) return rc;
	if (n >= 0x7fffffffull) { ssq_set_error("ssq_comm_mark_round: more than 2^31-1 pairs in one round"); return SSQ_EINVAL; }
	cudaStream_t st = (cudaStream_t)stream_;
	const int W = c->world;
	const unsigned g = (unsigned)((n + 255) / 256);
	if (c->dest.need((n + 1) * 4) || c->dest_s.need((n + 1) * 4) || c->idx.need((n + 1) * 4) || c->idx_s.need((n + 1) * 4) || c->cnt.need((W + 1) * 8) || c->allcnt.need((size_t)W * (W + 1) * 8) ||
	    c->sk1.need((n + 1) * 8) || c->sk2.need((n + 1) * 8) || c->sdup.need(n + 16)) return SSQ_ENOMEM;
	CK(cudaMemsetAsync(c->cnt.p, 0, (W + 1) * 8, st));
	if (n) {
		k_route<<<g, 256, 0, st>>>(n, W, d_k1, d_k2, d_valid, c->dest.as<u32>(), c->idx.as<u32>(), (unsigned long long*)c->cnt.p);
		size_t tb = 0;
		cub::DeviceRadixSort::SortPairs(0, tb, c->dest.as<u32>(), c->dest_s.as<u32>(), c->idx.as<u32>(), c->idx_s.as<u32>(), (int)n, 0, 4, st);
		if (c->tmp.need(tb)) return SSQ_ENOMEM;
		CK(cub::DeviceRadixSort::SortPairs(c->tmp.p, tb, c->dest.as<u32>(), c->dest_s.as<u32>(), c->idx.as<u32>(), c->idx_s.as<u32>(), (int)n, 0, 4, st)); // stable: input order kept inside every bucket
		k_gather_keys<<<g, 256, 0, st>>>(n, c->idx_s.as<u32>(), d_k1, d_k2, c->sk1.as<u64>(), c->sk2.as<u64>());
	}
	// count matrix: row r = what rank r sends to each owner
	NK(ncclAllGather(c->cnt.p, c->allcnt.p, (size_t)(W + 1), ncclUint64, c->comm, st));
	std::vector<u64> m((size_t)W * (W + 1));
	CK(cudaMemcpyAsync(m.data(), c->allcnt.p, m.size() * 8, cudaMemcpyDeviceToHost, st));
	CK(cudaStreamSynchronize(st));
	std::vector<u64> soff(W + 1, 0), roff(W + 1, 0);
	for (int p = 0; p < W; ++p) { soff[p + 1] = soff[p] + m[(size_t)c->rank * (W + 1) + p]; roff[p + 1] = roff[p] + m[(size_t)p * (W + 1) + c->rank]; }
	const u64 n_sent = soff[W], n_recv = roff[W];
	if (n_recv >= 0x7fffffffull) { ssq_set_error("ssq_comm_mark_round: an owner received more than 2^31-1 signatures in one round"); return SSQ_EINVAL; }
	if (c->rk1.need((n_recv + 1) * 8) || c->rk2.need((n_recv + 1) * 8) || c->rvalid.need(n_recv + 16) || c->rdup.need(n_recv + 16)) return SSQ_ENOMEM;
	NK(ncclGroupStart());
	for (int p = 0; p < W; ++p) {
		const u64 ns = soff[p + 1] - soff[p], nr = roff[p + 1] - roff[p];
		if (ns) { NK(ncclSend(c->sk1.as<u64>() + soff[p], ns, ncclUint64, p, c->comm, st)); NK(ncclSend(c->sk2.as<u64>() + soff[p], ns, ncclUint64, p, c->comm, st)); }
		if (nr) { NK(ncclRecv(c->rk1.as<u64>() + roff[p], nr, ncclUint64, p, c->comm, st)); NK(ncclRecv(c->rk2.as<u64>() + roff[p], nr, ncclUint64, p, c->comm, st)); }
	}
	NK(ncclGroupEnd());
	// owner side: the receive buffer is laid out by source rank = global input order within the round
	if (n_recv) {
		k_fill_u8<<<(unsigned)((n_recv + 255) / 256), 256, 0, st>>>(n_recv, c->rvalid.as<uint8_t>(), 1);
		if ((rc = ssq_dupset_mark_dev(c->owned, n_recv, c->rk1.as<u64>(), c->rk2.as<u64>(), c->rvalid.as<uint8_t>(), c->rdup.as<uint8_t>(), (void*)st))) return rc;
	}
	NK(ncclGroupStart());
	for (int p = 0; p < W; ++p) {
		const u64 ns = soff[p + 1] - soff[p], nr = roff[p + 1] - roff[p];
		if (nr) NK(ncclSend(c->rdup.as<uint8_t>() + roff[p], nr, ncclUint8, p, c->comm, st));
		if (ns) NK(ncclRecv(c->sdup.as<uint8_t>() + soff[p], ns, ncclUint8, p, c->comm, st));
	}
	NK(ncclGroupEnd());
	if (n) k_scatter_dup<<<g, 256, 0, st>>>(n_sent, n, c->idx_s.as<u32>(), c->sdup.as<uint8_t>(), d_is_dup);
	CK(cudaGetLastError());
	CK(cudaStreamSynchronize(st));
	c->bytes_out += 16 * (n_sent - m[(size_t)c->rank * (W + 1) + c->rank]); c->bytes_back += n_sent - m[(size_t)c->rank * (W + 1) + c->rank]; ++c->rounds;
	return SSQ_OK;
}
