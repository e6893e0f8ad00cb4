// sw_host.cpp — TEST-ONLY: the scalar Smith-Waterman routines the device kernels are held to, run on the host with any scoring:
// sw_global (banded global DP + traceback, ssq_dev2.cuh) on the task layout of ssq_sw_global_batch, sw_local (the striped kernel's
// evaluation order, ssq_dev2.cuh) on that of ssq_sw_local_batch, and sw_extend (ssq_dev.cuh) on that of ssq_sw_extend_batch.
// sc = {a, b, o_del, e_del, o_ins, e_ins}.  build: see tests/test_sw_kernels_cpu.py
#include <string.h>
#include <vector>
#include "../../speedseq_b200/csrc/ssq_dev2.cuh"

static ssq_opts_t scoring(const int32_t *sc)
{
	ssq_opts_t o;
	memset(&o, 0, sizeof o);
	o.a = sc[0]; o.b = sc[1]; o.o_del = sc[2]; o.e_del = sc[3]; o.o_ins = sc[4]; o.e_ins = sc[5];
	return o;
}

extern "C" {

// same task checks as ssq_sw_global_batch (buffer lengths aside: the caller passes none)
int swhost_global_batch(const int32_t *sc, uint64_t n, const ssq_swg_task_t *t, const uint8_t *qbuf, const uint8_t *tbuf, uint32_t *cig, ssq_swg_result_t *r)
{
	const ssq_opts_t opt = scoring(sc);
	for (uint64_t i = 0; i < n; ++i) {
		const int dl = t[i].tlen > t[i].qlen ? t[i].tlen - t[i].qlen : t[i].qlen - t[i].tlen;
		if (t[i].qlen < 1 || t[i].qlen > SSQ_MAX_READ_LEN || t[i].tlen < 1 || t[i].tlen > 2048 || t[i].w < 0 || dl > t[i].w || t[i].cig_cap < 0) return SSQ_EINVAL;
	}
	for (uint64_t i = 0; i < n; ++i) {
		const int qlen = t[i].qlen, tlen = t[i].tlen, w = t[i].w < qlen + tlen ? t[i].w : qlen + tlen, n_col = qlen < 2 * w + 1 ? qlen : 2 * w + 1;
		std::vector<i32> h(qlen + 2), e(qlen + 2);
		std::vector<uint8_t> z(t[i].cig_cap ? (size_t)n_col * tlen : 0);
		GlobalScratch S; S.h = h.data(); S.e = e.data(); S.z = t[i].cig_cap ? z.data() : 0; S.zcap = (long)z.size();
		int n_cig = 0;
		r[i].score = sw_global(opt, qlen, qbuf + t[i].q_off, tlen, tbuf + t[i].t_off, w, S, t[i].cig_cap ? cig + t[i].cig_off : 0, t[i].cig_cap, &n_cig);
		r[i].n_cigar = n_cig;
	}
	return 0;
}

int swhost_local_batch(const int32_t *sc, uint64_t n, const ssq_swl_task_t *t, const uint8_t *qbuf, const uint8_t *tbuf, ssq_swl_result_t *r)
{
	const ssq_opts_t opt = scoring(sc);
	for (uint64_t i = 0; i < n; ++i) {
		std::vector<uint8_t> q(qbuf + t[i].q_off, qbuf + t[i].q_off + t[i].qlen), tg(tbuf + t[i].t_off, tbuf + t[i].t_off + t[i].tlen);
		q.resize(t[i].qlen + 1); tg.resize(t[i].tlen + 1); // (sw_local reverses prefixes in place and restores them)
		std::vector<i32> H0(t[i].qlen + 32), H1(t[i].qlen + 32), E(t[i].qlen + 32), Hm(t[i].qlen + 32);
		std::vector<u64> b(t[i].tlen + 1);
		LocalScratch L; L.H0 = H0.data(); L.H1 = H1.data(); L.E = E.data(); L.Hmax = Hm.data(); L.b = b.data(); L.b_cap = t[i].tlen > 1 ? t[i].tlen : 1;
		const LocalRes x = sw_local(opt, t[i].qlen, q.data(), t[i].tlen, tg.data(), t[i].xtra, L);
		r[i].score = x.score; r[i].te = x.te; r[i].qe = x.qe; r[i].score2 = x.score2; r[i].te2 = x.te2; r[i].tb = x.tb; r[i].qb = x.qb;
	}
	return 0;
}

int swhost_extend_batch(const int32_t *sc, uint64_t n, const ssq_sw_task_t *t, const uint8_t *qbuf, const uint8_t *tbuf, ssq_sw_result_t *r)
{
	const ssq_opts_t opt = scoring(sc);
	for (uint64_t i = 0; i < n; ++i) {
		std::vector<u32> ehbuf(t[i].qlen + 4);
		EhAcc eh; eh.base = ehbuf.data(); eh.stride = 1;
		const uint8_t *q = qbuf + t[i].q_off, *tg = tbuf + t[i].t_off;
		unsigned long long cells = 0;
		r[i].score = sw_extend(opt, t[i].qlen, [&](int j) { return (int)q[j]; }, t[i].tlen, [&](int k) { return (int)tg[k]; }, t[i].w, t[i].end_bonus, t[i].zdrop, t[i].h0, eh,
		                       r[i].qle, r[i].tle, r[i].gtle, r[i].gscore, r[i].max_off, cells);
	}
	return 0;
}
}
